// ag_math.cuh — fp32 vector / quaternion helpers for the sm_90a kernels.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define AG_HD __host__ __device__ __forceinline__
#define AG_HDN __host__ __device__
#else
#define AG_HD inline
#define AG_HDN
#endif

#if defined(__CUDA_ARCH__)
#define AG_LDG(p) __ldg(p)
#else
#define AG_LDG(p) (*(p))
#endif

struct f3 {
  float x, y, z;
  AG_HD f3() : x(0.f), y(0.f), z(0.f) {}
  AG_HD f3(float a, float b, float c) : x(a), y(b), z(c) {}
};
AG_HD f3 operator+(f3 a, f3 b) { return f3(a.x + b.x, a.y + b.y, a.z + b.z); }
AG_HD f3 operator-(f3 a, f3 b) { return f3(a.x - b.x, a.y - b.y, a.z - b.z); }
AG_HD f3 operator-(f3 a) { return f3(-a.x, -a.y, -a.z); }
AG_HD f3 operator*(f3 a, float s) { return f3(a.x * s, a.y * s, a.z * s); }
AG_HD f3 operator*(float s, f3 a) { return f3(a.x * s, a.y * s, a.z * s); }
AG_HD f3& operator+=(f3& a, f3 b) { a.x += b.x; a.y += b.y; a.z += b.z; return a; }
AG_HD f3& operator-=(f3& a, f3 b) { a.x -= b.x; a.y -= b.y; a.z -= b.z; return a; }
AG_HD float dot(f3 a, f3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
AG_HD f3 cross(f3 a, f3 b) { return f3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
AG_HD float norm(f3 a) { return sqrtf(dot(a, a)); }
AG_HD float comp(f3 a, int i) { return i == 0 ? a.x : (i == 1 ? a.y : a.z); }
AG_HD f3 fmin3(f3 a, f3 b) { return f3(fminf(a.x, b.x), fminf(a.y, b.y), fminf(a.z, b.z)); }
AG_HD f3 fmax3(f3 a, f3 b) { return f3(fmaxf(a.x, b.x), fmaxf(a.y, b.y), fmaxf(a.z, b.z)); }
AG_HD float clampf(float v, float lo, float hi) { return fminf(hi, fmaxf(lo, v)); }

// double-precision 3-vector: used only inside the GJK simplex solve (a handful of flops per
// iteration), where fp32 cancellation on thin simplices of far-apart support points is fatal
struct d3 {
  double x, y, z;
  AG_HD d3() : x(0.0), y(0.0), z(0.0) {}
  AG_HD d3(double a, double b, double c) : x(a), y(b), z(c) {}
};
AG_HD d3 operator+(d3 a, d3 b) { return d3(a.x + b.x, a.y + b.y, a.z + b.z); }
AG_HD d3 operator-(d3 a, d3 b) { return d3(a.x - b.x, a.y - b.y, a.z - b.z); }
AG_HD d3 operator-(d3 a) { return d3(-a.x, -a.y, -a.z); }
AG_HD d3 operator*(d3 a, double s) { return d3(a.x * s, a.y * s, a.z * s); }
AG_HD double dot(d3 a, d3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
AG_HD d3 cross(d3 a, d3 b) { return d3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x); }
AG_HD d3 to_d3(f3 a) { return d3((double)a.x, (double)a.y, (double)a.z); }
AG_HD f3 to_f3(d3 a) { return f3((float)a.x, (float)a.y, (float)a.z); }

struct q4 {
  float x, y, z, w;
  AG_HD q4() : x(0.f), y(0.f), z(0.f), w(1.f) {}
  AG_HD q4(float a, float b, float c, float d) : x(a), y(b), z(c), w(d) {}
};
AG_HD q4 qmul(q4 a, q4 b) {
  return q4(a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x,
            a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w,
            a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z);
}
AG_HD q4 qconj(q4 q) { return q4(-q.x, -q.y, -q.z, q.w); }
AG_HD q4 qnormalize(q4 q) {
  float s = 1.0f / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  return q4(q.x * s, q.y * s, q.z * s, q.w * s);
}
AG_HD f3 qrot(q4 q, f3 v) {
  f3 u(q.x, q.y, q.z);
  f3 t = cross(u, v) * 2.0f;
  return v + t * q.w + cross(u, t);
}
AG_HD f3 qrot_inv(q4 q, f3 v) { return qrot(qconj(q), v); }
AG_HD q4 qaxis(f3 a, float ang) {
  float s, c;
#if defined(__CUDA_ARCH__)
  sincosf(0.5f * ang, &s, &c);
#else
  s = sinf(0.5f * ang); c = cosf(0.5f * ang);
#endif
  return q4(a.x * s, a.y * s, a.z * s, c);
}
AG_HD q4 qexp(f3 w) {   // rotation by vector w
  float a = norm(w);
  if (a < 1e-6f) return qnormalize(q4(0.5f * w.x, 0.5f * w.y, 0.5f * w.z, 1.0f));
  float s = sinf(0.5f * a) / a;
  return q4(w.x * s, w.y * s, w.z * s, cosf(0.5f * a));
}

// 3x3 matrix (row major)
struct m3 {
  float m[9];
  AG_HD float& operator()(int r, int c) { return m[3 * r + c]; }
  AG_HD float operator()(int r, int c) const { return m[3 * r + c]; }
};
AG_HD m3 qmat(q4 q) {
  m3 r;
  float x = q.x, y = q.y, z = q.z, w = q.w;
  r.m[0] = 1 - 2 * (y * y + z * z); r.m[1] = 2 * (x * y - z * w); r.m[2] = 2 * (x * z + y * w);
  r.m[3] = 2 * (x * y + z * w); r.m[4] = 1 - 2 * (x * x + z * z); r.m[5] = 2 * (y * z - x * w);
  r.m[6] = 2 * (x * z - y * w); r.m[7] = 2 * (y * z + x * w); r.m[8] = 1 - 2 * (x * x + y * y);
  return r;
}
AG_HD f3 mul(const m3& a, f3 v) {
  return f3(a.m[0] * v.x + a.m[1] * v.y + a.m[2] * v.z, a.m[3] * v.x + a.m[4] * v.y + a.m[5] * v.z, a.m[6] * v.x + a.m[7] * v.y + a.m[8] * v.z);
}
AG_HD f3 mulT(const m3& a, f3 v) {
  return f3(a.m[0] * v.x + a.m[3] * v.y + a.m[6] * v.z, a.m[1] * v.x + a.m[4] * v.y + a.m[7] * v.z, a.m[2] * v.x + a.m[5] * v.y + a.m[8] * v.z);
}
AG_HD m3 mul(const m3& a, const m3& b) {
  m3 r;
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r.m[3 * i + j] = a.m[3 * i] * b.m[j] + a.m[3 * i + 1] * b.m[3 + j] + a.m[3 * i + 2] * b.m[6 + j];
  return r;
}
AG_HD m3 transpose(const m3& a) { m3 r; for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) r.m[3 * i + j] = a.m[3 * j + i]; return r; }

// symmetric 3x3 stored as xx, yy, zz, xy, xz, yz
struct s3 {
  float xx, yy, zz, xy, xz, yz;
};
AG_HD f3 mul(const s3& a, f3 v) {
  return f3(a.xx * v.x + a.xy * v.y + a.xz * v.z, a.xy * v.x + a.yy * v.y + a.yz * v.z, a.xz * v.x + a.yz * v.y + a.zz * v.z);
}
// R * S * R^T for symmetric S
AG_HD s3 rot_sym(const m3& R, const s3& S) {
  f3 c0 = mul(S, f3(R.m[0], R.m[1], R.m[2]));   // S * row0(R)^T
  f3 c1 = mul(S, f3(R.m[3], R.m[4], R.m[5]));
  f3 c2 = mul(S, f3(R.m[6], R.m[7], R.m[8]));
  f3 r0(R.m[0], R.m[1], R.m[2]), r1(R.m[3], R.m[4], R.m[5]), r2(R.m[6], R.m[7], R.m[8]);
  s3 o;
  o.xx = dot(r0, c0); o.yy = dot(r1, c1); o.zz = dot(r2, c2);
  o.xy = dot(r0, c1); o.xz = dot(r0, c2); o.yz = dot(r1, c2);
  return o;
}
AG_HD s3 inverse_sym(const s3& a) {
  float c00 = a.yy * a.zz - a.yz * a.yz, c01 = a.xz * a.yz - a.xy * a.zz, c02 = a.xy * a.yz - a.xz * a.yy;
  float det = a.xx * c00 + a.xy * c01 + a.xz * c02;
  float id = 1.0f / det;
  s3 o;
  o.xx = c00 * id; o.xy = c01 * id; o.xz = c02 * id;
  o.yy = (a.xx * a.zz - a.xz * a.xz) * id; o.yz = (a.xz * a.xy - a.xx * a.yz) * id;
  o.zz = (a.xx * a.yy - a.xy * a.xy) * id;
  return o;
}

// orthonormal tangent pair for a unit normal (fixed rule; any rule works as long as it is deterministic)
AG_HD void plane_space(f3 n, f3& t1, f3& t2) {
  if (fabsf(n.z) > 0.70710678f) {
    float a = n.y * n.y + n.z * n.z; float k = 1.0f / sqrtf(a);
    t1 = f3(0.f, -n.z * k, n.y * k);
    t2 = f3(a * k, -n.x * t1.z, n.x * t1.y);
  } else {
    float a = n.x * n.x + n.y * n.y; float k = 1.0f / sqrtf(a);
    t1 = f3(-n.y * k, n.x * k, 0.f);
    t2 = f3(-n.z * t1.y, n.z * t1.x, a * k);
  }
}
