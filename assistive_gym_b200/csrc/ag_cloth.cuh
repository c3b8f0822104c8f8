// ag_cloth.cuh — K8: the cloth of the Dressing task (reference envs/dressing.py:25 getSoftBodyData, :146-154 loadCloth /
// clothParams, :184 numSubSteps = 8, :210 the attachment teleported to the end effector).
//
// What it restates (Bullet's btSoftBody position-based solver, recalled -- DESIGN.md section 9; every coefficient is a
// field of AgClothDesc): per substep of dt/numSubSteps
//   predictMotion:   v += g dt; aerodynamic drag (kDG, V_Point model incl. ApplyClampedForce); q = x; x += v dt
//   collisions:      node vs rigid shapes at the START-of-substep link poses, signed distance < margin -> rigid contact
//                    (normal, plane offset, friction switch c3 from the predicted motion)
//   position solver: piterations x [anchors (kAHR), rigid contacts (kCHR / kKHR, kDF), links (kLST) in list order]
//   velocities:      v = (x - q) / dt * (1 - kDP)
// Multibody link colliders are not btRigidBody, so Bullet of the reference's era treats them as static shapes with zero
// velocity: the coupling is one way (cloth feels the bodies, bodies do not feel the cloth).  That is what makes the GPU
// mapping below possible: the rigid substeps of one stepSimulation run first and leave the link poses of every substep in
// a snapshot buffer; ONE launch of k_cloth then advances the cloth through all numSubSteps substeps.
//
// GPU mapping.  One CTA of 1024 threads per env, the env's node positions resident in shared memory as float4 (64 KB) for
// the whole launch; previous positions q and velocities v of a thread's own nodes (node = k * 1024 + thread) live in its
// registers.  HBM traffic per env and launch: x and v read once and written once (190 KB) instead of once per substep.
// Links are relaxed colour by colour (links of one colour share no node; the list is colour-major, so this is the
// sequential Gauss-Seidel sweep of the list), one __syncthreads per colour.  Contacts are found by the owner thread of a
// node, slots are assigned by a block-wide prefix sum (deterministic order), solved by the owner thread.
#pragma once
#include "ag_device.cuh"

#define AG_CLOTH_T 1024          // threads per CTA (= envs are independent CTAs)
#define AG_CLOTH_MAXANCH 8
#define AG_CLOTH_MAXCL 96        // collider links per env
#define AG_CLOTH_MAXCOL 16       // link colours
#define AG_CLOTH_HITS 24         // contacts one thread can find per substep (over its <= NPT nodes)
#define AG_CLOTH_EPS 1.1920929e-7f
#define AG_CLOTH_LKS 24          // floats per collider link in shared memory: R 9, pos 3, bounding sphere 4, round shape: a 3, b 3, r, flag
#define AG_CLOTH_CCF 8           // floats per exported contact: node, x, y, z, fx, fy, fz, link

struct alignas(8) ClothLinkRec { unsigned ij; float rest2; };

struct ClothDev {
  int nn, nnp, nlinks, ncol, nanch, ncl, maxcc, K, piters, export_contacts;
  float dt, im, kLSTh, kDP, kDG, kLF, kDF, kCHR, kKHR, kAHR, margin, density;
  float gx, gy, gz;
  int col_off[AG_CLOTH_MAXCOL + 1];          // colour c = links [col_off[c], col_off[c + 1]) of link_ij / link_rest2 (list order)
  int tab_off[AG_CLOTH_MAXCOL], tab_end[AG_CLOTH_MAXCOL];   // the same colour inside link_tab: starts aligned to 32 entries (aligned quarter-warps)
  int anch_node[AG_CLOTH_MAXANCH];
  float anch_local[AG_CLOTH_MAXANCH][3];
  // template tables
  const unsigned* link_ij;     // [nlinks] node i | node j << 16, colour-major
  const float* link_rest2;     // [nlinks]
  const struct ClothLinkRec* link_tab;   // [nlinks] the two above interleaved (one 8-byte load per link)
  const struct ClothLinkRec* link_dense; // [ncol + 1][AG_CLOTH_T] one row per colour, thread t relaxes entry t; no link: ij = ~0.  Null if a colour is larger than the block
  const int* nf_off;           // [nn + 1]
  const unsigned* nf_pair;     // [nf] next | next-next << 16 (face winding)
  const float* node_area;      // [nn]
  const int* cl_link;          // [ncl] global link ids of the rigid links the cloth collides with
  const float* cl_bs;          // [ncl][4] bounding sphere of the link's colliders in the link frame
  const int* cl_static;        // [ncl] 1: static shape (kKHR), 0: movable (kCHR)
  // per-env state
  float* x;                    // [N][3][nnp]
  float* v;                    // [N][3][nnp]
  float* anchor_pos;           // [3][N] position of the (kinematic, identity-orientation) anchor body
  float* snap;                 // [K][ncl][7][N] link poses at the start of each substep
  // outputs of the last substep of a launch
  int* cc_count;               // [N]
  float* cc_data;              // [N][maxcc][AG_CLOTH_CCF]
  int* overflow;               // [N]
};

struct ClothContact { f3 n; float offset, c3, c4; f3 acc; int node, link; };

// signed distance of a point (link frame) to the union of the link's colliders, outward normal of the nearest one
// (colliders whose bounding box is farther than `reach` from the point are skipped: they cannot produce a distance below `reach`,
//  and only distances below the collision margin matter to the caller -- a link of the wheelchair is 44 hulls, one of PR2's up to 100 planes)
AG_HDN inline float cloth_sdf_link(const SimDev& S, int link, f3 p, f3& nrm, float reach = 1e30f, unsigned long long cmask = ~0ull, int* cbest = nullptr) {
  int c0 = AG_LDG(S.link_col0 + link), nc = AG_LDG(S.link_ncol + link);
  float best = 1e30f;
  nrm = f3(0.f, 0.f, 1.f);
  // colliders culled for the caller's whole warp (k_cloth) are not even visited: the loop walks the set bits of the mask (the first 64
  // colliders of the link; further ones are always visited), in ascending order
  unsigned long long todo = nc >= 64 ? cmask : (cmask & ((1ull << nc) - 1ull));
  int tail = nc > 64 ? 64 : nc;                       // [tail, nc): beyond the mask
  while (todo || tail < nc) {
    int c;
    if (todo) {
#if defined(__CUDA_ARCH__)
      c = c0 + __ffsll((long long)todo) - 1;
#else
      c = c0 + __builtin_ctzll(todo);
#endif
      todo &= todo - 1;
    } else c = c0 + tail++;
    int type = AG_LDG(S.col_type + c), v0 = AG_LDG(S.col_v0 + c);
    float r = AG_LDG(S.col_radius + c), d; f3 n;
    f3 bq(0.f, 0.f, 0.f);                     // signed per-axis distance of the point to the core's bounding box (link frame)
    if (type != 3) {
      f3 bc = tv3(S.col_center, c), bh = tv3(S.col_half, c);
      bq = f3(fabsf(p.x - bc.x) - bh.x, fabsf(p.y - bc.y) - bh.y, fabsf(p.z - bc.z) - bh.z);
      float lim = reach + r;
      if (type == 2) { if (fmaxf(bq.x, fmaxf(bq.y, bq.z)) > lim) continue; }        // hulls measure with planes: per-axis test (see below)
      else { f3 qc = fmax3(bq, f3(0.f, 0.f, 0.f)); if (dot(qc, qc) > lim * lim) continue; }
    }
    if (type == 0 /*sphere*/ || type == 1 /*capsule*/) {
      f3 a = tv3(S.verts, v0), cp = a;
      if (type == 1) {
        f3 ab = tv3(S.verts, v0 + 1) - a;
        float t = clampf(dot(p - a, ab) / fmaxf(dot(ab, ab), 1e-20f), 0.f, 1.f);
        cp = a + ab * t;
      }
      f3 w = p - cp; float L = norm(w);
      d = L - r; n = L > 1e-12f ? w * (1.f / L) : f3(0.f, 0.f, 1.f);
    } else {
      // hull / half-space: the plane the point is farthest outside of -- the hull's face planes and, for hulls, the six planes of
      // the core's bounding box (the box contains the hull, so this only tightens the lower bound outside and changes nothing inside)
      // A plane the point is farther outside of than `reach` (+ the rounding radius) ends the walk: the maximum can only grow, so this
      // collider cannot yield a distance below `reach` -- the same argument as the box test above.  Most nodes near a 124-plane gripper
      // hull are outside its margin shell and leave after a few planes.
      int p0 = AG_LDG(S.col_p0 + c), np = AG_LDG(S.col_np + c);
      float m = -1e30f; n = f3(0.f, 0.f, 1.f);
      const float lim = reach + r;
      bool sep = false;
      for (int k = p0; k < p0 + np && !sep; k += 4) {            // four planes per trip: their loads are in flight together
        f3 pn[4]; float sd[4];
#pragma unroll
        for (int j = 0; j < 4; j++) { int kk = k + j < p0 + np ? k + j : p0 + np - 1; float pd; ld_plane(S.planes, kk, pn[j], pd); sd[j] = dot(pn[j], p) - pd; }
#pragma unroll
        for (int j = 0; j < 4; j++) if (sd[j] > m) { m = sd[j]; n = pn[j]; }      // (a repeated last plane changes nothing: strict >)
        sep = m > lim;
      }
      if (sep) continue;
      if (type == 2) {
        f3 bc = tv3(S.col_center, c);
        if (bq.x > m) { m = bq.x; n = f3(p.x >= bc.x ? 1.f : -1.f, 0.f, 0.f); }
        if (bq.y > m) { m = bq.y; n = f3(0.f, p.y >= bc.y ? 1.f : -1.f, 0.f); }
        if (bq.z > m) { m = bq.z; n = f3(0.f, 0.f, p.z >= bc.z ? 1.f : -1.f); }
      }
      d = m - r;
    }
    if (d < best) { best = d; nrm = n; if (cbest) *cbest = c - c0; }
  }
  return best;
}

struct ClothLinkPose { m3 R; f3 pos; f3 bc; float br; };   // world pose of a collider link + its bounding sphere (margin included)

AG_HD ClothLinkPose cloth_link_pose(const ClothDev& C, int sub, int L, int N, int e) {
  const float* s = C.snap + ((size_t)(sub * C.ncl + L) * 7) * N + e;
  ClothLinkPose P;
  P.pos = f3(s[0], s[(size_t)N], s[2 * (size_t)N]);
  P.R = qmat(q4(s[3 * (size_t)N], s[4 * (size_t)N], s[5 * (size_t)N], s[6 * (size_t)N]));
  f3 bl(AG_LDG(C.cl_bs + 4 * L), AG_LDG(C.cl_bs + 4 * L + 1), AG_LDG(C.cl_bs + 4 * L + 2));
  P.bc = P.pos + mul(P.R, bl); P.br = AG_LDG(C.cl_bs + 4 * L + 3) + C.margin;
  return P;
}
// links of a body that is switched off in this env (the other-gender person) do not exist for the cloth
AG_HD bool cloth_link_active(const SimDev& S, const ClothDev& C, int L, int N, int e) {
  return S.body_mode[(size_t)AG_LDG(S.link_body + AG_LDG(C.cl_link + L)) * N + e] != 0;
}

// the contact record of a node at signed distance `dst` (margin already subtracted) from a shape with outward normal n
AG_HD void cloth_contact_fill(const SimDev& S, const ClothDev& C, int L, int link, int N, int e, f3 x, f3 q, f3 n, float dst, ClothContact& c) {
  c.n = n;
  c.offset = -dot(c.n, x - c.n * dst);
  f3 vr = x - q;                                   // va = 0 (static shape)
  float dn = dot(vr, c.n);
  f3 fv = vr - c.n * dn;
  float fc = C.kDF * S.friction[(size_t)link * N + e];
  c.c3 = dot(fv, fv) < (dn * fc) * (dn * fc) ? 0.f : 1.f - fc;
  c.c4 = AG_LDG(C.cl_static + L) ? C.kKHR : C.kCHR;
  c.acc = f3(0.f, 0.f, 0.f);
  c.link = link;
}
// node vs collider link L (Bullet btSoftColliders::CollideSDF_RS::DoNode + btSoftBody::checkContact, static shape)
// (cbest, if given, receives the index within the link of the collider that made the contact: evaluating that collider alone --
//  cmask = 1 << index -- reproduces the same record, which is how k_cloth writes the records after the slots are known)
AG_HD bool cloth_detect(const SimDev& S, const ClothDev& C, const ClothLinkPose& P, int L, int N, int e, f3 x, f3 q, ClothContact& c, unsigned long long cmask = ~0ull, int* cbest = nullptr) {
  f3 w = x - P.bc;
  if (!(P.br > 0.f) || dot(w, w) > P.br * P.br) return false;
  int link = AG_LDG(C.cl_link + L);
  f3 nl;
  float dst = cloth_sdf_link(S, link, mulT(P.R, x - P.pos), nl, C.margin, cmask, cbest) - C.margin;
  if (!(dst < 0.f)) return false;
  cloth_contact_fill(S, C, L, link, N, e, x, q, mul(P.R, nl), dst, c);
  return true;
}
// the same for a link that is ONE sphere or capsule (most links of the person), given in world space (a, b: the core's end points,
// r: its radius): the exact distance without the trip through the link frame, and a cheap rejection
AG_HD bool cloth_detect_round(const SimDev& S, const ClothDev& C, f3 a, f3 b, float r, int L, int N, int e, f3 x, f3 q, ClothContact& c) {
  f3 ab = b - a;
  float t = clampf(dot(x - a, ab) / fmaxf(dot(ab, ab), 1e-20f), 0.f, 1.f);
  f3 w = x - (a + ab * t);
  float d2 = dot(w, w), lim = r + C.margin;
  if (!(d2 < lim * lim)) return false;
  float Ln = sqrtf(d2), dst = Ln - r - C.margin;
  if (!(dst < 0.f)) return false;
  cloth_contact_fill(S, C, L, AG_LDG(C.cl_link + L), N, e, x, q, Ln > 1e-12f ? w * (1.f / Ln) : f3(0.f, 0.f, 1.f), dst, c);
  return true;
}

// btSoftBody::PSolve_RContacts for one contact of a node (c0 * c2 = identity for a static shape)
AG_HD void cloth_contact_solve(f3& x, f3 q, f3 n, float offset, float c3, float c4, float mrg, f3& acc) {
  f3 vr = x - q;
  float dn = dot(vr, n);
  if (dn <= AG_CLOTH_EPS) {
    float dp = fminf(dot(x, n) + offset, mrg);
    f3 fv = vr - n * dn;
    f3 d = vr - fv * c3 + n * (dp * c4);
    x -= d; acc += d;
  }
}
// btSoftBody::PSolve_Anchors for a static, identity-orientation anchor body at `ap`
AG_HD void cloth_anchor_solve(f3& x, f3 q, f3 wa, float kAHR) { x += (q - x) + (wa - x) * kAHR; }

// btSoftBody::predictMotion for one node: gravity, aerodynamics (addAeroForceToNode, V_Point; the reference sets kDG = 10),
// explicit Euler.  `nrm` is the node normal of the start-of-substep configuration (normalised sum of face cross products).
AG_HD void cloth_predict(const ClothDev& C, f3 nrm, float area, f3& x, f3& v) {
  const float dt = C.dt;
  v += f3(C.gx, C.gy, C.gz) * dt;
  f3 f(0.f, 0.f, 0.f);
  float v2 = dot(v, v);
  if ((C.kDG > 0.f || C.kLF > 0.f) && v2 > AG_CLOTH_EPS) {
    f3 vn = v * (1.f / sqrtf(v2));
    float dvn = dot(v, nrm);
    if (dvn < 0.f) { nrm = -nrm; dvn = -dvn; }       // Bullet flips the normal towards the flow for every V_ model
    if (dvn > 0.f) {
      float c1 = area * dvn * v2 * 0.5f * C.density;
      f3 force = nrm * (-c1 * C.kLF) + vn * (-c1 * C.kDG);
      float dtim = dt * C.im;
      f3 fd = force * dtim;
      if (dot(fd, fd) > v2) {                          // ApplyClampedForce: never reverse the velocity
        f3 fn = force * (1.f / norm(force));
        f -= fn * (dot(v, fn) / dtim);
      } else f += force;
    }
  }
  v += f * (C.im * dt);
  x += v * dt;
}

// btSoftBody::PSolve_Links for one link, uniform node mass: c0 = 2 im / kLST, k im = (c1 - len) / (c1 + len) * kLST / 2
AG_HD void cloth_link_solve(f3& a, f3& b, float rest2, float kLSTh) {
  f3 del = b - a;
  float len = dot(del, del), sum = rest2 + len;
#if defined(__CUDA_ARCH__)
  float s = (rest2 - len) * kLSTh * __frcp_rn(sum);                 // correctly rounded reciprocal: no IEEE-division slow path in the hot loop
#else
  float s = (rest2 - len) * kLSTh * (1.0f / sum);
#endif
  s = sum > AG_CLOTH_EPS ? s : 0.f;                                 // Bullet skips degenerate links; a select keeps the loop branch-free
  a -= del * s; b += del * s;
}

// ------------------------------------------------------------------ small per-lane kernels
// snapshot of the collider links' poses at the start of substep p.i0 (thread = (collider link, env))
AG_HDN inline void cloth_snap_body(int tid, const SimDev& S, const KP& p) {
  const ClothDev& C = *(const ClothDev*)p.p0;
  const int N = S.N, e = tid % N, L = tid / N;
  int link = AG_LDG(C.cl_link + L);
  float* s = C.snap + ((size_t)(p.i0 * C.ncl + L) * 7) * N + e;
  f3 lp = ld3(S.lpos, link, N, e); q4 lq = ld4(S.lquat, link, N, e);
  s[0] = lp.x; s[(size_t)N] = lp.y; s[2 * (size_t)N] = lp.z;
  s[3 * (size_t)N] = lq.x; s[4 * (size_t)N] = lq.y; s[5 * (size_t)N] = lq.z; s[6 * (size_t)N] = lq.w;
}
// the anchor body follows a link (reference dressing.py:210 update_targets; thread = env)
AG_HDN inline void cloth_follow_body(int tid, const SimDev& S, const KP& p) {
  const ClothDev& C = *(const ClothDev*)p.p0;
  st3(C.anchor_pos, 0, S.N, tid, ld3(S.lpos, p.i0, S.N, tid));
}

// ------------------------------------------------------------------ K8: the cloth kernel
#if defined(__CUDACC__) && !defined(AG_CPU_EMU)
// QS: previous positions q (during a substep) / velocities v (between substeps) of a thread's own nodes live in a second
// shared-memory array instead of registers (same arithmetic, bit-identical results; frees 6 NPT registers under the
// 64-register limit of a 1024-thread CTA)
// Can any node of a patch (bounding box lo..hi, bounding sphere wc / wr) be within the collision margin of collider link `o` (its entry
// of the link table in shared memory)?  Conservative, so the outcome of the search does not depend on it.  Limbs are long thin capsules:
// their bounding sphere is several times wider than they are, the distance to the core segment is what keeps the pair list short.
__device__ __forceinline__ bool cloth_patch_near(const float* o, f3 lo, f3 hi, f3 wc, float wr, float margin) {
  if (o[23] == 1.f) {                                                  // one sphere / capsule, core a..b in world space
    f3 a(o[16], o[17], o[18]), ab = f3(o[19], o[20], o[21]) - a;
    float tt = clampf(dot(wc - a, ab) / fmaxf(dot(ab, ab), 1e-20f), 0.f, 1.f);
    f3 w = wc - (a + ab * tt);
    float lim = o[22] + margin + wr + 1e-5f;
    return dot(w, w) <= lim * lim;
  }
  if (o[23] == 2.f) return o[16] * wc.x + o[17] * wc.y + o[18] * wc.z - o[19] - wr <= margin + o[22] + 1e-5f;      // a half-space (the floor)
  f3 bc(o[12], o[13], o[14]);
  f3 cp = fmax3(lo, fmin3(hi, bc)) - bc;                               // the box's point nearest to the link's bounding sphere
  return dot(cp, cp) <= o[15] * o[15];
}
__device__ __forceinline__ float4 cloth_lds4(unsigned a) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void cloth_sts4(unsigned a, float x, float y, float z) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" :: "r"(a), "f"(x), "f"(y), "f"(z), "f"(0.f) : "memory");
}
template <int NPT, bool QS>
__global__ void __launch_bounds__(AG_CLOTH_T, 1) k_cloth(SimDev S, ClothDev C) {
  extern __shared__ __align__(16) float cl_smem[];
  constexpr int T = AG_CLOTH_T;
  const int N = S.N, e = blockIdx.x, t = threadIdx.x;
  float4* xs = (float4*)cl_smem;                               // [NPT * T]
  unsigned xs_sa = (unsigned)__cvta_generic_to_shared(xs);     // its shared-memory address, pinned in a register for the colour passes
  asm volatile("" : "+r"(xs_sa));
  float* lk = cl_smem + 4 * NPT * T;                           // [ncl][AG_CLOTH_LKS]
  float* pool = lk + AG_CLOTH_LKS * AG_CLOTH_MAXCL;                      // [maxcc][12] n, offset | c3, c4, node, link | acc, -
  int* misc = (int*)(pool + 12 * C.maxcc);                     // [40] warp sums for the scan [0..31], total [32], active-link masks [34..36]
  float* wbox = (float*)(misc + 40);                           // [32][6] per-warp bounding boxes of the predicted nodes
  float4* qs = (float4*)(wbox + 192);                          // [NPT * T] (QS only)
  const int nn = C.nn;
  const size_t xb = (size_t)e * 3 * C.nnp;
  f3 q[QS ? 1 : NPT], v[QS ? 1 : NPT];
  auto getq = [&](int k, int i) -> f3 {
    if constexpr (QS) { float4 t4 = qs[i]; (void)k; return f3(t4.x, t4.y, t4.z); }
    else { f3 r(0.f, 0.f, 0.f); (void)i;
#pragma unroll
      for (int kk = 0; kk < NPT; kk++) if (kk == k) r = q[kk];
      return r; }
  };
  // ---- load
#pragma unroll
  for (int k = 0; k < NPT; k++) {
    int i = k * T + t;
    f3 xx(0.f, 0.f, 0.f), vv(0.f, 0.f, 0.f);
    if (i < nn) {
      xx = f3(C.x[xb + i], C.x[xb + C.nnp + i], C.x[xb + 2 * (size_t)C.nnp + i]);
      vv = f3(C.v[xb + i], C.v[xb + C.nnp + i], C.v[xb + 2 * (size_t)C.nnp + i]);
    }
    xs[i] = make_float4(xx.x, xx.y, xx.z, 0.f);
    if constexpr (QS) qs[i] = make_float4(vv.x, vv.y, vv.z, 0.f); else { q[k] = xx; v[k] = vv; }
  }
  const f3 ap = ld3(C.anchor_pos, 0, N, e);
  int total = 0;
  __syncthreads();
  for (int sub = 0; sub < C.K; sub++) {
    // ---- predict own nodes (reads the neighbours' start-of-substep positions for the node normal)
    f3 xn[NPT];
#pragma unroll
    for (int k = 0; k < NPT; k++) {
      int i = k * T + t;
      xn[k] = f3(0.f, 0.f, 0.f);
      if (i < nn) {
        float4 me = xs[i]; f3 a(me.x, me.y, me.z);
        f3 ns(0.f, 0.f, 0.f);
        int f0 = __ldg(C.nf_off + i), f1 = __ldg(C.nf_off + i + 1);
        for (int f = f0; f < f1; f++) {
          unsigned pr = __ldg(C.nf_pair + f);
          float4 b4 = xs[pr & 0xffffu], c4 = xs[pr >> 16];
          ns += cross(f3(b4.x, b4.y, b4.z) - a, f3(c4.x, c4.y, c4.z) - a);
        }
        float nl = norm(ns);
        if (nl > AG_CLOTH_EPS) ns = ns * (1.f / nl);
        f3 xx = a, vv;
        if constexpr (QS) { float4 v4 = qs[i]; vv = f3(v4.x, v4.y, v4.z); } else vv = v[k];
        cloth_predict(C, ns, __ldg(C.node_area + i), xx, vv);
        if constexpr (QS) qs[i] = make_float4(a.x, a.y, a.z, 0.f); else { q[k] = a; v[k] = vv; }
        xn[k] = xx;
      }
    }
    // bounding box of the predicted cloth, per warp -> shared memory
    {
      f3 lo(1e30f, 1e30f, 1e30f), hi(-1e30f, -1e30f, -1e30f);
#pragma unroll
      for (int k = 0; k < NPT; k++) if (k * T + t < nn) { lo = fmin3(lo, xn[k]); hi = fmax3(hi, xn[k]); }
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, d)); lo.y = fminf(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, d)); lo.z = fminf(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, d));
        hi.x = fmaxf(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, d)); hi.y = fmaxf(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, d)); hi.z = fmaxf(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, d));
      }
      if ((t & 31) == 0) { float* w = wbox + 6 * (t >> 5); w[0] = lo.x; w[1] = lo.y; w[2] = lo.z; w[3] = hi.x; w[4] = hi.y; w[5] = hi.z; }
    }
    __syncthreads();                                           // every normal is computed, the warp boxes are written
    // ---- collider link poses of this substep; a link whose bounding sphere misses the cloth's box is skipped by everyone
    if (t < AG_CLOTH_MAXCL) {                                  // warps 0..2, whole warps
      bool on = false;
      if (t < C.ncl) {
        ClothLinkPose P = cloth_link_pose(C, sub, t, N, e);
        float* o = lk + AG_CLOTH_LKS * t;
#pragma unroll
        for (int a = 0; a < 9; a++) o[a] = P.R.m[a];
        {                                                        // a link that is one sphere / capsule: its core in world space
          int link = __ldg(C.cl_link + t), c0 = __ldg(S.link_col0 + link);
          int ty = __ldg(S.link_ncol + link) == 1 ? __ldg(S.col_type + c0) : 2;
          o[23] = ty <= 1 ? 1.f : 0.f;
          if (__ldg(S.link_ncol + link) == 1 && __ldg(S.col_type + c0) == 3) {     // the ground: its plane in world space, for the patch-level test
            f3 pn; float pd; ld_plane(S.planes, __ldg(S.col_p0 + c0), pn, pd);
            f3 nw = mul(P.R, pn);
            o[16] = nw.x; o[17] = nw.y; o[18] = nw.z; o[19] = pd + dot(nw, P.pos); o[22] = __ldg(S.col_radius + c0); o[23] = 2.f;
          }
          if (ty <= 1) {
            int v0 = __ldg(S.col_v0 + c0);
            f3 aw = P.pos + mul(P.R, tv3(S.verts, v0)), bw = ty == 1 ? P.pos + mul(P.R, tv3(S.verts, v0 + 1)) : aw;
            o[16] = aw.x; o[17] = aw.y; o[18] = aw.z; o[19] = bw.x; o[20] = bw.y; o[21] = bw.z; o[22] = __ldg(S.col_radius + c0);
          }
        }
        f3 lo(1e30f, 1e30f, 1e30f), hi(-1e30f, -1e30f, -1e30f);
        for (int w = 0; w < T / 32; w++) { lo = fmin3(lo, f3(wbox[6 * w], wbox[6 * w + 1], wbox[6 * w + 2])); hi = fmax3(hi, f3(wbox[6 * w + 3], wbox[6 * w + 4], wbox[6 * w + 5])); }
        f3 cp = fmax3(lo, fmin3(hi, P.bc)) - P.bc;             // box point nearest to the sphere centre
        on = cloth_link_active(S, C, t, N, e) && dot(cp, cp) <= P.br * P.br;
        o[9] = P.pos.x; o[10] = P.pos.y; o[11] = P.pos.z; o[12] = P.bc.x; o[13] = P.bc.y; o[14] = P.bc.z; o[15] = on ? P.br : 0.f;
      }
      unsigned bits = __ballot_sync(0xffffffffu, on);          // the surviving links as bit masks: the node loop visits only those
      if ((t & 31) == 0) misc[34 + (t >> 5)] = (int)bits;
    }
    // ---- publish the prediction
#pragma unroll
    for (int k = 0; k < NPT; k++) { int i = k * T + t; if (i < nn) xs[i] = make_float4(xn[k].x, xn[k].y, xn[k].z, 0.f); }
    __syncthreads();
    // ---- find contacts of own nodes.  The 32 nodes a warp handles in one pass are neighbours on the mesh (breadth-first node
    // order), so links -- and, for links made of many hulls (the wheelchair: 44), colliders -- are first culled against the bounding
    // sphere of the warp's nodes, the lanes testing one collider each; every branch around the ballots is warp-uniform
    int hits[AG_CLOTH_HITS]; int nh = 0; bool over = false;
    const bool any_link = (misc[34] | misc[35] | misc[36]) != 0;      // block-uniform
#pragma unroll
    for (int k = 0; k < NPT; k++) {
      if (!any_link) break;
      const int i = k * T + t;
      bool valid = i < nn;
      if (valid) for (int a = 0; a < C.nanch; a++) valid &= C.anch_node[a] != i;
      f3 lo = valid ? xn[k] : f3(1e30f, 1e30f, 1e30f), hi = valid ? xn[k] : f3(-1e30f, -1e30f, -1e30f);
#pragma unroll
      for (int d = 16; d >= 1; d >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, d)); lo.y = fminf(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, d)); lo.z = fminf(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, d));
        hi.x = fmaxf(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, d)); hi.y = fmaxf(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, d)); hi.z = fmaxf(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, d));
      }
      if (!(hi.x >= lo.x)) continue;                                  // no node of this warp in this pass
      const f3 wc = (lo + hi) * 0.5f; const float wr = 0.5f * norm(hi - lo) + 1e-6f;
      for (int w = 0; w < AG_CLOTH_MAXCL / 32; w++) {
        // the lanes test 32 links at once against the warp's sphere; only the survivors are visited
        unsigned m = (unsigned)misc[34 + w];
        {
          bool near = false;
          if ((m >> (t & 31)) & 1u) {
            near = cloth_patch_near(lk + AG_CLOTH_LKS * ((w << 5) + (t & 31)), lo, hi, wc, wr, C.margin);
          }
          m = __ballot_sync(0xffffffffu, near);
        }
        while (m) {                                                   // ascending link index, as the sequential sweep visits them
          const int L = (w << 5) + __ffs(m) - 1;
          m &= m - 1;
          const float* o = lk + AG_CLOTH_LKS * L;
          if (o[23] == 2.f) {                                          // a half-space the whole patch is clear of (the floor, usually)
            if (o[16] * wc.x + o[17] * wc.y + o[18] * wc.z - o[19] - wr > C.margin + o[22]) continue;
          } else if (o[23] != 0.f) {                                   // one sphere / capsule: world-space fast path
            if (valid) {
              ClothContact c;
              if (cloth_detect_round(S, C, f3(o[16], o[17], o[18]), f3(o[19], o[20], o[21]), o[22], L, N, e, xn[k], getq(k, i), c)) { if (nh < AG_CLOTH_HITS) hits[nh++] = (k << 8) | L; else over = true; }
            }
            continue;
          }
          ClothLinkPose P;
          for (int a = 0; a < 9; a++) P.R.m[a] = o[a];
          P.pos = f3(o[9], o[10], o[11]); P.bc = f3(o[12], o[13], o[14]); P.br = o[15];
          unsigned long long cmask = ~0ull;
          const int link = __ldg(C.cl_link + L), nc = __ldg(S.link_ncol + link);
          if (nc > 2) {
            const f3 pl = mulT(P.R, wc - P.pos);
            const int c0 = __ldg(S.link_col0 + link);
            cmask = 0ull;
            for (int r = 0; r < 2; r++) {
              int c = c0 + r * 32 + (t & 31);
              bool ok = false;
              if (c < c0 + nc) {
                if (__ldg(S.col_type + c) == 3) ok = true;
                else {
                  f3 bc = tv3(S.col_center, c), bh = tv3(S.col_half, c);
                  f3 qd = fmax3(f3(fabsf(pl.x - bc.x) - bh.x, fabsf(pl.y - bc.y) - bh.y, fabsf(pl.z - bc.z) - bh.z), f3(0.f, 0.f, 0.f));
                  float lim = wr + C.margin + __ldg(S.col_radius + c);
                  ok = dot(qd, qd) <= lim * lim;
                }
              }
              cmask |= (unsigned long long)__ballot_sync(0xffffffffu, ok) << (32 * r);
            }
            if (cmask == 0ull && nc <= 64) continue;
          }
          if (valid) {
            f3 wv = xn[k] - P.bc;
            if (dot(wv, wv) <= P.br * P.br) {
              ClothContact c;
              int cb = 0;
              if (cloth_detect(S, C, P, L, N, e, xn[k], getq(k, i), c, cmask, &cb)) { if (nh < AG_CLOTH_HITS) hits[nh++] = (cb << 16) | (k << 8) | L; else over = true; }
            }
          }
        }
      }
    }
    // block-wide exclusive prefix sum of nh -> deterministic contact slots
    int incl = nh;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { int o = __shfl_up_sync(0xffffffffu, incl, d); if ((t & 31) >= d) incl += o; }
    if ((t & 31) == 31) misc[t >> 5] = incl;
    __syncthreads();
    if (t < 32) {
      int w = misc[t], wi = w;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { int o = __shfl_up_sync(0xffffffffu, wi, d); if (t >= d) wi += o; }
      misc[t] = wi - w;
      if (t == 31) misc[32] = wi;
    }
    __syncthreads();
    const int base = misc[t >> 5] + incl - nh;
    total = misc[32];
    if (total > C.maxcc) { over = true; total = C.maxcc; }
    // The records are written once the slots are known, from the (node, link, collider) triples of the hits; the distance evaluation
    // visits only the collider that made the contact.  In the QS variant the owner only posts the triple and the block then writes one
    // record per thread: the hits sit on the few threads whose nodes touch the body, which the others used to wait for.
    auto write_record = [&](int slot, int i, int L, int cb, f3 xk, f3 qk) {
      const float* o = lk + AG_CLOTH_LKS * L;
      ClothContact c;
      if (o[23] == 1.f) cloth_detect_round(S, C, f3(o[16], o[17], o[18]), f3(o[19], o[20], o[21]), o[22], L, N, e, xk, qk, c);
      else {
        ClothLinkPose P;
        for (int a = 0; a < 9; a++) P.R.m[a] = o[a];
        P.pos = f3(o[9], o[10], o[11]); P.bc = f3(o[12], o[13], o[14]); P.br = o[15];
        cloth_detect(S, C, P, L, N, e, xk, qk, c, cb < 64 ? 1ull << cb : 0ull);
      }
      float4* r4 = (float4*)(pool + 12 * slot);
      r4[0] = make_float4(c.n.x, c.n.y, c.n.z, c.offset);
      r4[1] = make_float4(c.c3, c.c4, __int_as_float(i), __int_as_float(c.link));
      r4[2] = make_float4(0.f, 0.f, 0.f, 0.f);
    };
    if constexpr (QS) {
      for (int h = 0; h < nh; h++) {
        int slot = base + h;
        if (slot >= C.maxcc) break;
        pool[12 * slot + 6] = __int_as_float(((hits[h] >> 8) & 0xff) * T + t);
        pool[12 * slot + 7] = __int_as_float((hits[h] & 0xff) | (hits[h] >> 16 << 8));
      }
      __syncthreads();
      for (int slot = t; slot < total; slot += T) {
        int i = __float_as_int(pool[12 * slot + 6]), lc = __float_as_int(pool[12 * slot + 7]);
        float4 x4 = xs[i], q4 = qs[i];
        write_record(slot, i, lc & 0xff, lc >> 8, f3(x4.x, x4.y, x4.z), f3(q4.x, q4.y, q4.z));
      }
    } else {
      for (int h = 0; h < nh; h++) {
        int slot = base + h;
        if (slot >= C.maxcc) break;
        int k = (hits[h] >> 8) & 0xff;
        f3 xk(0.f, 0.f, 0.f), qk = getq(k, k * T + t);
#pragma unroll
        for (int kk = 0; kk < NPT; kk++) if (kk == k) xk = xn[kk];
        write_record(slot, k * T + t, hits[h] & 0xff, hits[h] >> 16, xk, qk);
      }
    }
    if (over) C.overflow[e] = 1;
    __syncthreads();
    // ---- position solver
    for (int it = 0; it < C.piters; it++) {
      // anchors and rigid contacts touch only the owner's nodes
      for (int a = 0; a < C.nanch; a++) {
        int i = C.anch_node[a];
        if ((i & (T - 1)) == t) {
          float4 me = xs[i]; f3 xx(me.x, me.y, me.z), qq = getq(i / T, i);
          cloth_anchor_solve(xx, qq, ap + f3(C.anch_local[a][0], C.anch_local[a][1], C.anch_local[a][2]), C.kAHR);
          xs[i] = make_float4(xx.x, xx.y, xx.z, 0.f);
        }
      }
      if constexpr (QS) {
        // One thread per contact slot, not per owner: the contacts sit on the few hundred nodes that touch the body, whose owner threads
        // used to relax up to 4 nodes x several contacts each while the rest of the block waited at the barrier below.  A node's contacts
        // are consecutive slots (the hits are listed node by node); the thread of the first one relaxes the run in slot order, so the
        // result is the sequential sweep's.  Both node arrays are in shared memory in this variant, any thread can take any node.
        for (int s0 = t; s0 < total; s0 += T) {
          float4* r4 = (float4*)(pool + 12 * s0);
          const int i = __float_as_int(r4[1].z);
          if (s0 > 0 && __float_as_int(pool[12 * (s0 - 1) + 6]) == i) continue;
          float4 me = xs[i], q4 = qs[i];
          f3 xx(me.x, me.y, me.z), qq(q4.x, q4.y, q4.z);
          for (int s1 = s0;;) {
            float4 a = r4[0], b = r4[1], c = r4[2];
            f3 acc(c.x, c.y, c.z);
            cloth_contact_solve(xx, qq, f3(a.x, a.y, a.z), a.w, b.x, b.y, C.margin, acc);
            r4[2] = make_float4(acc.x, acc.y, acc.z, 0.f);
            if (++s1 >= total) break;
            r4 += 3;
            if (__float_as_int(r4[1].z) != i) break;
          }
          xs[i] = make_float4(xx.x, xx.y, xx.z, 0.f);
        }
      } else {
        for (int h = 0; h < nh; h++) {
          int slot = base + h;
          if (slot >= C.maxcc) break;
          int k = (hits[h] >> 8) & 0xff, i = k * T + t;
          float* r = pool + 12 * slot;
          float4 me = xs[i]; f3 xx(me.x, me.y, me.z), qq = getq(k, i), acc(r[8], r[9], r[10]);
          cloth_contact_solve(xx, qq, f3(r[0], r[1], r[2]), r[3], r[4], r[5], C.margin, acc);
          xs[i] = make_float4(xx.x, xx.y, xx.z, 0.f);
          r[8] = acc.x; r[9] = acc.y; r[10] = acc.z;
        }
      }
      __syncthreads();
      if (C.link_dense) {
        // One row of the table per colour, one entry per thread: a pass is two 16-byte loads, the relaxation, two 16-byte stores and
        // the barrier.  The pass is issue-bound (32 warps x ~40 instructions against 4 schedulers), so everything else is kept out
        // of it: the next colour's entry is fetched one pass ahead by bumping a pointer, and the node arrays are addressed through a
        // 32-bit shared-memory address held in a register (left to itself the compiler re-derives the base -- S2R SR_CgaCtaId,
        // a long-scoreboard wait -- in every pass: 7 % of the kernel's samples sat on it).
        const uint2* row = (const uint2*)C.link_dense + t;
        uint2 nxt = __ldg(row);
        for (int col = 0; col < C.ncol; col++) {
          const uint2 lt = nxt;
          row = col + 1 < C.ncol ? row + T : (const uint2*)C.link_dense + t;      // (the last pass fetches colour 0 of the next iteration)
          nxt = __ldg(row);
          if (lt.x != 0xffffffffu) {
            const unsigned ai = xs_sa + ((lt.x & 0xffffu) << 4), bi = xs_sa + ((lt.x >> 16) << 4);
            float4 a4 = cloth_lds4(ai), b4 = cloth_lds4(bi);
            f3 a(a4.x, a4.y, a4.z), b(b4.x, b4.y, b4.z);
            cloth_link_solve(a, b, __uint_as_float(lt.y), C.kLSTh);
            cloth_sts4(ai, a.x, a.y, a.z); cloth_sts4(bi, b.x, b.y, b.z);
          }
          __syncthreads();
        }
        continue;
      }
      // the first record of a colour is fetched while the previous colour is relaxed (the table lives in L2: the contact pool and
      // the node arrays leave the L1 too small for it)
      uint2 nxt = make_uint2(0u, 0u);
      if (C.tab_off[0] + t < C.tab_end[0]) nxt = __ldg((const uint2*)(C.link_tab + C.tab_off[0] + t));
      for (int col = 0; col < C.ncol; col++) {
        uint2 lt = nxt;
        int l = C.tab_off[col] + t;
        if (col + 1 < C.ncol && C.tab_off[col + 1] + t < C.tab_end[col + 1]) nxt = __ldg((const uint2*)(C.link_tab + C.tab_off[col + 1] + t));
        for (; l < C.tab_end[col]; l += T) {
          unsigned ij = lt.x;
          float r2 = __uint_as_float(lt.y);
          int i = ij & 0xffffu, j = ij >> 16;
          float4 a4 = xs[i], b4 = xs[j];
          f3 a(a4.x, a4.y, a4.z), b(b4.x, b4.y, b4.z);
          cloth_link_solve(a, b, r2, C.kLSTh);
          xs[i] = make_float4(a.x, a.y, a.z, 0.f); xs[j] = make_float4(b.x, b.y, b.z, 0.f);
          if (l + T < C.tab_end[col]) lt = __ldg((const uint2*)(C.link_tab + l + T));      // colours larger than the block (other meshes)
        }
        __syncthreads();
      }
    }
    // ---- velocities
    const float vc = (1.f - C.kDP) / C.dt;
#pragma unroll
    for (int k = 0; k < NPT; k++) {
      int i = k * T + t;
      if (i < nn) {
        float4 me = xs[i]; f3 vv = (f3(me.x, me.y, me.z) - getq(k, i)) * vc;
        if constexpr (QS) qs[i] = make_float4(vv.x, vv.y, vv.z, 0.f); else v[k] = vv;
      }
    }
    // (the next substep's prediction reads xs, final since the last colour's barrier; the contact pool is rewritten only
    //  after that substep's first barrier, the link poses before it -- both were last read before the barrier above)
  }
  // ---- store
#pragma unroll
  for (int k = 0; k < NPT; k++) {
    int i = k * T + t;
    if (i < nn) {
      float4 me = xs[i];
      C.x[xb + i] = me.x; C.x[xb + C.nnp + i] = me.y; C.x[xb + 2 * (size_t)C.nnp + i] = me.z;
      f3 vv;
      if constexpr (QS) { float4 v4 = qs[i]; vv = f3(v4.x, v4.y, v4.z); } else vv = v[k];
      C.v[xb + i] = vv.x; C.v[xb + C.nnp + i] = vv.y; C.v[xb + 2 * (size_t)C.nnp + i] = vv.z;
    }
  }
  // contacts of the last substep: node, position, force = accumulated correction / (im dt^2)
  if (t == 0) C.cc_count[e] = total;
  if (C.export_contacts) {
    const float fs = 1.f / (C.im * C.dt * C.dt);
    for (int s = t; s < total; s += T) {
      const float* r = pool + 12 * s;
      int i = __float_as_int(r[6]);
      float4 me = xs[i];
      float* o = C.cc_data + ((size_t)e * C.maxcc + s) * AG_CLOTH_CCF;
      o[0] = r[6]; o[1] = me.x; o[2] = me.y; o[3] = me.z; o[4] = -r[8] * fs; o[5] = -r[9] * fs; o[6] = -r[10] * fs; o[7] = r[7];
    }
  }
}
#endif

// ------------------------------------------------------------------ host restatement of the device loop (CPU harness)
// Same per-node / per-link functions, plain loops: nodes in thread-major order (so contact slots come out in the order the
// block-wide prefix sum gives them), links in list order.
#if !defined(__CUDA_ARCH__)
#include <vector>
static inline void cloth_env_host(const SimDev& S, const ClothDev& C, int e) {
  const int N = S.N, T = AG_CLOTH_T, nn = C.nn, NPT = (nn + T - 1) / T;
  const size_t xb = (size_t)e * 3 * C.nnp;
  std::vector<f3> x(nn), q(nn), v(nn), xn(nn);
  for (int i = 0; i < nn; i++) {
    x[i] = f3(C.x[xb + i], C.x[xb + C.nnp + i], C.x[xb + 2 * (size_t)C.nnp + i]);
    v[i] = f3(C.v[xb + i], C.v[xb + C.nnp + i], C.v[xb + 2 * (size_t)C.nnp + i]);
  }
  const f3 ap = ld3(C.anchor_pos, 0, N, e);
  std::vector<ClothContact> cc;
  for (int sub = 0; sub < C.K; sub++) {
    std::vector<ClothLinkPose> P(C.ncl);
    for (int L = 0; L < C.ncl; L++) { P[L] = cloth_link_pose(C, sub, L, N, e); if (!cloth_link_active(S, C, L, N, e)) P[L].br = 0.f; }
    for (int i = 0; i < nn; i++) {
      q[i] = x[i];
      f3 ns(0.f, 0.f, 0.f);
      for (int f = C.nf_off[i]; f < C.nf_off[i + 1]; f++) {
        unsigned pr = C.nf_pair[f];
        ns += cross(x[pr & 0xffffu] - x[i], x[pr >> 16] - x[i]);
      }
      float nl = norm(ns);
      if (nl > AG_CLOTH_EPS) ns = ns * (1.f / nl);
      xn[i] = x[i];
      cloth_predict(C, ns, C.node_area[i], xn[i], v[i]);
    }
    x = xn;
    cc.clear();
    bool over = false;
    for (int t = 0; t < T; t++) {
      int nh = 0;
      for (int k = 0; k < NPT; k++) {
        int i = k * T + t;
        if (i >= nn) continue;
        bool anchored = false;
        for (int a = 0; a < C.nanch; a++) anchored |= C.anch_node[a] == i;
        if (anchored) continue;
        for (int L = 0; L < C.ncl; L++) {
          ClothContact c;
          if (cloth_detect(S, C, P[L], L, N, e, x[i], q[i], c)) {
            if (nh < AG_CLOTH_HITS) { nh++; c.node = i; cc.push_back(c); } else over = true;
          }
        }
      }
    }
    if ((int)cc.size() > C.maxcc) { over = true; cc.resize(C.maxcc); }
    if (over) C.overflow[e] = 1;
    for (int it = 0; it < C.piters; it++) {
      for (int a = 0; a < C.nanch; a++) {
        int i = C.anch_node[a];
        cloth_anchor_solve(x[i], q[i], ap + f3(C.anch_local[a][0], C.anch_local[a][1], C.anch_local[a][2]), C.kAHR);
      }
      for (auto& c : cc) cloth_contact_solve(x[c.node], q[c.node], c.n, c.offset, c.c3, c.c4, C.margin, c.acc);
      for (int l = 0; l < C.nlinks; l++) {
        unsigned ij = C.link_ij[l];
        cloth_link_solve(x[ij & 0xffffu], x[ij >> 16], C.link_rest2[l], C.kLSTh);
      }
    }
    const float vc = (1.f - C.kDP) / C.dt;
    for (int i = 0; i < nn; i++) v[i] = (x[i] - q[i]) * vc;
  }
  for (int i = 0; i < nn; i++) {
    C.x[xb + i] = x[i].x; C.x[xb + C.nnp + i] = x[i].y; C.x[xb + 2 * (size_t)C.nnp + i] = x[i].z;
    C.v[xb + i] = v[i].x; C.v[xb + C.nnp + i] = v[i].y; C.v[xb + 2 * (size_t)C.nnp + i] = v[i].z;
  }
  C.cc_count[e] = (int)cc.size();
  if (C.export_contacts) {
    const float fs = 1.f / (C.im * C.dt * C.dt);
    for (size_t s = 0; s < cc.size(); s++) {
      float* o = C.cc_data + ((size_t)e * C.maxcc + s) * AG_CLOTH_CCF;
      int i = cc[s].node;
      union { int i; float f; } u; u.i = i; o[0] = u.f;
      o[1] = x[i].x; o[2] = x[i].y; o[3] = x[i].z; o[4] = -cc[s].acc.x * fs; o[5] = -cc[s].acc.y * fs; o[6] = -cc[s].acc.z * fs;
      u.i = cc[s].link; o[7] = u.f;
    }
  }
}
#endif
