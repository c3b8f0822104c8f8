// ag_readback.cuh — read-back kernels (K6a-d of SURVEY.md §8(a)): what the per-call API asks the simulation for.
//
// Reference semantics restated here:
//   gather/linkstate    p.getJointStates / p.getLinkState / p.getBasePositionAndOrientation (agents/agent.py:40,49,52,72)
//   contact_query       p.getContactPoints (agents/agent.py:100-116)
//   closest             p.getClosestPoints (agents/agent.py:118-130)
#pragma once
#include <string.h>
#include "ag_task.cuh"

// ---- env-major host layout <-> SoA.  thread = (column j, env e), env fastest
AG_HDN inline void gather_body(int tid, const SimDev& S, const KP& p) {
  const int N = S.N;
  int e = tid % N, j = tid / N;
  int comp = p.i0, K = p.i0 * p.i1;
  int item = ((const int*)p.p2)[j / comp], c = j % comp;
  ((float*)p.p1)[(size_t)e * K + j] = ((const float*)p.p0)[((size_t)item * comp + c) * N + e];
}
AG_HDN inline void scatter_body(int tid, const SimDev& S, const KP& p) {
  const int N = S.N;
  int e = tid % N, j = tid / N;
  if (p.p3 && !((const int*)p.p3)[e]) return;
  int comp = p.i0, K = p.i0 * p.i1;
  int item = ((const int*)p.p2)[j / comp], c = j % comp;
  ((float*)p.p1)[((size_t)item * comp + c) * N + e] = ((const float*)p.p0)[(size_t)e * K + j];
}

AG_HDN inline void linkstate_body(int tid, const SimDev& S, const KP& p) {
  const int N = S.N;
  int e = tid % N, j = tid / N, n = p.i1;
  int k = ((const int*)p.p2)[j];
  float* o = (float*)p.p1 + ((size_t)e * n + j) * 20;
  f3 com; q4 cq; link_com_pose(S, e, k, com, cq);
  f3 lin, ang; link_velocity(S, e, k, com, lin, ang);
  int i = put3(o, 0, ld3(S.lpos, k, N, e)); i = put4(o, i, ld4(S.lquat, k, N, e));
  i = put3(o, i, com); i = put4(o, i, cq);
  i = put3(o, i, lin); put3(o, i, ang);
}

AG_HD float i2f(int v) { float f; memcpy(&f, &v, 4); return f; }

AG_HD void write_contact(float* o, int la, int lb, f3 pa, f3 pb, f3 n, float d, float f) {
  o[0] = i2f(la); o[1] = i2f(lb);
  o[2] = pa.x; o[3] = pa.y; o[4] = pa.z; o[5] = pb.x; o[6] = pb.y; o[7] = pb.z; o[8] = n.x; o[9] = n.y; o[10] = n.z;
  o[11] = d; o[12] = f;
}

// does link k belong to (body, link filter)?  lf = -2 any, else a global link id
AG_HD bool link_matches(const SimDev& S, int k, int body, int lf) {
  if (AG_LDG(S.link_body + k) != body) return false;
  return lf == -2 || lf == k;
}

// one lane per env.  i0 = bodyA, i1 = bodyB (-2 any), i2 / i3 = link filters, f0 = max_pts,
// p1 = out records [N][max_pts][13], p2 = counts, p3 = force sums
AG_HDN inline void contact_query_body(int e, const SimDev& S, const KP& p) {
  const int N = S.N;
  int max_pts = (int)p.f0;
  int cnt = n_contacts(S, e);
  int n = 0; float fsum = 0.f;
  for (int s = 0; s < cnt; s++) {
    Contact c = contact_at(S, e, s);
    bool fwd = link_matches(S, c.la, p.i0, p.i2) && (p.i1 < 0 || link_matches(S, c.lb, p.i1, p.i3));
    bool rev = link_matches(S, c.lb, p.i0, p.i2) && (p.i1 < 0 || link_matches(S, c.la, p.i1, p.i3));
    if (!fwd && !rev) continue;
    float force = contact_force(S, e, s);
    fsum += force;
    if (n < max_pts) {
      f3 pa = contact_point_a(S, e, s), pb = contact_point_b(S, e, s);
      f3 nn(cf_ld(S.s_data, s, CF_NX, N, e), cf_ld(S.s_data, s, CF_NY, N, e), cf_ld(S.s_data, s, CF_NZ, N, e));
      float* o = (float*)p.p1 + ((size_t)e * max_pts + n) * 13;
      if (fwd) write_contact(o, c.la, c.lb, pa, pb, nn, cf_ld(S.s_data, s, CF_DIST, N, e), force);
      else write_contact(o, c.lb, c.la, pb, pa, -nn, cf_ld(S.s_data, s, CF_DIST, N, e), force);
    }
    n++;
  }
  ((int*)p.p2)[e] = n;
  if (p.p3) ((float*)p.p3)[e] = fsum;
}

// one lane per env.  i0 = bodyA, i1 = bodyB, i2 = max_pts, f0 = distance
AG_HDN inline void closest_body(int e, const SimDev& S, const KP& p) {
  const int N = S.N;
  int ba = p.i0, bb = p.i1, max_pts = p.i2; float dist = p.f0;
  int a0 = AG_LDG(S.body_link0 + ba), an = AG_LDG(S.body_nlinks + ba), b0 = AG_LDG(S.body_link0 + bb), bn = AG_LDG(S.body_nlinks + bb);
  int n = 0;
  if (S.body_mode[(size_t)ba * N + e] == 0 || S.body_mode[(size_t)bb * N + e] == 0) { ((int*)p.p2)[e] = 0; return; }
  for (int la = a0; la < a0 + an; la++) {
    int nca = AG_LDG(S.link_ncol + la); if (!nca) continue;
    f3 lamin = ld3(S.lmin, la, N, e), lamax = ld3(S.lmax, la, N, e);
    for (int lb = b0; lb < b0 + bn; lb++) {
      int ncb = AG_LDG(S.link_ncol + lb); if (!ncb) continue;
      if (!aabb_ov(lamin, lamax, ld3(S.lmin, lb, N, e), ld3(S.lmax, lb, N, e), dist)) continue;
      int ca0 = AG_LDG(S.link_col0 + la), cb0 = AG_LDG(S.link_col0 + lb);
      for (int ca = ca0; ca < ca0 + nca; ca++) {
        f3 amin = ld3(S.cmin, ca, N, e), amax = ld3(S.cmax, ca, N, e);
        for (int cb = cb0; cb < cb0 + ncb; cb++) {
          if (!aabb_ov(amin, amax, ld3(S.cmin, cb, N, e), ld3(S.cmax, cb, N, e), dist)) continue;
          NpOut c;
          if (!narrow_closest(S, e, ca, cb, dist, c)) continue;
          if (n < max_pts) write_contact((float*)p.p1 + ((size_t)e * max_pts + n) * 13, la, lb, c.pa, c.pb, c.n, c.d, 0.f);
          n++;
        }
      }
    }
  }
  ((int*)p.p2)[e] = n;
}
