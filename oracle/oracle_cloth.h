// oracle_cloth.h — CPU restatement of the cloth step of the Dressing task.  TEST INFRASTRUCTURE (see README.md): only
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may use it.
//
// Follows, call by call, what `p.stepSimulation` does to the `btSoftBody` the reference creates with
// p.loadCloth / p.clothParams (envs/dressing.py:146-154) -- Bullet's soft-body code is not in the reference repository
// (third-party: bullet3, Zackory fork, pinned by setup.py:21 only as "pybullet"), so this restates its published
// algorithm as recalled (btSoftBody.cpp: predictMotion, addAeroForceToNode, ApplyClampedForce, solveConstraints,
// PSolve_Anchors, PSolve_RContacts, PSolve_Links; btSoftBodyInternals.h: CollideSDF_RS::DoNode, checkContact).
// PARITY UNPINNED against Bullet itself; pinned are the node numbering and placement convention (tests/test_cloth_model.py,
// against constants embedded in dressing.py) and analytic known answers (tests/test_cloth_oracle.py).
//
// Deliberately not a transcription of the CUDA side: double precision, AoS, plain sequential sweeps in list order,
// distances evaluated in the WORLD frame against the world-space collider data the rigid oracle maintains (the CUDA
// kernel transforms the node into the link frame), contacts kept in one list in node order.
#pragma once
#include <vector>
#include <algorithm>
#include <cmath>

struct OCloth {
  int nn = 0, piters = 0, maxcc = 1024;
  std::vector<int> links;            // [nl][2]
  std::vector<real> rest2;
  std::vector<int> nf_off, nf_pair;  // pair: [nf][2]
  std::vector<real> area;
  real im = 0, kLST = 0, kDP = 0, kDG = 0, kLF = 0, kDF = 0, kCHR = 0, kKHR = 0, kAHR = 0, margin = 0, density = 0;
  V3 gravity;
  std::vector<int> anchor_node; std::vector<V3> anchor_local;
  std::vector<int> col_links, col_static;
  std::vector<V3> bs_c; std::vector<real> bs_r;
};
struct OClothContact { int node, link; V3 n; real offset, c3, c4; V3 acc; };
struct OClothEnv {
  std::vector<V3> x, v, q;
  V3 anchor_pos;
  std::vector<OClothContact> contacts;   // of the last substep
  int overflow = 0;
};

const real OCLOTH_EPS = (real)1.1920929e-7;   // SIMD_EPSILON of a single-precision Bullet build; the product uses the same value

// signed distance from a world point to collider c (world-space data of the env), outward normal
inline real ocloth_sdf_collider(const Scene& s, const Env& e, int c, V3 p, V3& n) {
  real r = s.col_radius[c];
  int v0 = s.col_v0[c];
  if (s.col_type[c] == AG_COL_SPHERE || s.col_type[c] == AG_COL_CAPSULE) {
    V3 a = e.wverts[v0], cp = a;
    if (s.col_type[c] == AG_COL_CAPSULE) {
      V3 ab = e.wverts[v0 + 1] - a;
      real t = dot(p - a, ab) / std::max(dot(ab, ab), (real)1e-20);
      t = std::min((real)1, std::max((real)0, t));
      cp = a + ab * t;
    }
    V3 w = p - cp; real L = norm(w);
    n = L > (real)1e-12 ? w * (1 / L) : V3(0, 0, 1);
    return L - r;
  }
  // hulls / the ground plane: the plane the point is farthest outside of (exact inside, a lower bound of the distance outside);
  // for hulls the six planes of the core's bounding box (link frame) take part as well
  real m = -1e30; n = V3(0, 0, 1);
  for (int k = s.col_p0[c]; k < s.col_p0[c] + s.col_np[c]; k++) {
    V3 pn(e.wplanes[4 * k], e.wplanes[4 * k + 1], e.wplanes[4 * k + 2]);
    real d = dot(pn, p) - e.wplanes[4 * k + 3];
    if (d > m) { m = d; n = pn; }
  }
  if (s.col_type[c] == AG_COL_HULL) {
    int link = s.col_link[c];
    Quat lq = e.lquat[link];
    V3 pl = qrot(qconj(lq), p - e.lpos[link]);
    for (int a = 0; a < 3; a++) {
      real side = pl[a] >= s.col_center[c][a] ? 1 : -1;
      real d = std::fabs(pl[a] - s.col_center[c][a]) - s.col_half[c][a];
      if (d > m) { m = d; V3 ax; ax[a] = side; n = qrot(lq, ax); }
    }
  }
  return m - r;
}

// one substep of dt for one env's cloth; e.lpos / e.lquat / e.wverts / e.wplanes hold the START-of-substep poses
inline void ocloth_substep(const Scene& s, const Env& e, const OCloth& C, OClothEnv& ce, real dt) {
  const int nn = C.nn;
  std::vector<V3>& x = ce.x; std::vector<V3>& v = ce.v; std::vector<V3>& q = ce.q;
  // --- predictMotion: gravity, aerodynamics with the normals of the current configuration, explicit Euler
  std::vector<V3> nrm(nn);
  for (int i = 0; i < nn; i++) {
    V3 ns;
    for (int f = C.nf_off[i]; f < C.nf_off[i + 1]; f++) ns = ns + cross(x[C.nf_pair[2 * f]] - x[i], x[C.nf_pair[2 * f + 1]] - x[i]);
    real L = norm(ns);
    nrm[i] = L > OCLOTH_EPS ? ns * (1 / L) : ns;
  }
  for (int i = 0; i < nn; i++) {
    q[i] = x[i];
    V3 vi = v[i] + C.gravity * dt, f;
    real v2 = dot(vi, vi);
    if ((C.kDG > 0 || C.kLF > 0) && v2 > OCLOTH_EPS) {
      V3 vn = vi * (1 / std::sqrt(v2)), n = nrm[i];
      real dvn = dot(vi, n);
      if (dvn < 0) { n = n * (real)-1; dvn = -dvn; }
      if (dvn > 0) {
        real c1 = C.area[i] * dvn * v2 * (real)0.5 * C.density;
        V3 force = n * (-c1 * C.kLF) + vn * (-c1 * C.kDG);
        real dtim = dt * C.im;
        V3 fd = force * dtim;
        if (dot(fd, fd) > v2) { V3 fn = force * (1 / norm(force)); f = f - fn * (dot(vi, fn) / dtim); }
        else f = f + force;
      }
    }
    vi = vi + f * (C.im * dt);
    v[i] = vi; x[i] = x[i] + vi * dt;
  }
  // --- rigid contacts (node order, collider links in list order)
  std::vector<char> anchored(nn, 0);
  for (int a : C.anchor_node) anchored[a] = 1;
  ce.contacts.clear();
  for (int i = 0; i < nn; i++) {
    if (anchored[i]) continue;
    for (size_t L = 0; L < C.col_links.size(); L++) {
      int link = C.col_links[L];
      if (e.body_mode[s.link_body[link]] == 0) continue;       // a body switched off in this env does not exist for the cloth
      V3 bc = e.lpos[link] + qrot(e.lquat[link], C.bs_c[L]);
      real br = C.bs_r[L] + C.margin;
      if (dot(x[i] - bc, x[i] - bc) > br * br) continue;
      real best = 1e30; V3 bn(0, 0, 1);
      for (int c = s.link_col0[link]; c < s.link_col0[link] + s.link_ncol[link]; c++) {
        V3 n; real d = ocloth_sdf_collider(s, e, c, x[i], n);
        if (d < best) { best = d; bn = n; }
      }
      real dst = best - C.margin;
      if (!(dst < 0)) continue;
      OClothContact c;
      c.node = i; c.link = link; c.n = bn;
      c.offset = -dot(bn, x[i] - bn * dst);
      V3 vr = x[i] - q[i];
      real dn = dot(vr, bn);
      V3 fv = vr - bn * dn;
      real fc = C.kDF * e.friction[link];
      c.c3 = dot(fv, fv) < (dn * fc) * (dn * fc) ? 0 : 1 - fc;
      c.c4 = C.col_static[L] ? C.kKHR : C.kCHR;
      ce.contacts.push_back(c);
    }
  }
  if ((int)ce.contacts.size() > C.maxcc) ce.overflow = 1;      // the product truncates (in its own slot order): flagged, not compared
  // --- position solver
  for (int it = 0; it < C.piters; it++) {
    for (size_t a = 0; a < C.anchor_node.size(); a++) {
      int i = C.anchor_node[a];
      V3 wa = ce.anchor_pos + C.anchor_local[a];
      x[i] = x[i] + (q[i] - x[i]) + (wa - x[i]) * C.kAHR;
    }
    for (auto& c : ce.contacts) {
      V3 vr = x[c.node] - q[c.node];
      real dn = dot(vr, c.n);
      if (dn <= OCLOTH_EPS) {
        real dp = std::min(dot(x[c.node], c.n) + c.offset, C.margin);
        V3 fv = vr - c.n * dn;
        V3 d = vr - fv * c.c3 + c.n * (dp * c.c4);
        x[c.node] = x[c.node] - d; c.acc = c.acc + d;
      }
    }
    for (size_t l = 0; l < C.rest2.size(); l++) {
      V3& a = x[C.links[2 * l]]; V3& b = x[C.links[2 * l + 1]];
      V3 del = b - a;
      real len = dot(del, del), c1 = C.rest2[l];
      if (c1 + len > OCLOTH_EPS) {
        real c0 = (C.im + C.im) / C.kLST;
        real k = (c1 - len) / (c0 * (c1 + len));
        a = a - del * (k * C.im); b = b + del * (k * C.im);
      }
    }
  }
  real vc = (1 - C.kDP) / dt;
  for (int i = 0; i < nn; i++) v[i] = (x[i] - q[i]) * vc;
}
