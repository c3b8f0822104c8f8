// ag_task.cuh — what the fused env-step kernels of every task share (ag_feeding / ag_scratch / ag_bathing / ag_dressing /
// ag_drinking / ag_coop) and the read-back kernels (ag_readback.cuh): frames and poses as PyBullet reports them, the pieces of
// an observation row, the decode of a sorted contact record, and the parts of AssistiveEnv.take_step (envs/env.py:174-222)
// that do not depend on the task.  Each helper is one fixed sequence of floating-point operations: a task's results are
// pinned bit for bit (tests/golden/fused_step_pin.npz), so a change here changes every task at once, and is meant to.
#pragma once
#include "ag_device.cuh"

AG_HD unsigned long long xorshift64s(unsigned long long& s) {
  s ^= s >> 12; s ^= s << 25; s ^= s >> 27;
  return s * 2685821657736338717ull;
}
AG_HD float rng_uniform(unsigned long long& s) { return (float)(xorshift64s(s) >> 40) * (1.0f / 16777216.0f); }

// ---- poses
// a link's COM pose (world), the `linkWorldPosition / Orientation` of p.getLinkState (agent.py:72)
AG_HD void link_com_pose(const SimDev& S, int e, int k, f3& pos, q4& quat) {
  const int N = S.N;
  q4 q = ld4(S.lquat, k, N, e);
  pos = ld3(S.lpos, k, N, e) + qrot(q, tv3(S.link_com, k));
  quat = qmul(q, tv4(S.link_iquat, k));
}
AG_HD f3 link_com(const SimDev& S, int e, int k) {
  const int N = S.N;
  return ld3(S.lpos, k, N, e) + qrot(ld4(S.lquat, k, N, e), tv3(S.link_com, k));
}

// a body's base frame = its inertial frame, as p.getBasePositionAndOrientation reports it (agent.py:49,58-63): the origin
// and the inverse rotation, so that observations are expressed in it
struct Frame { f3 p; q4 qi; };
AG_HD Frame body_frame(const SimDev& S, int e, int body) {
  Frame fr; q4 q;
  link_com_pose(S, e, AG_LDG(S.body_link0 + body), fr.p, q);
  fr.qi = qconj(q);
  return fr;
}
AG_HD f3 to_frame(const Frame& fr, f3 pos) { return qrot(fr.qi, pos - fr.p); }
AG_HD q4 to_frame(const Frame& fr, q4 quat) { return qmul(fr.qi, quat); }

// the head link's frame and the mouth target in it (feeding.py:101-104, drinking.py:24-26); `mouth` is the person's offset
AG_HD f3 mouth_target(const SimDev& S, int e, int head_link, const float mouth[3], f3& hp, q4& hq) {
  const int N = S.N;
  hp = ld3(S.lpos, head_link, N, e); hq = ld4(S.lquat, head_link, N, e);
  return hp + qrot(hq, f3(mouth[0], mouth[1], mouth[2]));
}

// spatial velocity of a link's COM (world): linear velocity of the COM, angular velocity
AG_HDN inline void link_velocity(const SimDev& S, int e, int k, f3 com, f3& lin, f3& ang) {
  const int N = S.N;
  int b = AG_LDG(S.link_body + k);
  int kind = AG_LDG(S.body_kind + b);
  lin = f3(); ang = f3();
  if (kind == BK_FREE) { lin = ld3(S.base_lin, b, N, e); ang = ld3(S.base_ang, b, N, e); return; }
  if (kind != BK_ART) return;
  int d = AG_LDG(S.link_dl + k);
  while (d >= 0) {
    int kj = AG_LDG(S.dl_link + d);
    f3 a = qrot(ld4(S.lquat, kj, N, e), tv3(S.link_axis, kj));
    float qd = ld1(S.jqd, kj, N, e);
    if (AG_LDG(S.dl_type + d) == 1) { ang += a * qd; lin += cross(a, com - ld3(S.lpos, kj, N, e)) * qd; }
    else lin += a * qd;
    d = AG_LDG(S.dl_parent + d);
  }
}
// speed of the end effector link's COM, the velocity term of the human preferences (env.py:244)
AG_HD float ee_speed(const SimDev& S, int e, int ee_link) {
  f3 lin, ang; link_velocity(S, e, ee_link, link_com(S, e, ee_link), lin, ang);
  return norm(lin);
}

// ---- pieces of an observation row: write at o[i], return the next index
AG_HD int put3(float* o, int i, f3 v) { o[i] = v.x; o[i + 1] = v.y; o[i + 2] = v.z; return i + 3; }
AG_HD int put4(float* o, int i, q4 v) { o[i] = v.x; o[i + 1] = v.y; o[i + 2] = v.z; o[i + 3] = v.w; return i + 4; }
// the robot's 7 arm angles wrapped to [-pi, pi) (`(angles + pi) % (2 pi) - pi` in every task's _get_obs)
AG_HD int put_arm_angles(const SimDev& S, int e, const int32_t* arm_links, float* o, int i) {
  const float PI = 3.14159265358979323846f;
  for (int j = 0; j < 7; j++) {
    float q = ld1(S.jq, arm_links[j], S.N, e) + PI;
    o[i + j] = q - 2.f * PI * floorf(q / (2.f * PI)) - PI;
  }
  return i + 7;
}
// the person's shoulder, elbow and wrist link positions in a frame
AG_HD int put_arm_points(const SimDev& S, int e, const Frame& fr, const int32_t* links3, float* o, int i) {
  for (int j = 0; j < 3; j++) i = put3(o, i, to_frame(fr, ld3(S.lpos, links3[j], S.N, e)));
  return i;
}

// ---- the sorted contact records of an env (p.getContactPoints, agent.py:100-116).  A record's key holds its collider
// pair above two bits of point index; links and bodies follow from the colliders, the force from the normal impulse.
struct Contact { int la, lb, ba, bb; };
AG_HD int n_contacts(const SimDev& S, int e) { int cnt = S.c_count[e]; return cnt > S.maxc ? S.maxc : cnt; }
AG_HD Contact contact_at(const SimDev& S, int e, int s) {
  const int N = S.N;
  unsigned pk = S.s_key[(size_t)s * N + e] >> 2;
  int ca = (int)(pk / (unsigned)S.nc), cb = (int)(pk % (unsigned)S.nc);
  Contact c;
  c.la = AG_LDG(S.col_link + ca); c.lb = AG_LDG(S.col_link + cb);
  c.ba = AG_LDG(S.link_body + c.la); c.bb = AG_LDG(S.link_body + c.lb);
  return c;
}
AG_HD float contact_force(const SimDev& S, int e, int s) { return cf_ld(S.s_data, s, CF_LAM_N, S.N, e) / S.dt; }
AG_HD f3 contact_point_a(const SimDev& S, int e, int s) {
  const int N = S.N;
  return f3(cf_ld(S.s_data, s, CF_PAX, N, e), cf_ld(S.s_data, s, CF_PAY, N, e), cf_ld(S.s_data, s, CF_PAZ, N, e));
}
AG_HD f3 contact_point_b(const SimDev& S, int e, int s) {
  const int N = S.N;
  return f3(cf_ld(S.s_data, s, CF_PBX, N, e), cf_ld(S.s_data, s, CF_PBY, N, e), cf_ld(S.s_data, s, CF_PBZ, N, e));
}
// the contact point on `body`'s side of a record that `body` takes part in
AG_HD f3 contact_point_on(const SimDev& S, int e, int s, const Contact& c, int body) {
  return c.ba == body ? contact_point_a(S, e, s) : contact_point_b(S, e, s);
}
// is the person one side of the contact, and then which body and link is the other side
AG_HD bool other_of(const Contact& c, int human_body, int& other_body, int& other_link) {
  if (c.ba == human_body) { other_body = c.bb; other_link = c.lb; return true; }
  if (c.bb == human_body) { other_body = c.ba; other_link = c.la; return true; }
  return false;
}

// ---- the task-independent parts of an env step
// The robot's half of take_step (env.py:186-197) for a 7-joint arm: the raw action row is kept in `action` [7][N] (the reward's
// action term), clipped to [-1, 1], scaled, accumulated frame_skip times inside the joint limits; the result is each joint's
// PD target.  Every task's pre kernel calls it.
AG_HD void arm_action_targets(const SimDev& S, int e, const float* act, float* action, const int32_t* arm_links, const float* lower,
                              const float* upper, float multiplier, int frame_skip) {
  const int N = S.N;
  for (int j = 0; j < 7; j++) {
    float raw = act[j];
    action[(size_t)j * N + e] = raw;
    float a = clampf(raw, -1.f, 1.f) * multiplier;
    int k = arm_links[j];
    float q = ld1(S.jq, k, N, e);
    float lo = lower[j], hi = upper[j];
    for (int s = 0; s < frame_skip; s++) {
      if (q + a < lo) { a = 0.f; q = lo; }
      if (q + a > hi) { a = 0.f; q = hi; }
      q += a;
    }
    st1(S.motor_target, k, N, e, q);
  }
}
// tremor (env.py:212-215): the joints are driven to rest +- amplitude, the sign flips every env step.  rest, amp = [n][N]
AG_HD void tremor_targets(const SimDev& S, int e, int n, const int32_t* links, const float* rest, const float* amp, int iteration) {
  const int N = S.N;
  float sgn = (iteration % 2 == 0) ? 1.f : -1.f;
  for (int j = 0; j < n; j++) st1(S.motor_target, links[j], N, e, rest[(size_t)j * N + e] + sgn * amp[(size_t)j * N + e]);
}
// norm of the whole raw action row: the robot's 7 kept by arm_action_targets, then the person's i0 entries of act [N][7 + i0]
AG_HD float action_norm(const SimDev& S, int e, const float* action, const float* act, int i0) {
  const int N = S.N;
  float an = 0.f;
  for (int j = 0; j < 7; j++) { float a = action[(size_t)j * N + e]; an += a * a; }
  for (int j = 0; j < i0; j++) { float a = act[(size_t)e * (7 + i0) + 7 + j]; an += a * a; }
  return sqrtf(an);
}
AG_HD float episode_done(int iteration) { return iteration >= 200 ? 1.f : 0.f; }

// is any collider of link `tool_link` within `dist` of collider `col`?  (p.getClosestPoints of a food / water particle and the
// tool, feeding.py:71, drinking.py:62)
AG_HD bool tool_within(const SimDev& S, int e, int col, int tool_link, float dist) {
  const int N = S.N;
  f3 pmin = ld3(S.cmin, col, N, e), pmax = ld3(S.cmax, col, N, e);
  if (!aabb_ov(pmin, pmax, ld3(S.lmin, tool_link, N, e), ld3(S.lmax, tool_link, N, e), dist)) return false;
  int c0 = AG_LDG(S.link_col0 + tool_link), ncl = AG_LDG(S.link_ncol + tool_link);
  for (int c = c0; c < c0 + ncl; c++) {
    if (!aabb_ov(pmin, pmax, ld3(S.cmin, c, N, e), ld3(S.cmax, c, N, e), dist)) continue;
    NpOut out;
    if (narrow_closest(S, e, col, c, dist, out)) return true;
  }
  return false;
}
// a consumed particle (free body `body`) leaves the scene: a random point far away, its link pose reset with it
// (feeding.py:60-61, drinking.py:70-71)
AG_HD void send_far(const SimDev& S, int e, int body, unsigned long long& rs) {
  const int N = S.N;
  int l0 = AG_LDG(S.body_link0 + body);
  f3 far(1000.f + 1000.f * rng_uniform(rs), 1000.f + 1000.f * rng_uniform(rs), 1000.f + 1000.f * rng_uniform(rs));
  st3(S.base_pos, body, N, e, far); st4(S.base_quat, body, N, e, q4());
  st3(S.lpos, l0, N, e, far); st4(S.lquat, l0, N, e, q4());
}
