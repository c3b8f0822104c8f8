// ag_ik.cuh — batched damped-least-squares inverse kinematics with random restarts, one env per thread.
// Restates what the reference asks PyBullet for at reset time: Robot.ik_random_restarts (agents/robot.py:84-121,
// called from AssistiveEnv.init_robot_pose, envs/env.py:296): joint angles inside the limits that bring the end
// effector's link frame to a target pose, re-drawn from random rest poses until position and orientation errors are
// below a threshold.  SURVEY.md §8(f)1 (batched reset).  Kinematics only: reads the scene template and the body's
// base pose, writes nothing but its outputs.
#pragma once
#include "ag_task.cuh"        // xorshift64s / rng_uniform

#define AG_IK_MAXCHAIN 32      // links on the path base -> end effector
#define AG_IK_MAXJ 8           // joints solved for

struct IkDev {
  int body, ee_link, n_chain, n_joints, max_restarts, iters;
  float threshold, damping, step_clip;
  unsigned long long seed;
  int chain[AG_IK_MAXCHAIN];   // global link ids from the first link below the base down to the end effector
  int chain_joint[AG_IK_MAXCHAIN];   // column of the solved joint this link's joint is, or -1 (held at its current angle)
  float lower[AG_IK_MAXJ], upper[AG_IK_MAXJ];
  int col_jtype[AG_IK_MAXJ];   // 1 revolute, 2 prismatic
};

// FK along the chain for joint values qj; fills the joint origins / axes needed by the Jacobian and the ee pose
AG_HDN inline void ik_fk(const SimDev& S, int e, const IkDev& K, const float* qj, f3* org, f3* axw, f3& ep, q4& eq) {
  const int N = S.N;
  int l0 = AG_LDG(S.body_link0 + K.body);
  f3 p = ld3(S.base_pos, K.body, N, e); q4 q = ld4(S.base_quat, K.body, N, e);
  // the base link frame: base pose is the base link's frame origin in this backend's state layout
  (void)l0;
  for (int i = 0; i < K.n_chain; i++) {
    int k = K.chain[i];
    f3 jp = p + qrot(q, tv3(S.link_jpos, k));
    q4 jq = qmul(q, tv4(S.link_jquat, k));
    int jt = AG_LDG(S.link_jtype + k);
    int c = K.chain_joint[i];
    float val = c >= 0 ? qj[c] : ld1(S.jq, k, N, e);
    f3 ax = tv3(S.link_axis, k);
    if (jt == 1) jq = qmul(jq, qaxis(ax, val));
    else if (jt == 2) jp = jp + qrot(jq, ax * val);
    jq = qnormalize(jq);
    if (c >= 0) { org[c] = jp; axw[c] = qrot(jq, ax); }
    p = jp; q = jq;
  }
  ep = p; eq = q;
}

// 6x6 SPD solve by Cholesky (in place); returns false if not positive definite
AG_HDN inline bool ik_chol_solve(float* A, float* b) {
  for (int i = 0; i < 6; i++) {
    for (int j = 0; j <= i; j++) {
      float s = A[i * 6 + j];
      for (int k = 0; k < j; k++) s -= A[i * 6 + k] * A[j * 6 + k];
      if (i == j) { if (!(s > 0.f)) return false; A[i * 6 + i] = sqrtf(s); }
      else A[i * 6 + j] = s / A[j * 6 + j];
    }
  }
  for (int i = 0; i < 6; i++) { float s = b[i]; for (int k = 0; k < i; k++) s -= A[i * 6 + k] * b[k]; b[i] = s / A[i * 6 + i]; }
  for (int i = 5; i >= 0; i--) { float s = b[i]; for (int k = i + 1; k < 6; k++) s -= A[k * 6 + i] * b[k]; b[i] = s / A[i * 6 + i]; }
  return true;
}

// p.p0 = IkDev*, p.p1 = target_pos [N][3], p.p2 = target_quat [N][4], p.p3 = q_out [N][n_joints], p.p4 = err_out [N],
// p.p5 = env mask (int [N]) or null
AG_HDN inline void ik_body(int e, const SimDev& S, const KP& p) {
  const IkDev& K = *(const IkDev*)p.p0;
  const int* mask = (const int*)p.p5;
  float* qo = (float*)p.p3 + (size_t)e * K.n_joints;
  if (mask && !mask[e]) return;
  const float* tpp = (const float*)p.p1 + (size_t)e * 3;
  const float* tqp = (const float*)p.p2 + (size_t)e * 4;
  f3 tp(tpp[0], tpp[1], tpp[2]); q4 tq(tqp[0], tqp[1], tqp[2], tqp[3]);
  const bool pos_only = !(tq.w == tq.w);         // a NaN target orientation: position-only goal (`target_orient=None`, robot.py:86,100)
  const int nj = K.n_joints;
  unsigned long long rs = (K.seed + 0x9E3779B97F4A7C15ull * (unsigned long long)(e + 1)) | 1ull;
  float best[AG_IK_MAXJ], best_err = 1e30f;
  const float PI = 3.14159265358979323846f;
  for (int r = 0; r < K.max_restarts && best_err >= K.threshold; r++) {
    float q[AG_IK_MAXJ];
    for (int j = 0; j < nj; j++) {       // random rest pose inside the limits (continuous joints: one turn)
      float lo = fmaxf(K.lower[j], -PI), hi = fminf(K.upper[j], PI);
      q[j] = lo + (hi - lo) * rng_uniform(rs);
    }
    float err = 1e30f;
    for (int it = 0; it <= K.iters; it++) {
      f3 org[AG_IK_MAXJ], axw[AG_IK_MAXJ], ep; q4 eq;
      ik_fk(S, e, K, q, org, axw, ep, eq);
      f3 dp = tp - ep;
      q4 qe = qmul(tq, qconj(eq));
      if (qe.w < 0.f) qe = q4(-qe.x, -qe.y, -qe.z, -qe.w);
      if (pos_only) qe = q4(0.f, 0.f, 0.f, 1.f);
      float er[6] = {dp.x, dp.y, dp.z, 2.f * qe.x, 2.f * qe.y, 2.f * qe.z};
      // the reference's success test: position distance and orientation (quaternion) distance (robot.py:100-104)
      float oe = fminf(sqrtf((tq.x - eq.x) * (tq.x - eq.x) + (tq.y - eq.y) * (tq.y - eq.y) + (tq.z - eq.z) * (tq.z - eq.z) + (tq.w - eq.w) * (tq.w - eq.w)),
                       sqrtf((tq.x + eq.x) * (tq.x + eq.x) + (tq.y + eq.y) * (tq.y + eq.y) + (tq.z + eq.z) * (tq.z + eq.z) + (tq.w + eq.w) * (tq.w + eq.w)));
      err = pos_only ? norm(dp) : fmaxf(norm(dp), oe);
      float m6 = 0.f; for (int i = 0; i < 6; i++) m6 = fmaxf(m6, fabsf(er[i]));
      if (it == K.iters || m6 < 1e-5f) break;
      float J[6 * AG_IK_MAXJ];
      for (int j = 0; j < nj; j++) {
        f3 a = axw[j];
        int jt = K.col_jtype[j];
        f3 lin = jt == 1 ? cross(a, ep - org[j]) : a, ang = (jt == 1 && !pos_only) ? a : f3();
        J[0 * nj + j] = lin.x; J[1 * nj + j] = lin.y; J[2 * nj + j] = lin.z; J[3 * nj + j] = ang.x; J[4 * nj + j] = ang.y; J[5 * nj + j] = ang.z;
      }
      float A[36];
      for (int i = 0; i < 6; i++) for (int k = 0; k <= i; k++) {
        float s = 0.f; for (int j = 0; j < nj; j++) s += J[i * nj + j] * J[k * nj + j];
        A[i * 6 + k] = s + (i == k ? K.damping * K.damping : 0.f); A[k * 6 + i] = A[i * 6 + k];
      }
      float y[6] = {er[0], er[1], er[2], er[3], er[4], er[5]};
      if (!ik_chol_solve(A, y)) break;
      for (int j = 0; j < nj; j++) {
        float d = 0.f; for (int i = 0; i < 6; i++) d += J[i * nj + j] * y[i];
        q[j] = clampf(q[j] + clampf(d, -K.step_clip, K.step_clip), K.lower[j], K.upper[j]);
      }
    }
    if (err < best_err) { best_err = err; for (int j = 0; j < nj; j++) best[j] = q[j]; }
  }
  for (int j = 0; j < nj; j++) qo[j] = best[j];
  ((float*)p.p4)[e] = best_err;
}
