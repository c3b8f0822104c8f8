// ag_coop.cuh — the person's half of the fused co-optimisation step (FeedingJacoHuman-v1, ScratchItchJacoHuman-v1,
// BedBathingSawyerHuman-v1, DressingPR2Human-v1).
//
// Reference semantics restated here:
//   coop_pre      AssistiveEnv.take_step for the Human agent (envs/env.py:174-222): the human slice of the action, clipped and
//                 x 0.05 (the Robot-only action_multiplier does not apply), accumulated frame_skip times inside the person's
//                 controllable limits (scaled per env by Human.set_limit_scale) -> motor targets; for a tremor person
//                 (ag_coop_set_tremor) accumulated into the env's target_joint_angles instead, the motors driven to
//                 target +- amplitude (env.py:212-215).  The task's own tremor (k_feed_pre / k_dress_pre) is off in this step.
//   coop_limits   after every stepSimulation (env.py:223-231): Human.enforce_joint_limits over every joint of the person, then
//                 Human.enforce_realistic_joint_limits (agents/human.py:134-152): the joint-limit MLP classifies the arm pose,
//                 an unreachable pose is replaced by the env's last reachable one
//   coop_obs      the person's observation in its own base frame: FeedingEnv._get_obs (feeding.py:101-111, 23 floats),
//                 ScratchItchEnv._get_obs (scratch_itch.py:75-84, 34 floats), BedBathingEnv._get_obs (bed_bathing.py:97-105, 28 floats),
//                 DressingEnv._get_obs (dressing.py:96-105, 28 floats)
// The robot's half, the reward, done and info are the task's own kernels (k_feed_* / k_scratch_* / k_bath_* / k_dress_*), which
// read the wider action rows through KP.i0.
//
// The limit arithmetic and the classifier's input mapping run in fp64, as the per-call path does on the host, so that the
// clamps, the motor targets and the fp32 classifier inputs are the host's values.  The classifier itself is plain fp32 FMAs
// in the layer order of limits_model.ArmLimitsModel.predict.
#pragma once
#include <math.h>
#include "ag_task.cuh"
#include "ag_bathing.cuh"
#include "ag_dressing.cuh"
#include "ag_feeding.cuh"
#include "ag_scratch.cuh"
#include "../../include/agphys.h"

#define AG_MLP_H 64
#define AG_MLP_FLOATS (4 * AG_MLP_H + AG_MLP_H + 2 * (AG_MLP_H * AG_MLP_H + AG_MLP_H) + AG_MLP_H + 1)     // 8705 (34 820 B)

struct CoopDev {
  AgCoopParams P;
  int frame_skip;
  int mlp_on;
  const int* male;          // the task's per-env gender flags
  double* limit_scale;      // [N]
  float* prev_pose;         // [4][N] last reachable shoulder x/y/z + elbow; NaN = none yet (human.py:68 `None`)
  const float* mlp;         // [AG_MLP_FLOATS], packed as in agphys.h
  const int* iteration;     // the task's per-env step counter, advanced by the task's pre kernel before k_coop_pre runs
  int* tremor_on;           // [N] the person's impairment is 'tremor' (human.py:80-92); all 0 unless ag_coop_set_tremor
  double* tremor_target;    // [AG_COOP_MAXC][N] target_joint_angles (human.py:123), accumulated by the action (env.py:214)
  float* tremor_amp;        // [AG_COOP_MAXC][N] the tremor amplitudes (human.py:87-92)
};

// The 4-64-64-64-1 classifier: tanh hidden layers, sigmoid output.  `h` is the caller's scratch of 2 x 64 floats with element
// i at h[i * hs] (a per-thread column of shared memory on the device).  Each neuron sums its inputs in order, then adds the bias.
AG_HD void coop_mlp_layer(const float* in, float* out, int hs, const float* W, const float* b) {
  for (int j = 0; j < AG_MLP_H; j++) {
    float acc = 0.f;
    for (int i = 0; i < AG_MLP_H; i++) acc = fmaf(in[i * hs], W[i * AG_MLP_H + j], acc);
    out[j * hs] = tanhf(acc + b[j]);
  }
}
AG_HD float coop_mlp(const float* w, const float x[4], float* h, int hs) {
  const float* W1 = w;
  const float* b1 = W1 + 4 * AG_MLP_H;
  const float* W2 = b1 + AG_MLP_H;
  const float* b2 = W2 + AG_MLP_H * AG_MLP_H;
  const float* W3 = b2 + AG_MLP_H;
  const float* b3 = W3 + AG_MLP_H * AG_MLP_H;
  const float* W4 = b3 + AG_MLP_H;
  const float* b4 = W4 + AG_MLP_H;
  float* ha = h;
  float* hb = h + AG_MLP_H * hs;
  for (int j = 0; j < AG_MLP_H; j++) {
    float acc = 0.f;
    for (int i = 0; i < 4; i++) acc = fmaf(x[i], W1[i * AG_MLP_H + j], acc);
    ha[j * hs] = tanhf(acc + b1[j]);
  }
  coop_mlp_layer(ha, hb, hs, W2, b2);
  coop_mlp_layer(hb, ha, hs, W3, b3);
  float acc = 0.f;
  for (int i = 0; i < AG_MLP_H; i++) acc = fmaf(ha[i * hs], W4[i], acc);
  return 1.f / (1.f + expf(-(acc + b4[0])));
}

// Python's float `%` for a positive modulus (the sign of the result follows the modulus)
AG_HD double py_mod(double v, double m) {
  double r = fmod(v, m);
  if (r < 0.0) r += m;
  return r;
}

// the classifier's input convention (human.py:141-144): angles of shoulder x/y/z and elbow -> x[4]
AG_HD void coop_mlp_input(const float ang[4], double sign, float x[4]) {
  const double two_pi = 2.0 * 3.141592653589793;
  x[0] = (float)py_mod(sign * (double)ang[0] + two_pi, two_pi);
  x[1] = (float)py_mod((double)ang[1] + two_pi, two_pi);
  x[2] = (float)(sign * (double)ang[2]);
  x[3] = (float)py_mod(-(double)ang[3] + two_pi, two_pi);
}

// p0 = action [N][7 + n_ctrl] (env-major), p1 = CoopDev*.  A tremor person (env.py:205-215): the limit checks and the zeroing of
// the action run against the angles of the previous pass, the action accumulates into the env's target, and the angles become
// target + amplitude, its sign flipping with the task's step counter (already advanced for this step).
AG_HDN inline void coop_pre_body(int e, const SimDev& S, const KP& p) {
  const int N = S.N;
  const CoopDev& C = *(const CoopDev*)p.p1;
  const AgCoopParams& P = C.P;
  const float* act = (const float*)p.p0 + (size_t)e * (7 + P.n_ctrl) + 7;
  const int* links = C.male[e] ? P.joint_links_m : P.joint_links_f;
  const double sc = C.limit_scale[e];
  const bool tremor = C.tremor_on[e] != 0;
  for (int c = 0; c < P.n_ctrl; c++) {
    const int j = P.ctrl[c], k = links[j];
    double a = fmin(fmax((double)act[c], -1.0), 1.0) * 0.05;
    double q = ld1(S.jq, k, N, e);
    const double lo = (double)P.joint_lower[j] * sc, hi = (double)P.joint_upper[j] * sc;
    if (!tremor) {
      for (int s = 0; s < C.frame_skip; s++) {
        if (q + a < lo) { a = 0.0; q = lo; }
        if (q + a > hi) { a = 0.0; q = hi; }
        q += a;
      }
    } else {
      const double wobble = (double)C.tremor_amp[(size_t)c * N + e] * (C.iteration[e] % 2 == 0 ? 1.0 : -1.0);
      double t = C.tremor_target[(size_t)c * N + e];
      for (int s = 0; s < C.frame_skip; s++) {
        if (q + a < lo) { a = 0.0; q = lo; }
        if (q + a > hi) { a = 0.0; q = hi; }
        t += a;
        q = t + wobble;
      }
      C.tremor_target[(size_t)c * N + e] = t;
    }
    st1(S.motor_target, k, N, e, (float)q);
  }
}

// after one stepSimulation.  w = classifier weights, h = scratch for coop_mlp
AG_HDN inline void coop_limits_body(int e, const SimDev& S, const CoopDev& C, const float* w, float* h, int hs) {
  const int N = S.N;
  const AgCoopParams& P = C.P;
  const int* links = C.male[e] ? P.joint_links_m : P.joint_links_f;
  const double sc = C.limit_scale[e];
  for (int j = 0; j < P.n_joints; j++) {
    const int k = links[j];
    const double q = ld1(S.jq, k, N, e);
    const double lo = (double)P.joint_lower[j] * sc, hi = (double)P.joint_upper[j] * sc;
    if (q < lo || q > hi) { st1(S.jq, k, N, e, (float)fmin(fmax(q, lo), hi)); st1(S.jqd, k, N, e, 0.f); }
  }
  if (!C.mlp_on) return;
  float ang[4], x[4];
  for (int s = 0; s < 4; s++) ang[s] = ld1(S.jq, links[P.mlp_slots[s]], N, e);
  coop_mlp_input(ang, (double)P.mlp_sign, x);
  const float prob = coop_mlp(w, x, h, hs);
  float* prev = C.prev_pose;
  if (prob > 0.5f) {
    for (int s = 0; s < 4; s++) prev[(size_t)s * N + e] = ang[s];
  } else if (!isnan(prev[e])) {               // restore the last reachable pose, clipped to the template limits, at rest
    for (int s = 0; s < 4; s++) {
      const int j = P.mlp_slots[s], k = links[j];
      const double q = prev[(size_t)s * N + e];
      st1(S.jq, k, N, e, (float)fmin(fmax(q, (double)P.joint_lower[j]), (double)P.joint_upper[j]));
      st1(S.jqd, k, N, e, 0.f);
    }
  }
}

// p1 = CoopDev*, p2 = FeedDev* | ScratchDev* | BathDev* | DressPost*, p3 = obs_human [N][23 | 34 | 28 | 28], p4 = info [N][4]
// written by the task's post kernel
AG_HDN inline void coop_obs_body(int e, const SimDev& S, const KP& p) {
  const int N = S.N;
  const CoopDev& C = *(const CoopDev*)p.p1;
  const AgCoopParams& P = C.P;
  const bool male = C.male[e] != 0;
  const int* links = male ? P.joint_links_m : P.joint_links_f;
  const Frame fr = body_frame(S, e, male ? P.human_body_m : P.human_body_f);      // the person's base frame
  const float* info = (const float*)p.p4 + (size_t)e * 4;
  int i = 0;
  if (P.task == 0) {                          // feeding.py:101-111
    const FeedDev& F = *(const FeedDev*)p.p2;
    f3 sp, hp; q4 sq, hq;
    link_com_pose(S, e, AG_LDG(S.body_link0 + F.P.tool_body), sp, sq);
    f3 target = mouth_target(S, e, male ? F.P.head_link_m : F.P.head_link_f, male ? F.P.mouth_m : F.P.mouth_f, hp, hq);
    float* o = (float*)p.p3 + (size_t)e * 23;
    f3 sp_h = to_frame(fr, sp), tg_h = to_frame(fr, target);
    i = put3(o, i, sp_h); i = put4(o, i, to_frame(fr, sq)); i = put3(o, i, sp_h - tg_h);
    for (int c = 0; c < P.n_ctrl; c++) o[i++] = ld1(S.jq, links[P.ctrl[c]], N, e);
    i = put3(o, i, to_frame(fr, hp)); i = put4(o, i, to_frame(fr, hq));
    o[i++] = info[2];                         // robot force on the person
    o[i++] = info[3];                         // spoon force on the person
  } else if (P.task == 2) {                   // bed_bathing.py:97-105
    const BathDev& B = *(const BathDev*)p.p2;
    float* o = (float*)p.p3 + (size_t)e * 28;
    i = put3(o, i, to_frame(fr, ld3(S.lpos, B.P.cloth_link, N, e))); i = put4(o, i, to_frame(fr, ld4(S.lquat, B.P.cloth_link, N, e)));
    for (int c = 0; c < P.n_ctrl; c++) o[i++] = ld1(S.jq, links[P.ctrl[c]], N, e);
    i = put_arm_points(S, e, fr, male ? B.P.arm_points_m : B.P.arm_points_f, o, i);
    o[i++] = info[0];                         // total force on the person
    o[i++] = info[2];                         // wiper-cloth force on the person
  } else if (P.task == 3) {                   // dressing.py:96-105
    const DressDev& D = ((const DressPost*)p.p2)->D;
    float* o = (float*)p.p3 + (size_t)e * 28;
    i = put3(o, i, to_frame(fr, ld3(S.lpos, D.P.ee_link, N, e))); i = put4(o, i, to_frame(fr, ld4(S.lquat, D.P.ee_link, N, e)));
    for (int c = 0; c < P.n_ctrl; c++) o[i++] = ld1(S.jq, links[P.ctrl[c]], N, e);
    i = put_arm_points(S, e, fr, male ? D.P.arm_points_m : D.P.arm_points_f, o, i);
    o[i++] = D.person_force[e];               // cloth force sum (k_dress_post)
    o[i++] = D.person_force[(size_t)N + e];   // robot force on the person
  } else {                                    // scratch_itch.py:75-84
    const ScratchDev& D = *(const ScratchDev*)p.p2;
    const int limb = D.limb_link[e];
    f3 target = ld3(S.lpos, limb, N, e) + qrot(ld4(S.lquat, limb, N, e), ld3(D.target_local, 0, N, e));
    float* o = (float*)p.p3 + (size_t)e * 34;
    f3 tp_h = to_frame(fr, ld3(S.lpos, D.P.tool_tip_link, N, e)), tg_h = to_frame(fr, target);
    i = put3(o, i, tp_h); i = put4(o, i, to_frame(fr, ld4(S.lquat, D.P.tool_tip_link, N, e))); i = put3(o, i, tp_h - tg_h); i = put3(o, i, tg_h);
    for (int c = 0; c < P.n_ctrl; c++) o[i++] = ld1(S.jq, links[P.ctrl[c]], N, e);
    i = put_arm_points(S, e, fr, male ? D.P.arm_points_m : D.P.arm_points_f, o, i);
    o[i++] = info[0];                         // total force on the person
    o[i++] = info[2];                         // tool force at the target
  }
}
