// ag_feeding.cuh — the fused FeedingEnv step.
//
// Reference semantics restated here:
//   feeding_pre         AssistiveEnv.take_step action -> PD targets (envs/env.py:174-222)
//   feeding_food/post   FeedingEnv._get_obs / get_food_rewards / reward assembly (envs/feeding.py:12-112),
//                       AssistiveEnv.human_preferences (envs/env.py:237-274)
#pragma once
#include "ag_task.cuh"
#include "../../include/agphys.h"

struct FeedDev {
  AgFeedingParams P;
  int *male, *food_state, *iteration, *task_success, *food_near;
  float* action;
  unsigned long long* rng;
  int* tremor_on; float *tremor_rest, *tremor_amp;     // [N], [4][N], [4][N]
};

// action -> PD targets.  p0 = action [N][7 + i0] (env-major; the robot's 7 come first), p1 = FeedDev*
AG_HDN inline void feeding_pre_body(int e, const SimDev& S, const KP& p) {
  const FeedDev& F = *(const FeedDev*)p.p1;
  const float* act = (const float*)p.p0 + (size_t)e * (7 + p.i0);
  F.iteration[e] += 1;
  arm_action_targets(S, e, act, F.action, F.P.arm_links, F.P.arm_lower, F.P.arm_upper, F.P.action_multiplier, F.P.frame_skip);
  // the head joints of a tremor person
  if (F.tremor_on[e]) tremor_targets(S, e, 4, F.male[e] != 0 ? F.P.head_joints_m : F.P.head_joints_f, F.tremor_rest, F.tremor_amp, F.iteration[e]);
}

// thread = (food i, env e): is any spoon collider within 0.1 of the food sphere? (feeding.py:71)
AG_HDN inline void feeding_food_body(int tid, const SimDev& S, const KP& p) {
  const int N = S.N;
  const FeedDev& F = *(const FeedDev*)p.p1;
  int e = tid % N, i = tid / N;
  int near = 0;
  if ((F.food_state[e] >> i) & 1) {
    int lf = AG_LDG(S.body_link0 + F.P.food_body0 + i), lt = AG_LDG(S.body_link0 + F.P.tool_body);
    near = tool_within(S, e, AG_LDG(S.link_col0 + lf), lt, 0.1f);
  }
  F.food_near[(size_t)i * N + e] = near;
}

// obs / reward / done.  p0 = action [N][7 + i0], p1 = FeedDev*, p2 = obs [N][25], p3 = reward, p4 = done, p5 = info [N][4].
// The reward's action term is the norm of the whole raw action row (the person's i0 entries too, step_reference_api).
AG_HDN inline void feeding_post_body(int e, const SimDev& S, const KP& p) {
  const int N = S.N;
  const FeedDev& F = *(const FeedDev*)p.p1;
  const AgFeedingParams& P = F.P;
  bool male = F.male[e] != 0;
  int hb = male ? P.human_body_m : P.human_body_f;
  // poses: the spoon's COM frame, the head and the mouth target, in the robot's base frame
  Frame fr = body_frame(S, e, P.robot_body);
  f3 sp, hp; q4 sq, hq;
  link_com_pose(S, e, AG_LDG(S.body_link0 + P.tool_body), sp, sq);
  f3 target = mouth_target(S, e, male ? P.head_link_m : P.head_link_f, male ? P.mouth_m : P.mouth_f, hp, hq);
  f3 sp_r = to_frame(fr, sp), tg_r = to_frame(fr, target);
  // contact forces on the human from the robot and from the spoon; food-human contacts
  float robot_force = 0.f, spoon_force = 0.f;
  int food_hit_mask = 0;
  int cnt = n_contacts(S, e);
  for (int s = 0; s < cnt; s++) {
    Contact c = contact_at(S, e, s);
    int other, other_link;
    if (!other_of(c, hb, other, other_link)) continue;
    float force = contact_force(S, e, s);
    if (other == P.robot_body) robot_force += force;
    else if (other == P.tool_body) spoon_force += force;
    else if (other >= P.food_body0 && other < P.food_body0 + P.n_foods) food_hit_mask |= 1 << (other - P.food_body0);
  }
  float total_force = robot_force + spoon_force;
  float* obs = (float*)p.p2 + (size_t)e * 25;
  int o = put3(obs, 0, sp_r); o = put4(obs, o, to_frame(fr, sq)); o = put3(obs, o, sp_r - tg_r);
  o = put_arm_angles(S, e, P.arm_links, obs, o);
  o = put3(obs, o, to_frame(fr, hp)); o = put4(obs, o, to_frame(fr, hq));
  obs[o] = spoon_force;
  // food bookkeeping (feeding.py:50-83)
  int st = F.food_state[e];
  int foods = st & 0xffff, active = (st >> 16) & 0xffff;
  float food_reward = 0.f, vel_sum = 0.f, food_hit = 0.f;
  int success = F.task_success[e];
  unsigned long long rs = F.rng[e];
  int active_at_entry = active;
  for (int i = 0; i < P.n_foods; i++) {
    if (!((foods >> i) & 1)) continue;
    int fb = P.food_body0 + i;
    f3 fp = ld3(S.lpos, AG_LDG(S.body_link0 + fb), N, e);
    if (norm(target - fp) < 0.03f) {
      food_reward += 20.f; success += 1;
      vel_sum += norm(ld3(S.base_lin, fb, N, e));
      foods &= ~(1 << i); active &= ~(1 << i);
      send_far(S, e, fb, rs);
    } else if (!F.food_near[(size_t)i * N + e]) {
      food_reward -= 5.f; foods &= ~(1 << i);
    }
  }
  for (int i = 0; i < P.n_foods; i++) {
    if (!((active_at_entry >> i) & 1)) continue;
    if ((food_hit_mask >> i) & 1) { food_hit -= 1.f; active &= ~(1 << i); }
  }
  F.food_state[e] = foods | (active << 16);
  F.task_success[e] = success;
  F.rng[e] = rs;
  float ee_vel = ee_speed(S, e, P.ee_link);
  // human preferences (env.py:237-274), task == 'feeding'
  float r_vel = -ee_vel;
  float r_high = spoon_force < 10.f ? 0.f : -spoon_force;
  float r_nontarget = -total_force;
  float pref = P.c_v * r_vel + P.c_f * r_nontarget + P.c_hf * r_high + P.c_fd * food_hit + P.c_fdv * (-vel_sum);
  float an = action_norm(S, e, F.action, (const float*)p.p0, p.i0);
  float reward = P.w_distance * (-norm(target - sp)) + P.w_action * (-an) + P.w_food * food_reward + pref;
  ((float*)p.p3)[e] = reward;
  ((float*)p.p4)[e] = episode_done(F.iteration[e]);
  float* info = (float*)p.p5 + (size_t)e * 4;
  info[0] = total_force; info[1] = ((float)success >= P.n_foods * P.task_success_threshold) ? 1.f : 0.f;
  info[2] = robot_force; info[3] = spoon_force;
}
