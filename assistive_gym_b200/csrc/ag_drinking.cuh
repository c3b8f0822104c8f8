// ag_drinking.cuh — fused DrinkingEnv step (reference envs/drinking.py:10-117 + envs/env.py:174-274): action -> PD targets ->
// frame_skip substeps -> obs[25] / reward / done, with the water bookkeeping of get_water_rewards (drinking.py:51-82) and the
// human preferences of task 'drinking' (env.py:237-274).
//
//   drinking_pre    take_step's robot half (the same arithmetic as Feeding's, arm_action_targets)
//   drinking_water  one thread per (particle, env): in the cup (util.points_in_cylinder), swallowed, spilled, or outside the
//                   cup but still near it (p.getClosestPoints(water, cup, 0.1), asked only of particles that left the cup)
//   drinking_post   one thread per env: observation, forces and water hits from the contact records, the bookkeeping, reward
#pragma once
#include "ag_task.cuh"
#include "../../include/agphys.h"

struct DrinkDev {
  AgDrinkingParams P;
  int *male, *iteration, *task_success;
  unsigned long long *waters, *waters_active;   // [N] bit i: particle i still in play / can still hit the person
  unsigned long long* rng;                      // [N] xorshift state: where swallowed particles go
  int* status;                                  // [64][N] drinking_water -> drinking_post (DW_*)
  float* action;                                // [7][N] the raw action
};
enum { DW_IN = 0, DW_NEAR = 1, DW_SWALLOWED = 2, DW_SPILLED = 3 };

// the cup's COM frame, the mouth target and the cup's top / bottom centres (drinking.py:24-26, 54-57, 192-196)
struct DrinkPose { f3 cp; q4 cq; f3 hp; q4 hq; f3 target; q4 fq; f3 top, bottom; };
AG_HD DrinkPose drink_pose(const SimDev& S, const AgDrinkingParams& P, int e, bool male) {
  DrinkPose c;
  link_com_pose(S, e, AG_LDG(S.body_link0 + P.tool_body), c.cp, c.cq);
  c.target = mouth_target(S, e, male ? P.head_link_m : P.head_link_f, male ? P.mouth_m : P.mouth_f, c.hp, c.hq);
  f3 fp = c.cp + qrot(c.cq, f3(P.cup_frame_pos[0], P.cup_frame_pos[1], P.cup_frame_pos[2]));
  c.fq = qmul(c.cq, q4(P.cup_frame_quat[0], P.cup_frame_quat[1], P.cup_frame_quat[2], P.cup_frame_quat[3]));
  c.top = fp + qrot(c.fq, f3(P.cup_top[0], P.cup_top[1], P.cup_top[2]));
  c.bottom = fp + qrot(c.fq, f3(P.cup_bottom[0], P.cup_bottom[1], P.cup_bottom[2]));
  return c;
}

// util.points_in_cylinder (util.py:53-56): q between the end caps and within r of the axis pt1 -> pt2
AG_HD bool in_cylinder(f3 pt1, f3 pt2, float r, f3 q) {
  f3 v = pt2 - pt1, a = q - pt1, b = q - pt2;
  return dot(a, v) >= 0.f && dot(b, v) <= 0.f && norm(cross(a, v)) <= r * norm(v);
}

// p0 = action [N][7 + i0] (env-major; the robot's 7 come first), p1 = DrinkDev*
AG_HDN inline void drinking_pre_body(int e, const SimDev& S, const KP& p) {
  const DrinkDev& D = *(const DrinkDev*)p.p1;
  const float* act = (const float*)p.p0 + (size_t)e * (7 + p.i0);
  D.iteration[e] += 1;
  arm_action_targets(S, e, act, D.action, D.P.arm_links, D.P.arm_lower, D.P.arm_upper, D.P.action_multiplier, D.P.frame_skip);
}

// thread = (particle i, env e), env fastest.  p1 = DrinkDev*.  Writes status[i][e].
AG_HDN inline void drinking_water_body(int tid, const SimDev& S, const KP& p) {
  const int N = S.N;
  const DrinkDev& D = *(const DrinkDev*)p.p1;
  const AgDrinkingParams& P = D.P;
  int e = tid % N, i = tid / N;
  int st = DW_IN;
  if ((D.waters[e] >> i) & 1ull) {
    DrinkPose c = drink_pose(S, P, e, D.male[e] != 0);
    int lw = AG_LDG(S.body_link0 + P.water_body0 + i);
    f3 wp = ld3(S.lpos, lw, N, e);
    if (!in_cylinder(c.top, c.bottom, 0.05f, wp)) {
      if (norm(c.target - wp) < 0.03f) st = DW_SWALLOWED;
      else                               // drinking.py:62: is any cup collider within 0.1 of the particle?
        st = tool_within(S, e, AG_LDG(S.link_col0 + lw), AG_LDG(S.body_link0 + P.tool_body), 0.1f) ? DW_NEAR : DW_SPILLED;
    }
  }
  D.status[(size_t)i * N + e] = st;
}

// obs / reward / done.  p0 = action [N][7 + i0], p1 = DrinkDev*, p2 = obs [N][25], p3 = reward, p4 = done, p5 = info [N][4].
AG_HDN inline void drinking_post_body(int e, const SimDev& S, const KP& p) {
  const int N = S.N;
  const DrinkDev& D = *(const DrinkDev*)p.p1;
  const AgDrinkingParams& P = D.P;
  bool male = D.male[e] != 0;
  int hb = male ? P.human_body_m : P.human_body_f;
  DrinkPose c = drink_pose(S, P, e, male);
  Frame fr = body_frame(S, e, P.robot_body);
  f3 cp_r = to_frame(fr, c.cp), tg_r = to_frame(fr, c.target);
  // contact forces on the person from the robot and from the cup (drinking.py:46-49); particles touching the person
  float robot_force = 0.f, cup_force = 0.f;
  unsigned long long hit = 0ull;
  int cnt = n_contacts(S, e);
  for (int s = 0; s < cnt; s++) {
    Contact k = contact_at(S, e, s);
    int other, other_link;
    if (!other_of(k, hb, other, other_link)) continue;
    float force = contact_force(S, e, s);
    if (other == P.robot_body) robot_force += force;
    else if (other == P.tool_body) cup_force += force;
    else if (other >= P.water_body0 && other < P.water_body0 + P.n_water) hit |= 1ull << (other - P.water_body0);
  }
  float total_force = robot_force + cup_force;
  float* obs = (float*)p.p2 + (size_t)e * 25;
  int o = put3(obs, 0, cp_r); o = put4(obs, o, to_frame(fr, c.cq)); o = put3(obs, o, cp_r - tg_r);
  o = put_arm_angles(S, e, P.arm_links, obs, o);
  o = put3(obs, o, to_frame(fr, c.hp)); o = put4(obs, o, to_frame(fr, c.hq));
  obs[o] = cup_force;
  // water bookkeeping (drinking.py:51-82)
  unsigned long long waters = D.waters[e], active = D.waters_active[e];
  const unsigned long long active_at_entry = active;
  float water_reward = 0.f, vel_sum = 0.f, water_hit = 0.f;
  int success = D.task_success[e];
  unsigned long long rs = D.rng[e];
  for (int i = 0; i < P.n_water; i++) {
    int st = D.status[(size_t)i * N + e];
    unsigned long long bit = 1ull << i;
    if (st == DW_SWALLOWED) {
      int wb = P.water_body0 + i;
      water_reward += 10.f; success += 1;
      vel_sum += norm(ld3(S.base_lin, wb, N, e));
      waters &= ~bit; active &= ~bit;
      send_far(S, e, wb, rs);
    } else if (st == DW_SPILLED) {
      water_reward -= 1.f; waters &= ~bit;
    }
  }
  hit &= active_at_entry;
  for (int i = 0; i < P.n_water; i++) if ((hit >> i) & 1ull) water_hit -= 1.f;
  active &= ~hit;
  D.waters[e] = waters; D.waters_active[e] = active;
  D.task_success[e] = success;
  D.rng[e] = rs;
  // human preferences (env.py:237-274), task == 'drinking'
  float r_high = cup_force < 10.f ? 0.f : -cup_force;
  float pref = P.c_v * (-ee_speed(S, e, P.ee_link)) + P.c_f * (-total_force) + P.c_hf * r_high + P.c_fd * water_hit + P.c_fdv * (-vel_sum);
  float an = action_norm(S, e, D.action, (const float*)p.p0, p.i0);
  // the cup's tilt: roll of its centres' frame (getEulerFromQuaternion(...)[0]) away from upright (pi / 2)
  const float PI = 3.14159265358979323846f;
  float roll = atan2f(2.f * (c.fq.w * c.fq.x + c.fq.y * c.fq.z), 1.f - 2.f * (c.fq.x * c.fq.x + c.fq.y * c.fq.y));
  float reward = P.w_distance * (-norm(c.target - c.top)) + P.w_action * (-an) + P.w_cup_tilt * (-fabsf(roll - 0.5f * PI)) +
                 P.w_drinking * water_reward + pref;
  ((float*)p.p3)[e] = reward;
  ((float*)p.p4)[e] = episode_done(D.iteration[e]);
  float* info = (float*)p.p5 + (size_t)e * 4;
  info[0] = total_force; info[1] = ((float)success >= P.n_water * P.task_success_threshold) ? 1.f : 0.f;
  info[2] = robot_force; info[3] = cup_force;
}
