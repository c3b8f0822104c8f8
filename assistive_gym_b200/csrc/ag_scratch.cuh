// ag_scratch.cuh — fused ScratchItchEnv step (reference envs/scratch_itch.py:10-91 + envs/env.py:174-274): action -> PD targets ->
// frame_skip substeps -> obs[30] / reward / done, with the scratch bookkeeping of get_total_force (scratch_itch.py:46-58) and
// the "moved more than 1 cm along the target" reward (scratch_itch.py:26-30).  SURVEY.md section 8(f)3.
#pragma once
#include "ag_task.cuh"
#include "../../include/agphys.h"

struct ScratchDev {
  AgScratchParams P;
  int *male, *iteration, *task_success;
  int* limb_link;                 // [N] global link id of the limb that carries the target (upper arm or forearm)
  float* target_local;            // [3][N] target point in that link's frame (util.point_on_capsule)
  float* prev_contact;            // [3][N] prev_target_contact_pos
  float* action;                  // [7][N]
};

// p0 = action [N][7 + i0] (env-major; the robot's 7 come first), p1 = ScratchDev*
AG_HDN inline void scratch_pre_body(int e, const SimDev& S, const KP& p) {
  const ScratchDev& D = *(const ScratchDev*)p.p1;
  const float* act = (const float*)p.p0 + (size_t)e * (7 + p.i0);
  D.iteration[e] += 1;
  arm_action_targets(S, e, act, D.action, D.P.arm_links, D.P.arm_lower, D.P.arm_upper, D.P.action_multiplier, D.P.frame_skip);
}

// p0 = action [N][7 + i0] (the reward's action term covers the whole raw row), p1 = ScratchDev*, p2 = obs [N][30], p3 = reward, p4 = done, p5 = info [N][4] = total force on the person, task
// success, tool force at the target, scratches so far
AG_HDN inline void scratch_post_body(int e, const SimDev& S, const KP& p) {
  const int N = S.N;
  const ScratchDev& D = *(const ScratchDev*)p.p1;
  const AgScratchParams& P = D.P;
  bool male = D.male[e] != 0;
  int hb = male ? P.human_body_m : P.human_body_f;
  Frame fr = body_frame(S, e, P.robot_body);
  f3 tp = ld3(S.lpos, P.tool_tip_link, N, e); q4 tq = ld4(S.lquat, P.tool_tip_link, N, e);
  int limb = D.limb_link[e];
  f3 target = ld3(S.lpos, limb, N, e) + qrot(ld4(S.lquat, limb, N, e), ld3(D.target_local, 0, N, e));     // update_targets (scratch_itch.py:149-153)
  f3 tp_r = to_frame(fr, tp), tg_r = to_frame(fr, target);
  float* obs = (float*)p.p2 + (size_t)e * 30;
  int o = put3(obs, 0, tp_r); o = put4(obs, o, to_frame(fr, tq)); o = put3(obs, o, tp_r - tg_r); o = put3(obs, o, tg_r);
  o = put_arm_angles(S, e, P.arm_links, obs, o);
  o = put_arm_points(S, e, fr, male ? P.arm_points_m : P.arm_points_f, obs, o);
  // forces (scratch_itch.py:46-58)
  float tool_force = 0.f, at_target = 0.f, total_on_human = 0.f;
  f3 contact_pos(0.f, 0.f, 0.f); bool have_contact = false;
  int cnt = n_contacts(S, e);
  for (int s = 0; s < cnt; s++) {
    Contact c = contact_at(S, e, s);
    float force = contact_force(S, e, s);
    if (c.ba == P.tool_body || c.bb == P.tool_body) tool_force += force;
    int other, lo;
    if (!other_of(c, hb, other, lo)) continue;
    if (other == P.robot_body) total_on_human += force;
    else if (other == P.tool_body) {
      total_on_human += force;
      f3 ph = contact_point_on(S, e, s, c, hb);
      if ((lo == P.tool_link0 || lo == P.tool_tip_link) && norm(ph - target) < 0.025f) { at_target += force; contact_pos = ph; have_contact = true; }
    }
  }
  obs[o] = tool_force;
  float scratch = 0.f;
  int success = D.task_success[e];
  if (have_contact && norm(contact_pos - ld3(D.prev_contact, 0, N, e)) > 0.01f && at_target < 10.f) {
    scratch = 5.f; st3(D.prev_contact, 0, N, e, contact_pos); success += 1;
  }
  D.task_success[e] = success;
  float pref = P.c_v * (-ee_speed(S, e, P.ee_link)) + P.c_f * (-(total_on_human - at_target)) + P.c_hf * (at_target < 10.f ? 0.f : -at_target);
  float an = action_norm(S, e, D.action, (const float*)p.p0, p.i0);
  ((float*)p.p3)[e] = P.w_distance * (-norm(target - tp)) + P.w_action * (-an) + P.w_scratch * scratch + pref;
  ((float*)p.p4)[e] = episode_done(D.iteration[e]);
  float* info = (float*)p.p5 + (size_t)e * 4;
  info[0] = total_on_human; info[1] = (float)success >= P.task_success_threshold ? 1.f : 0.f; info[2] = at_target; info[3] = (float)success;
}
