// ag_bathing.cuh — fused BedBathingEnv step (reference envs/bed_bathing.py:12-111 + envs/env.py:174-274):
// action -> PD targets -> frame_skip substeps -> obs[24] / reward / done, with the wiping-target bookkeeping
// of get_total_force (bed_bathing.py:41-78) as a per-env bit-free mask over the target points.
// With a controllable person (BedBathingSawyerHuman-v1, run by ag_coop.cuh) the right arm moves, and bathing_track_body
// re-places every target on its upper-arm / forearm link (update_targets, bed_bathing.py:190-203).
#pragma once
#include "ag_task.cuh"
#include "../../include/agphys.h"

struct BathDev {
  AgBathingParams P;
  int *male, *iteration, *task_success, *total_targets;
  float* action;                  // [7][N]
  float* targets;                 // [T][3][N] world positions (fixed at reset for a static person, re-placed by k_bath_track)
  int* alive;                     // [T][N] 1 = not wiped yet (0 for padding beyond the env's target count)
  int* target_link;               // [T][N] global link the target rides on, -1 = padding (ag_bathing_set_target_frames)
  float* target_local;            // [T][3][N] the target in that link's frame
  float* dist_part;               // [human collider slot][N] partial minima of the tool-person distance
  int n_slots;                    // max colliders of a person
};

// action -> PD targets (env.py:187-217), same accumulate-with-limit-clamp rule as the feeding path.
// p0 = action [N][7 + i0] (env-major; the robot's 7 come first), p1 = BathDev*
AG_HDN inline void bathing_pre_body(int e, const SimDev& S, const KP& p) {
  const BathDev& B = *(const BathDev*)p.p1;
  const float* act = (const float*)p.p0 + (size_t)e * (7 + p.i0);
  B.iteration[e] += 1;
  arm_action_targets(S, e, act, B.action, B.P.arm_links, B.P.arm_lower, B.P.arm_upper, B.P.action_multiplier, B.P.frame_skip);
}

// thread = (collider slot of the person, env): distance from that collider to the nearest wiper collider,
// cut off at 5 m (`tool.get_closest_points(human, distance=5.0)`, bed_bathing.py:23)
AG_HDN inline void bathing_dist_body(int tid, const SimDev& S, const KP& p) {
  const int N = S.N;
  const BathDev& B = *(const BathDev*)p.p1;
  int e = tid % N, slot = tid / N;
  bool male = B.male[e] != 0;
  int c0 = male ? B.P.human_col0_m : B.P.human_col0_f, nc = male ? B.P.human_ncol_m : B.P.human_ncol_f;
  float best = 5.0f;
  if (slot < nc) {
    int ch = c0 + slot;
    int lt = AG_LDG(S.body_link0 + B.P.tool_body), nlt = AG_LDG(S.body_nlinks + B.P.tool_body);
    for (int l = lt; l < lt + nlt; l++) {
      int t0 = AG_LDG(S.link_col0 + l), tn = AG_LDG(S.link_ncol + l);
      for (int ct = t0; ct < t0 + tn; ct++) {
        NpOut c;
        int ca = ct < ch ? ct : ch, cb = ct < ch ? ch : ct;
        if (narrow_closest(S, e, ca, cb, 5.0f, c)) best = fminf(best, c.d);
      }
    }
  }
  B.dist_part[(size_t)slot * N + e] = best;
}

// thread = (target, env): update_targets (bed_bathing.py:190-203) from the current link poses, after the step's final k_fk
AG_HDN inline void bathing_track_body(int tid, const SimDev& S, const KP& p) {
  const int N = S.N;
  const BathDev& B = *(const BathDev*)p.p1;
  const int e = tid % N, t = tid / N;
  const int link = B.target_link[(size_t)t * N + e];
  if (link < 0) return;
  st3(B.targets, t, N, e, ld3(S.lpos, link, N, e) + qrot(ld4(S.lquat, link, N, e), ld3(B.target_local, t, N, e)));
}

// obs / reward / done.  p0 = action [N][7 + i0] (the reward's action term covers the whole raw row), p1 = BathDev*, p2 = obs [N][24],
// p3 = reward, p4 = done, p5 = info [N][4]
AG_HDN inline void bathing_post_body(int e, const SimDev& S, const KP& p) {
  const int N = S.N;
  const BathDev& B = *(const BathDev*)p.p1;
  const AgBathingParams& P = B.P;
  bool male = B.male[e] != 0;
  int hb = male ? P.human_body_m : P.human_body_f;
  Frame fr = body_frame(S, e, P.robot_body);
  // tool link 1 (the cloth) link-frame pose in the robot frame (bed_bathing.py:81-82)
  f3 tp = ld3(S.lpos, P.cloth_link, N, e); q4 tq = ld4(S.lquat, P.cloth_link, N, e);
  float* obs = (float*)p.p2 + (size_t)e * 24;
  int o = put3(obs, 0, to_frame(fr, tp)); o = put4(obs, o, to_frame(fr, tq));
  o = put_arm_angles(S, e, P.arm_links, obs, o);
  o = put_arm_points(S, e, fr, male ? P.arm_points_m : P.arm_points_f, obs, o);
  // forces and wiped targets (bed_bathing.py:41-78)
  float tool_force = 0.f, tool_on_human = 0.f, total_on_human = 0.f;
  int new_pts = 0;
  int cnt = n_contacts(S, e);
  const int T = P.n_targets_max;
  for (int s = 0; s < cnt; s++) {
    Contact c = contact_at(S, e, s);
    float force = contact_force(S, e, s);
    if (c.ba == P.tool_body || c.bb == P.tool_body) tool_force += force;
    int other, lo;
    if (!other_of(c, hb, other, lo)) continue;
    if (other == P.robot_body) total_on_human += force;
    else if (other == P.tool_body) {
      total_on_human += force;
      if (lo != P.cloth_link) continue;
      tool_on_human += force;
      f3 ph = contact_point_on(S, e, s, c, hb);
      for (int t = 0; t < T; t++) {
        if (!B.alive[(size_t)t * N + e]) continue;
        f3 tw = ld3(B.targets, t, N, e);
        if (norm(ph - tw) < 0.025f) { B.alive[(size_t)t * N + e] = 0; new_pts++; }
      }
    }
  }
  obs[o] = tool_force;
  int success = B.task_success[e] + new_pts;
  B.task_success[e] = success;
  float dmin = 5.0f;
  for (int i = 0; i < B.n_slots; i++) dmin = fminf(dmin, B.dist_part[(size_t)i * N + e]);
  // human preferences (env.py:237-274), task == 'bed_bathing'
  float pref = P.c_v * (-ee_speed(S, e, P.ee_link)) + P.c_f * (-(total_on_human - tool_on_human)) + P.c_hf * (tool_on_human < 10.f ? 0.f : -tool_on_human);
  float an = action_norm(S, e, B.action, (const float*)p.p0, p.i0);
  ((float*)p.p3)[e] = P.w_distance * (-dmin) + P.w_action * (-an) + P.w_wiping * (float)new_pts + pref;
  ((float*)p.p4)[e] = episode_done(B.iteration[e]);
  float* info = (float*)p.p5 + (size_t)e * 4;
  info[0] = total_on_human; info[1] = ((float)success >= (float)B.total_targets[e] * P.task_success_threshold) ? 1.f : 0.f;
  info[2] = tool_on_human; info[3] = (float)new_pts;
}
