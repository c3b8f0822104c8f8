"""Golden rollouts of the reference's OWN `ScratchItchEnv.step` with Sawyer and with PR2, and of `ScratchItchSawyerHumanEnv.step` /
`ScratchItchPR2HumanEnv.step`, on the CPU oracle through the pybullet facade of make_golden_feeding_semantics.py (the same wiring as
make_golden_scratch_semantics.py and make_golden_scratch_coop_semantics.py, with the robot's reference class in place of Jaco).

The start state: the robot's base pose and start angles come from this repo's TOC reset (`ScratchItchSawyerBatch` /
`ScratchItchPR2Batch`) on the kernel bodies compiled for the host (the oracle has no batched IK).  For the single-agent rollouts the
arm is then moved by IK so that the scratcher's tip sits on the itch target, as in scratch_semantics.npz, so that scratches are counted.
The oracle replays that placement and its state is stored.  The reference's robot is given the joint limits its own
`Agent.update_joint_limits` derives from the URDF (agent.py:209-230: a joint reported as (0, -1) is +-1e10), so PR2's two continuous
arm joints go through the reference's unlimited action clamp.  In the co-optimisation rollouts the person raises the upper arm
sideways until the joint-limit classifier (the repo's evaluation of the reference's own weights) sends it back.

Output: tests/golden/scratch_{sawyer,pr2}_semantics.npz and scratch_{sawyer,pr2}_coop_semantics.npz, replayed by
tests/test_scratch_robots_semantics.py.

usage: python tests/golden/make_golden_scratch_robots_semantics.py [/root/reference]   (needs tests/kernel_harness/libagphys_emu.so)"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

N_STEPS, N_COOP = 16, 45
CASES = {'sawyer': ('ScratchItchSawyerEnv', 'ScratchItchSawyerBatch', 3, False), 'pr2': ('ScratchItchPR2Env', 'ScratchItchPR2Batch', 3, False),
         'sawyer_coop': ('ScratchItchSawyerHumanEnv', 'ScratchItchSawyerBatch', 7, True), 'pr2_coop': ('ScratchItchPR2HumanEnv', 'ScratchItchPR2Batch', 7, True)}


def start(batch_cls, seed, coop):
    """TOC placement on the host-compiled kernels (pressed onto the target for the single-agent rollouts), then the oracle's own
    reset with that placement."""
    from assistive_gym_b200 import capi
    from assistive_gym_b200.sim import BatchSim
    from oracle.oracle_py import OracleSim
    from tests.test_scratch_itch import _press_tip_on_target
    sb = batch_cls()
    cfg = capi.default_config(residual_threshold=0.0)
    emu = BatchSim(sb.scene, cfg, 1, _lib=capi.load_library(os.path.join(ROOT, 'tests', 'kernel_harness', 'libagphys_emu.so')))
    for s in range(seed, seed + 40):
        smp = sb.sample(1, np.random.default_rng(s))
        smp['impairment'][:] = 0; smp['strength'] = np.ones(1); smp['limit_scale'] = np.ones(1)
        smp = sb.reset(emu, np.random.default_rng(s), sample=smp)
        if sb.unresolved or int(smp['goals_reached'][0]) < 1:
            continue
        if coop:
            break
        q7, ok = _press_tip_on_target(sb, emu, smp)
        if ok[0]:
            smp['q7'] = q7
            break
    else:
        raise RuntimeError('no usable start pose')
    emu.close()
    sim = OracleSim(sb.scene, cfg, 1)
    sb.reset(sim, np.random.default_rng(0), sample=smp)
    return sb, sim, smp, s


sent_back = []                  # the classifier's verdicts during a co-optimisation step: 0 sends the arm back to its last valid pose


def wire(env, sb, sim, smp, coop):
    from make_golden_feeding_robots_semantics import reference_limits
    from make_golden_feeding_semantics import Facade
    from assistive_gym_b200.scratch_itch_batch import RIGHT_ARM_JOINTS
    p = sys.modules['pybullet']
    fac = Facade(sim, sb.scene, f32_targets=True)           # motor targets reach the physics in fp32, as through the repo's `Agent.control`
    fac.install(p)
    male = bool(smp['male'][0])
    hb = sb.humans['male' if male else 'female']
    env.robot.body, env.tool.body, env.human.body = sb.robot, sb.tool, hb
    env.human.gender = 'male' if male else 'female'
    for a in (env.robot, env.tool, env.human):
        a.id = 0
    lo, hi = reference_limits(sb.R['asset'], env.robot.controllable_joint_indices)
    env.robot.controllable_joint_lower_limits, env.robot.controllable_joint_upper_limits = lo, hi
    env.agents = [env.robot]
    k = 7
    if coop:
        from assistive_gym_b200.limits_model import load_model

        def resetJointState(body, jointIndex=None, targetValue=0.0, targetVelocity=0.0, physicsClientId=None):
            sim.set_joint_state([fac.gl(body, jointIndex)], q=np.array([[float(targetValue)]]), qd=np.array([[float(targetVelocity)]]))
            sim.forward_kinematics()
        p.resetJointState = resetJointState
        sc, h = sb.scene, env.human
        h.all_joint_indices = list(range(int(sc['body_nlinks'][hb]) - 1))
        h.lower_limits = {j: float(sc['link_lower'][fac.gl(hb, j)]) for j in h.all_joint_indices}
        h.upper_limits = {j: float(sc['link_upper'][fac.gl(hb, j)]) for j in h.all_joint_indices}
        h.controllable_joint_lower_limits = np.array([h.lower_limits[j] for j in RIGHT_ARM_JOINTS])
        h.controllable_joint_upper_limits = np.array([h.upper_limits[j] for j in RIGHT_ARM_JOINTS])
        h.impairment, h.tremors, h.strength = 'none', np.zeros(10), 1.0
        h.arm_previous_valid_pose = {True: None, False: None}
        model = load_model()

        def predict_classes(x):
            r = model.predict_classes(x)
            sent_back.append(int(np.asarray(r).ravel()[0]) == 0)
            return r
        h.limits_model = types.SimpleNamespace(predict_classes=predict_classes)
        env.agents.append(h)
        env.action_robot_len, env.action_human_len = 7, 10
        k = 17
    env.limb = int(smp['limb_joint'][0])
    env.target_on_arm = np.array(smp['target_local'][0], dtype=np.float64)
    env.target = types.SimpleNamespace(set_base_pos_orient=lambda *a, **k: None)
    env.prev_target_contact_pos = np.zeros(3)
    env.iteration, env.task_success, env.last_sim_time, env.gui = 0, 0, None, False
    env.action_space = types.SimpleNamespace(low=-np.ones(k), high=np.ones(k))
    env.update_targets()
    return fac, hb


def record(key, ref_envs):
    import assistive_gym_b200.scratch_itch_robots_batch as srb
    from assistive_gym_b200.scratch_itch_batch import RIGHT_ARM_JOINTS
    env_name, batch_name, seed, coop = CASES[key]
    sb, sim, smp, used_seed = start(getattr(srb, batch_name), seed, coop)
    env = getattr(ref_envs, env_name)()
    fac, hb = wire(env, sb, sim, smp, coop)
    start_state = sim.state_get()
    out = {('sample_' + k): np.asarray(v) for k, v in smp.items()}
    if coop:
        a_h = np.zeros(10); a_h[3] = 1.0                                # j_right_shoulder_x up
        obs_r, obs_h, rew, arm, back = [], [], [], [], []
        for t in range(N_COOP):
            del sent_back[:]
            o, r, d, info = env.step({'robot': np.zeros(7), 'human': a_h.copy()})
            back.append(any(sent_back))
            obs_r.append(np.asarray(o['robot'], dtype=np.float64)); obs_h.append(np.asarray(o['human'], dtype=np.float64)); rew.append(float(r['robot']))
            arm.append(sim.get_joint_states([fac.gl(hb, j) for j in RIGHT_ARM_JOINTS])[0][0].copy())
        arm = np.array(arm)
        out.update(human_action=a_h, obs_robot=np.array(obs_r), obs_human=np.array(obs_h), reward=np.array(rew), arm_q=arm, sent_back=np.array(back))
        print(key, 'seed', used_seed, 'steps with the arm sent back', np.flatnonzero(back), 'shoulder_x (deg) every 5 steps', np.round(np.rad2deg(arm[::5, 3]), 1), 'max', np.round(np.rad2deg(arm[:, 3].max()), 1),
              'final', np.round(np.rad2deg(arm[-1, 3]), 1))
    else:
        arng = np.random.default_rng(used_seed + 1)
        actions = np.concatenate([np.zeros((4, 7)), arng.uniform(-1, 1, size=(N_STEPS - 4, 7)) * 0.15])      # hold the press, then wiggle
        obs, rew, done, total, at_target, success = [], [], [], [], [], []
        for t in range(N_STEPS):
            o, r, d, info = env.step(actions[t].copy())
            obs.append(np.asarray(o, dtype=np.float64)); rew.append(float(r)); done.append(bool(d)); total.append(float(info['total_force_on_human']))
            at_target.append(float(env.tool_force_at_target)); success.append(int(env.task_success))
        out.update(actions=actions, obs=np.array(obs), reward=np.array(rew), done=np.array(done), total_force=np.array(total), force_at_target=np.array(at_target),
                   task_success=np.array(success))
        print(key, 'seed', used_seed, 'scratches counted', success[-1], 'force at target', np.round(at_target, 2), 'reward', np.round(rew, 2))
    out['seed'] = np.array(used_seed)
    out['robot_lower'], out['robot_upper'] = env.robot.controllable_joint_lower_limits, env.robot.controllable_joint_upper_limits
    out['start_state'] = start_state
    np.savez_compressed(os.path.join(HERE, 'scratch_%s_semantics.npz' % key), **out)


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    from make_golden_env_logic import install_stubs
    install_stubs(ref)
    import assistive_gym  # noqa: F401  (the reference package)
    from assistive_gym.envs import scratch_itch_envs
    for key in (sys.argv[2:] or CASES):
        record(key, scratch_itch_envs)


if __name__ == '__main__':
    main()
