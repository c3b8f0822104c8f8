"""Golden rollout of the reference's OWN co-optimisation ScratchItch step with a `tremor` person: `ScratchItchEnv.step` with a
controllable person (envs/scratch_itch.py:10-91), `AssistiveEnv.take_step` with the controllable tremor branch (env.py:205-215: the
person's action accumulates into target_joint_angles, the right arm is driven to target +- tremors), `Human.enforce_joint_limits` and
`Human.enforce_realistic_joint_limits` (agents/human.py:134-152) after every substep, executed on the CPU oracle through the pybullet
facade of make_golden_feeding_semantics.py, with the classifier evaluated as make_golden_scratch_coop_semantics.py does.  The person
raises the upper arm sideways until the classifier puts it back; the elbow is pushed into its limit, where the clamp zeroes that part
of the action.  Output: tests/golden/scratch_coop_tremor_semantics.npz, replayed by tests/test_coop_tremor.py on the per-call env
(oracle) and on the fused step (kernel bodies compiled for the host).

usage: python tests/golden/make_golden_scratch_coop_tremor_semantics.py [reference checkout]"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

N_STEPS, SEED = 16, 9


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    from assistive_gym_b200 import capi
    from assistive_gym_b200.limits_model import load_model
    from assistive_gym_b200.scratch_itch_batch import RIGHT_ARM_JOINTS, ScratchItchBatch
    from assistive_gym_b200.sim import BatchSim
    from oracle.oracle_py import OracleSim
    sb = ScratchItchBatch()
    cfg = capi.default_config()
    emu = capi.load_library(os.path.join(ROOT, 'tests', 'kernel_harness', 'libagphys_emu.so'))
    prod = BatchSim(sb.scene, cfg, 1, _lib=emu)
    rng = np.random.default_rng(SEED)
    smp = sb.sample(1, rng)
    smp['impairment'][:] = 0; smp['strength'] = np.ones(1); smp['limit_scale'] = np.ones(1)
    smp = sb.reset(prod, rng, sample=smp)                                # the reset needs the product's IK; its outcome is stored
    sim = OracleSim(sb.scene, cfg, 1)
    sb.reset(sim, np.random.default_rng(0), sample=smp)
    male = bool(smp['male'][0])
    hb = sb.humans['male' if male else 'female']
    from make_golden_env_logic import install_stubs
    from make_golden_feeding_semantics import Facade
    install_stubs(ref)
    import assistive_gym  # noqa: F401  (the reference package)
    from assistive_gym.envs.scratch_itch_envs import ScratchItchJacoHumanEnv
    env = ScratchItchJacoHumanEnv()
    p = sys.modules['pybullet']
    fac = Facade(sim, sb.scene, f32_targets=True)
    fac.install(p)

    def resetJointState(body, jointIndex=None, targetValue=0.0, targetVelocity=0.0, physicsClientId=None):
        sim.set_joint_state([fac.gl(body, jointIndex)], q=np.array([[float(targetValue)]]), qd=np.array([[float(targetVelocity)]]))
        sim.forward_kinematics()
    p.resetJointState = resetJointState
    env.robot.body, env.tool.body, env.human.body = sb.robot, sb.tool, hb
    env.human.gender = 'male' if male else 'female'
    for a in (env.robot, env.tool, env.human):
        a.id = 0
    sc = sb.scene
    env.robot.controllable_joint_lower_limits = np.array(sb.arm_lower, dtype=np.float64)
    env.robot.controllable_joint_upper_limits = np.array(sb.arm_upper, dtype=np.float64)
    h = env.human
    h.all_joint_indices = list(range(int(sc['body_nlinks'][hb]) - 1))
    h.lower_limits = {j: float(sc['link_lower'][fac.gl(hb, j)]) for j in h.all_joint_indices}
    h.upper_limits = {j: float(sc['link_upper'][fac.gl(hb, j)]) for j in h.all_joint_indices}
    h.controllable_joint_lower_limits = np.array([h.lower_limits[j] for j in RIGHT_ARM_JOINTS])
    h.controllable_joint_upper_limits = np.array([h.upper_limits[j] for j in RIGHT_ARM_JOINTS])
    tremors = np.random.default_rng(SEED + 2).uniform(np.deg2rad(-10), np.deg2rad(10), size=10).astype(np.float32).astype(np.float64)
    target0 = sb.coop_tremor_target(smp)[0].copy()                      # setup_joints' target_joint_angles (human.py:123)
    h.impairment, h.tremors, h.strength, h.target_joint_angles = 'tremor', tremors.copy(), 1.0, target0.copy()
    h.arm_previous_valid_pose = {True: None, False: None}
    model = load_model()
    restores = [0]

    def predict_classes(x):                          # count the restorations: an unreachable pose with a reachable one on record
        c = model.predict_classes(x)
        restores[0] += int(c.reshape(-1)[0] == 0 and h.arm_previous_valid_pose[True] is not None)
        return c
    h.limits_model = types.SimpleNamespace(predict_classes=predict_classes)
    env.agents = [env.robot, env.human]
    env.limb = int(smp['limb_joint'][0])
    env.target_on_arm = np.array(smp['target_local'][0], dtype=np.float64)
    env.target = types.SimpleNamespace(set_base_pos_orient=lambda *a, **k: None)
    env.prev_target_contact_pos = np.zeros(3)
    env.iteration, env.task_success, env.last_sim_time, env.gui = 0, 0, None, False
    env.action_space = types.SimpleNamespace(low=-np.ones(17), high=np.ones(17))
    env.action_robot_len, env.action_human_len = 7, 10
    env.update_targets()
    a_h = np.zeros(10); a_h[3] = 1.0; a_h[6] = -1.0                    # j_right_shoulder_x up, the elbow into its limit
    obs_r, obs_h, rew, arm, target, nrest = [], [], [], [], [], []
    for t in range(N_STEPS):
        o, r, d, info = env.step({'robot': np.zeros(7), 'human': a_h.copy()})
        obs_r.append(np.asarray(o['robot'], dtype=np.float64)); obs_h.append(np.asarray(o['human'], dtype=np.float64)); rew.append(float(r['robot']))
        arm.append(sim.get_joint_states([fac.gl(hb, j) for j in RIGHT_ARM_JOINTS])[0][0].copy())
        target.append(np.array(h.target_joint_angles, dtype=np.float64)); nrest.append(restores[0])
    arm = np.array(arm)
    out = {('sample_' + k): np.asarray(v) for k, v in smp.items()}
    out.update(human_action=a_h, obs_robot=np.array(obs_r), obs_human=np.array(obs_h), reward=np.array(rew), arm_q=arm,
               tremors=tremors, target0=target0, target_q=np.array(target), restores=np.array(nrest))
    np.savez_compressed(os.path.join(HERE, 'scratch_coop_tremor_semantics.npz'), **out)
    print('restorations after each step', nrest)
    print('target travel per step (rad)', np.round(np.abs(np.diff(np.vstack([target0, np.array(target)]), axis=0)).max(axis=1), 3))
    print('steps', N_STEPS, 'shoulder_x (deg) every 5 steps', np.round(np.rad2deg(arm[::5, 3]), 1), 'final', np.round(np.rad2deg(arm[-1, 3]), 1))


if __name__ == '__main__':
    main()
