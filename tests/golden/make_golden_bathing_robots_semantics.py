"""Golden rollout of the reference's OWN `BedBathingEnv.step` with PR2 (BedBathingPR2Env), on the CPU oracle through the pybullet
facade of make_golden_feeding_semantics.py (the wiring of make_golden_bathing_semantics.py, with PR2's reference class in place of
Sawyer's).

The start state: PR2's base pose comes from this repo's TOC reset (`BedBathingPR2Batch`) on the kernel bodies compiled for the host
(the oracle has no batched IK); the arm is then moved by IK so that the wiper hovers 5 mm above the person's right forearm, with its
motors aiming 5 cm lower (tests/test_bathing_robots.press_pad).  The oracle replays that placement and its state is stored.  The
reference's robot is given the joint limits its own `Agent.update_joint_limits` derives from the URDF (a joint reported as (0, -1) is
+-1e10).  The robot keeps pressing, so targets are wiped.

Output: tests/golden/bathing_pr2_semantics.npz, replayed by tests/test_bathing_robots_semantics.py.

usage: python tests/golden/make_golden_bathing_robots_semantics.py [/root/reference]   (needs tests/kernel_harness/libagphys_emu.so)"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

N_STEPS, N_COOP, SEED = 16, 35, 3
MOTOR_GAIN, MOTOR_FORCE = 0.1, 5.0            # the pressing arm of make_golden_bathing_semantics.py
PRESS_DEPTH = 0.15                            # the pressing pose, this far below the start pose: the actions close a fifth of the gap per step


def start(coop):
    """The TOC placement on the host-compiled kernels, then the oracle's own reset with that placement.  The single-agent start also
    takes the pressed-pad pose, from the first seed whose press wipes at least two targets with more than 3 N of cloth force on the
    fp32 kernels.  The co-optimisation start keeps the TOC start pose, with the pad clear of the arm, so that the person's arm is
    free to move."""
    from assistive_gym_b200 import capi
    from assistive_gym_b200.bed_bathing_robots_batch import BedBathingPR2Batch
    from assistive_gym_b200.sim import BatchSim
    from oracle.oracle_py import OracleSim
    from tests.test_bathing_robots import press_pad
    bb = BedBathingPR2Batch(controllable_person=coop)
    cfg = capi.default_config(residual_threshold=0.0)
    emu = BatchSim(bb.scene, cfg, 1, _lib=capi.load_library(os.path.join(ROOT, 'tests', 'kernel_harness', 'libagphys_emu.so')))
    q_lo = None
    for s in range(SEED, SEED + 60):
        smp = bb.sample(1, np.random.default_rng(s))
        if coop:
            smp['impairment'][:] = 0; smp['strength'] = np.ones(1); smp['limit_scale'] = np.ones(1)
        smp = bb.reset(emu, np.random.default_rng(s), sample=smp)
        if bb.unresolved or int(smp['goals_reached'][0]) < 1:
            continue
        if coop:
            break
        q_hi, q_lo, err = press_pad(bb, emu, smp, depth=PRESS_DEPTH)
        tw, alive = bb.targets_world(emu, smp)         # try the press on the fp32 kernels first
        wiped, force = 0, 0.0
        for _ in range(N_STEPS * 5):
            emu.step(1)
            _tf, on_human, _total, new = bb.total_force(emu, tw, alive)
            wiped += int(new[0]); force = max(force, float(on_human[0]))
        if err[0] < 1e-3 and wiped >= 2 and force > 3:
            smp['q7'] = q_hi
            break
    else:
        raise RuntimeError('no usable start pose')
    emu.close()
    sim = OracleSim(bb.scene, cfg, 1)
    bb.reset(sim, np.random.default_rng(0), sample=smp)
    if not coop:
        sim.set_motor(bb.arm_links, 1, target=q_lo, kp=[MOTOR_GAIN] * 7, kd=[1.0] * 7, max_force=[MOTOR_FORCE] * 7)
    return bb, sim, smp, q_lo, s


def human_actions():
    """The co-optimisation person's action per step: the elbow bent (j_right_elbow down), the upper arm raised (j_right_shoulder_x up)
    and turned (j_right_shoulder_z up), until the classifier objects to the raised, turned arm with the elbow bent."""
    a = np.zeros((N_COOP, 10))
    a[:, 3] = 1.0
    a[:, 5] = 1.0
    a[:, 6] = -1.0
    return a


def record(coop, ref_envs):
    from make_golden_feeding_robots_semantics import reference_limits
    from make_golden_feeding_semantics import Facade
    from assistive_gym_b200.bed_bathing_batch import RIGHT_ARM_JOINTS
    bb, sim, smp, q_lo, used_seed = start(coop)
    start_state = sim.state_get()
    env = (ref_envs.BedBathingPR2HumanEnv if coop else ref_envs.BedBathingPR2Env)()
    p = sys.modules['pybullet']
    fac = Facade(sim, bb.scene, f32_targets=True)           # motor targets reach the physics in fp32, as through `Agent.control`
    fac.install(p)
    male = bool(smp['male'][0])
    hb = bb.humans['male' if male else 'female']
    sc = bb.scene
    env.robot.body, env.tool.body, env.human.body = bb.robot, bb.tool, hb
    env.human.gender = 'male' if male else 'female'
    for a in (env.robot, env.tool, env.human):
        a.id = 0
    env.human.all_joint_indices = list(range(int(sc['body_nlinks'][hb]) - 1))
    env.robot.controllable_joint_lower_limits, env.robot.controllable_joint_upper_limits = reference_limits('pr2', env.robot.controllable_joint_indices)
    env.agents = [env.robot]
    k = 7
    restores = [0]
    if coop:
        from assistive_gym_b200.limits_model import load_model

        def resetJointState(body, jointIndex=None, targetValue=0.0, targetVelocity=0.0, physicsClientId=None):
            sim.set_joint_state([fac.gl(body, jointIndex)], q=np.array([[float(targetValue)]]), qd=np.array([[float(targetVelocity)]]))
            sim.forward_kinematics()
        p.resetJointState = resetJointState
        h = env.human
        h.lower_limits = {j: float(sc['link_lower'][fac.gl(hb, j)]) for j in h.all_joint_indices}
        h.upper_limits = {j: float(sc['link_upper'][fac.gl(hb, j)]) for j in h.all_joint_indices}
        h.controllable_joint_lower_limits = np.array([h.lower_limits[j] for j in RIGHT_ARM_JOINTS])
        h.controllable_joint_upper_limits = np.array([h.upper_limits[j] for j in RIGHT_ARM_JOINTS])
        h.impairment, h.tremors, h.strength = 'none', np.zeros(10), 1.0
        h.arm_previous_valid_pose = {True: None, False: None}
        model = load_model()

        def predict_classes(x):                 # counts the classifier's objections that send the arm back (human.py:150-152)
            c = model.predict_classes(x)
            if int(np.asarray(c).ravel()[0]) == 0 and h.arm_previous_valid_pose[True] is not None:
                restores[0] += 1
            return c
        h.limits_model = types.SimpleNamespace(predict_classes=predict_classes)
        env.agents.append(h)
        env.action_robot_len, env.action_human_len = 7, 10
        k = 17
    else:
        env.robot.motor_gains, env.robot.motor_forces = MOTOR_GAIN, MOTOR_FORCE
    env.iteration, env.task_success, env.last_sim_time, env.gui = 0, 0, None, False
    env.action_space = types.SimpleNamespace(low=-np.ones(k), high=np.ones(k))
    env.np_random = np.random.RandomState(0)
    if getattr(env, 'util', None) is None:
        from assistive_gym.envs.util import Util
        env.util = Util(0, env.np_random)
    env.create_spheres = lambda radius=0.01, mass=0.0, batch_positions=(), **kw: [types.SimpleNamespace(set_base_pos_orient=lambda *a, **kk: None) for _ in batch_positions]
    env.generate_targets()
    out = {('sample_' + key): np.asarray(v) for key, v in smp.items()}
    if coop:
        a_h = human_actions()
        obs_r, obs_h, rew, done, arm, n_restore = [], [], [], [], [], []
        for t in range(N_COOP):
            o, r, d, info = env.step({'robot': np.zeros(7), 'human': a_h[t].copy()})
            obs_r.append(np.asarray(o['robot'], dtype=np.float64)); obs_h.append(np.asarray(o['human'], dtype=np.float64))
            rew.append(float(r['robot'])); done.append(bool(d['__all__']))
            arm.append(sim.get_joint_states([fac.gl(hb, j) for j in RIGHT_ARM_JOINTS])[0][0].copy()); n_restore.append(restores[0])
        arm = np.array(arm)
        print('coop seed', used_seed, 'restores per step', n_restore, 'shoulder_x (deg) every 5 steps', np.round(np.rad2deg(arm[::5, 3]), 1),
              'elbow (deg)', np.round(np.rad2deg(arm[::5, 6]), 1))
        assert n_restore[-1] >= 1, 'the classifier never sent the arm back'
        out.update(human_actions=a_h, obs_robot=np.array(obs_r), obs_human=np.array(obs_h), reward=np.array(rew), done=np.array(done), arm_q=arm,
                   restores=np.array(n_restore))
        name = 'bathing_pr2_coop_semantics.npz'
    else:
        actions, obs, rew, done, total, on_human, new_pts, success = [], [], [], [], [], [], [], []
        for t in range(N_STEPS):
            q = sim.get_joint_states(bb.arm_links)[0]
            a = np.clip((q_lo - q) / 0.25, -1, 1)[0]                    # keep pressing (tests/test_bed_bathing._check_fused_wiping)
            o, r, d, info = env.step(a.copy())
            actions.append(a); obs.append(np.asarray(o, dtype=np.float64)); rew.append(float(r)); done.append(bool(d)); total.append(float(info['total_force_on_human']))
            on_human.append(float(env.tool_force_on_human)); new_pts.append(int(env.new_contact_points)); success.append(int(env.task_success))
        print('seed', used_seed, 'targets', env.total_target_count, 'wiped per step', new_pts, 'cloth force', np.round(on_human, 2), 'reward', np.round(rew, 2))
        assert sum(new_pts) >= 1 and max(on_human) > 3, 'the pad does not press'
        out.update(actions=np.array(actions), obs=np.array(obs), reward=np.array(rew), done=np.array(done), total_force=np.array(total),
                   tool_force_on_human=np.array(on_human), new_contact_points=np.array(new_pts), task_success=np.array(success),
                   total_target_count=np.array(env.total_target_count), q_press=q_lo, motor_gain=np.array(MOTOR_GAIN), motor_force=np.array(MOTOR_FORCE))
        name = 'bathing_pr2_semantics.npz'
    out.update(seed=np.array(used_seed), start_state=start_state,
               robot_lower=env.robot.controllable_joint_lower_limits, robot_upper=env.robot.controllable_joint_upper_limits)
    np.savez_compressed(os.path.join(HERE, name), **out)


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    from make_golden_env_logic import install_stubs
    install_stubs(ref)
    import assistive_gym  # noqa: F401  (the reference package)
    from assistive_gym.envs import bed_bathing_envs
    for coop in [c == 'coop' for c in sys.argv[2:]] or (False, True):
        record(coop, bed_bathing_envs)


if __name__ == '__main__':
    main()
