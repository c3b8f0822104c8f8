"""Golden rollout of the reference's OWN co-optimisation step of BedBathing: `BedBathingEnv.step` with a controllable person
(envs/bed_bathing.py:12-111 with dict actions / observations, `generate_targets` / `update_targets` :173-203; `AssistiveEnv.take_step`
driving the person's right arm; `Human.enforce_joint_limits` and `Human.enforce_realistic_joint_limits` -- agents/human.py:134-152 --
and `update_targets` after every substep), executed on the CPU oracle through the pybullet facade of make_golden_feeding_semantics.py.
The Keras classifier is replaced by the repo's evaluation of the SAME weights (`assistive_gym_b200/limits_model.py`).

The start state is the repo's co-optimisation reset (`BedBathingBatch(controllable_person=True)`) with the wiper pad pressed onto
the forearm (tests/test_bed_bathing._pressed_pair).  The robot keeps pressing; the person first rolls the forearm under the pad, so
that targets that started away from the pad are wiped where the arm has carried them; then the robot lifts the pad and the
person turns the upper arm until the joint-limit classifier sends it back.  Output: tests/golden/bathing_coop_semantics.npz, replayed by
tests/test_reference_bathing_coop_semantics.py (per-call step on the oracle) and tests/test_bathing_coop.py (kernel bodies).

usage: python tests/golden/make_golden_bathing_coop_semantics.py [/root/reference]"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

SEED = 8
N_ROLL, N_RAISE = 12, 32                       # steps of each phase of the person's action


def human_actions():
    """The person's action per step: the forearm roll (j_right_forearm) first; then, with the pad lifted, the upper arm turns
    (j_right_shoulder_z up, the elbow bent for the first eight steps) until the classifier stops it at about 81 degrees."""
    a = np.zeros((N_ROLL + N_RAISE, 10))
    a[:N_ROLL, 7] = 1.0
    a[N_ROLL:, 5] = 1.0
    a[N_ROLL:N_ROLL + 8, 6] = -1.0
    return a


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    from assistive_gym_b200.bed_bathing_batch import RIGHT_ARM_JOINTS, SAWYER, BedBathingBatch
    from assistive_gym_b200.limits_model import load_model
    from oracle.oracle_py import OracleSim
    from tests.test_bed_bathing import _pressed_pair
    bb = BedBathingBatch(controllable_person=True)
    sim, _other, smp, ik = _pressed_pair(bb, lambda sc, cfg, n: OracleSim(sc, cfg, n), 1, seed=SEED)
    smp['impairment'][:] = 0; smp['limit_scale'] = np.ones(1); smp['strength'] = np.ones(1)
    start_state = sim.state_get()
    q_hi = sim.get_joint_states(bb.arm_links)[0]                         # the start pose, 5 mm above the skin
    male = bool(smp['male'][0])
    hb = bb.humans['male' if male else 'female']
    arm = np.array(SAWYER['arm']) + 1
    q_lo = ik[2][:, arm]
    from make_golden_env_logic import install_stubs
    from make_golden_feeding_semantics import Facade
    install_stubs(ref)
    import assistive_gym  # noqa: F401  (the reference package)
    from assistive_gym.envs.bed_bathing_envs import BedBathingSawyerHumanEnv
    env = BedBathingSawyerHumanEnv()
    p = sys.modules['pybullet']
    fac = Facade(sim, bb.scene, f32_targets=True)
    fac.install(p)

    def resetJointState(body, jointIndex=None, targetValue=0.0, targetVelocity=0.0, physicsClientId=None):
        sim.set_joint_state([fac.gl(body, jointIndex)], q=np.array([[float(targetValue)]]), qd=np.array([[float(targetVelocity)]]))
        sim.forward_kinematics()
    p.resetJointState = resetJointState
    env.robot.body, env.tool.body, env.human.body = bb.robot, bb.tool, hb
    env.human.gender = 'male' if male else 'female'
    for a in (env.robot, env.tool, env.human):
        a.id = 0
    sc = bb.scene
    env.robot.controllable_joint_lower_limits = np.array(bb.arm_lower, dtype=np.float64)
    env.robot.controllable_joint_upper_limits = np.array(bb.arm_upper, dtype=np.float64)
    env.robot.motor_gains, env.robot.motor_forces = 0.1, 5.0             # the pressing arm of make_golden_bathing_semantics.py
    h = env.human
    h.all_joint_indices = list(range(int(sc['body_nlinks'][hb]) - 1))
    h.lower_limits = {j: float(sc['link_lower'][fac.gl(hb, j)]) for j in h.all_joint_indices}
    h.upper_limits = {j: float(sc['link_upper'][fac.gl(hb, j)]) for j in h.all_joint_indices}
    h.controllable_joint_lower_limits = np.array([h.lower_limits[j] for j in RIGHT_ARM_JOINTS])
    h.controllable_joint_upper_limits = np.array([h.upper_limits[j] for j in RIGHT_ARM_JOINTS])
    h.impairment, h.tremors, h.strength = 'none', np.zeros(10), 1.0
    h.arm_previous_valid_pose = {True: None, False: None}
    model = load_model()
    restores = [0]

    def predict_classes(x):                     # counts the classifier's objections that send the arm back (human.py:150-152)
        c = model.predict_classes(x)
        if int(c[0, 0]) == 0 and h.arm_previous_valid_pose[True] is not None:
            restores[0] += 1
        return c
    h.limits_model = types.SimpleNamespace(predict_classes=predict_classes)
    env.agents = [env.robot, env.human]
    env.iteration, env.task_success, env.last_sim_time, env.gui = 0, 0, None, False
    env.action_space = types.SimpleNamespace(low=-np.ones(17), high=np.ones(17))
    env.action_robot_len, env.action_human_len = 7, 10
    env.np_random = np.random.RandomState(0)
    if getattr(env, 'util', None) is None:
        from assistive_gym.envs.util import Util
        env.util = Util(0, env.np_random)
    history = []                                # every position the reference gives each target marker

    def create_spheres(radius=0.01, mass=0.0, batch_positions=(), **k):
        out = []
        for _ in batch_positions:
            rec = []
            history.append(rec)
            out.append(types.SimpleNamespace(set_base_pos_orient=lambda pos, orient, rec=rec: rec.append(np.array(pos, dtype=np.float64))))
        return out
    env.create_spheres = create_spheres
    env.generate_targets()
    reset_pos = np.array([r[0] for r in history])
    a_h = human_actions()
    actions, obs_r, obs_h, rew, done, total, on_human, new_pts, success, arm_q, n_restore = [], [], [], [], [], [], [], [], [], [], []
    wiped = []                                  # (step, target, world position at the wipe)
    for t in range(len(a_h)):
        q = sim.get_joint_states(bb.arm_links)[0]
        q_goal = q_lo if t < N_ROLL else q_hi                            # press (make_golden_bathing_semantics.py), then lift the pad
        a = np.clip((q_goal - q) / 0.25, -1, 1)[0]
        n_hist = [len(r) for r in history]
        o, r, d, info = env.step({'robot': a.copy(), 'human': a_h[t].copy()})
        for i, rec in enumerate(history):
            if len(rec) > n_hist[i] and rec[-1][0] >= 1000:              # sent away: wiped at its previous position (bed_bathing.py:60,72)
                wiped.append((t, i, rec[-2]))
        actions.append(np.concatenate([a, a_h[t]])); obs_r.append(np.asarray(o['robot'], dtype=np.float64)); obs_h.append(np.asarray(o['human'], dtype=np.float64))
        rew.append(float(r['robot'])); done.append(bool(d['__all__'])); total.append(float(info['robot']['total_force_on_human']))
        on_human.append(float(env.tool_force_on_human)); new_pts.append(int(env.new_contact_points)); success.append(int(env.task_success))
        arm_q.append(sim.get_joint_states([fac.gl(hb, j) for j in RIGHT_ARM_JOINTS])[0][0].copy()); n_restore.append(restores[0])
    moved = np.array([np.linalg.norm(w - reset_pos[i]) for _, i, w in wiped])
    print('steps', len(a_h), 'targets', env.total_target_count, 'wiped per step', new_pts, 'moved (cm)', np.round(100 * moved, 1),
          'restores', n_restore[-1], 'cloth force', np.round(on_human, 2))
    assert int((moved >= 0.01).sum()) >= 3, 'fewer than 3 targets wiped away from their reset positions'
    assert n_restore[-1] >= 1, 'the classifier never sent the arm back'
    out = {('sample_' + k): np.asarray(v) for k, v in smp.items()}
    out.update(start_state=start_state, q_press=q_lo, actions=np.array(actions), obs_robot=np.array(obs_r), obs_human=np.array(obs_h), reward=np.array(rew),
               done=np.array(done), total_force=np.array(total), tool_force_on_human=np.array(on_human), new_contact_points=np.array(new_pts),
               task_success=np.array(success), total_target_count=np.array(env.total_target_count), arm_q=np.array(arm_q), restores=np.array(n_restore),
               targets_reset=reset_pos, wiped_step=np.array([w[0] for w in wiped]), wiped_target=np.array([w[1] for w in wiped]),
               wiped_pos=np.array([w[2] for w in wiped]).reshape(-1, 3), motor_gain=np.array(0.1), motor_force=np.array(5.0))
    np.savez_compressed(os.path.join(HERE, 'bathing_coop_semantics.npz'), **out)


if __name__ == '__main__':
    main()
