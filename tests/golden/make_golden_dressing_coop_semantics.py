"""Golden rollout of the reference's OWN co-optimisation step of Dressing: `DressingEnv.step` with a controllable person
(envs/dressing.py:12-106 with dict actions / observations, `update_targets` :199-210; `AssistiveEnv.take_step` driving the person's
left arm; `Human.enforce_joint_limits` and `Human.enforce_realistic_joint_limits` -- agents/human.py:134-152 -- after every
stepSimulation; util.sleeve_on_arm_reward; all unmodified), executed on the CPU oracle (rigid bodies + cloth) through the pybullet
facade of make_golden_feeding_semantics.py, extended by `getSoftBodyData` as in make_golden_dressing_semantics.py.  The Keras
classifier is replaced by the repo's evaluation of the SAME weights (`assistive_gym_b200/limits_model.py`).

The start state is the repo's co-optimisation reset (`DressingBatch(controllable_person=True)`: the arm held with gain 0.05 and
force 1 while the gown settles; the robot base-pose search with the product's IK, host-compiled kernel bodies, is stored in the
sample).  The robot makes small random moves with the gown; the person lifts the left arm sideways (shoulder y) inside the gown
until the joint reaches its limit and the joint-limit classifier sends the arm back.  Output:
tests/golden/dressing_coop_semantics.npz, replayed by tests/test_reference_dressing_coop_semantics.py (per-call step on the oracle)
and tests/test_dressing_coop.py (kernel bodies).

usage: python tests/golden/make_golden_dressing_coop_semantics.py [/root/reference]"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

N_STEPS, SEED = 16, 0
SETTLE = 3                                      # a short settle at half gravity (dressing.py:178-193), as in make_golden_dressing_semantics.py


def actions():
    """[N_STEPS, 17]: the robot's small random moves, then the person's shoulder y at full action"""
    a = np.zeros((N_STEPS, 17))
    a[:, :7] = np.random.default_rng(SEED + 1).uniform(-0.5, 0.5, size=(N_STEPS, 7))
    a[:, 7 + 4] = 1.0
    return a


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    from assistive_gym_b200 import capi
    from assistive_gym_b200.dressing_batch import LEFT_ARM_JOINTS, RADII, DressingBatch
    from assistive_gym_b200.limits_model import load_model
    from assistive_gym_b200.sim import BatchSim
    from oracle.oracle_py import OracleSim
    db = DressingBatch(controllable_person=True)
    cfg = DressingBatch.config()
    emu = capi.load_library(os.path.join(ROOT, 'tests', 'kernel_harness', 'libagphys_emu.so'))
    prod = BatchSim(db.scene, cfg, 1, _lib=emu)
    rng = np.random.default_rng(SEED)
    smp = db.sample(1, rng)
    smp['impairment'][:] = 0; smp['strength'] = np.ones(1); smp['tremors'] = np.zeros((1, 10)); smp['limit_scale'] = np.ones(1)
    smp = db.reset(prod, rng, sample=smp, attempts=12, settle_steps=0)
    assert db.unresolved == 0
    prod.close()
    sim = OracleSim(db.scene, cfg, 1)
    db.reset(sim, np.random.default_rng(SEED), sample=smp, settle_steps=0)
    sim.cloth_set_gravity([0, 0, -9.81 / 2]); sim.step(SETTLE); sim.cloth_set_gravity([0, 0, -9.81])
    male = bool(smp['male'][0])
    hb = db.humans['male' if male else 'female']
    from make_golden_env_logic import install_stubs
    from make_golden_feeding_semantics import Facade
    install_stubs(ref)
    import assistive_gym  # noqa: F401  (the reference package)
    from assistive_gym.envs.dressing_envs import DressingPR2HumanEnv
    from assistive_gym.envs.util import Util
    env = DressingPR2HumanEnv()
    p = sys.modules['pybullet']
    fac = Facade(sim, db.scene, f32_targets=True)
    fac.install(p)

    def resetJointState(body, jointIndex=None, targetValue=0.0, targetVelocity=0.0, physicsClientId=None):
        sim.set_joint_state([fac.gl(body, jointIndex)], q=np.array([[float(targetValue)]]), qd=np.array([[float(targetVelocity)]]))
        sim.forward_kinematics()
    p.resetJointState = resetJointState

    def getSoftBodyData(cloth, physicsClientId=None):
        x, _ = sim.cloth_get_state()
        cnt, node, cpos, force, link = sim.cloth_get_contacts(2048)
        k = int(cnt[0])
        return (x[0, :, 0], x[0, :, 1], x[0, :, 2], cpos[0, :k, 0], cpos[0, :k, 1], cpos[0, :k, 2], force[0, :k, 0], force[0, :k, 1], force[0, :k, 2])
    p.getSoftBodyData = getSoftBodyData
    env.robot.body, env.human.body = db.robot, hb
    env.human.gender = 'male' if male else 'female'
    env.human.hand_radius, env.human.elbow_radius, env.human.shoulder_radius = RADII['male' if male else 'female']
    for a in (env.robot, env.human):
        a.id = 0
    sc = db.scene
    env.robot.controllable_joint_lower_limits = np.array(db.arm_lower, dtype=np.float64)
    env.robot.controllable_joint_upper_limits = np.array(db.arm_upper, dtype=np.float64)
    env.robot.motor_gains = env.human.motor_gains = 0.01                 # dressing.py:121
    h = env.human
    h.all_joint_indices = list(range(int(sc['body_nlinks'][hb]) - 1))
    h.lower_limits = {j: float(sc['link_lower'][fac.gl(hb, j)]) for j in h.all_joint_indices}
    h.upper_limits = {j: float(sc['link_upper'][fac.gl(hb, j)]) for j in h.all_joint_indices}
    h.controllable_joint_lower_limits = np.array([h.lower_limits[j] for j in LEFT_ARM_JOINTS])
    h.controllable_joint_upper_limits = np.array([h.upper_limits[j] for j in LEFT_ARM_JOINTS])
    h.impairment, h.tremors, h.strength = 'none', np.zeros(10), 1.0
    h.arm_previous_valid_pose = {True: None, False: None}
    model = load_model()
    restores = [0]

    def predict_classes(x):                     # counts the classifier's objections that send the arm back (human.py:150-152)
        c = model.predict_classes(x)
        if int(c[0, 0]) == 0 and h.arm_previous_valid_pose[False] is not None:
            restores[0] += 1
        return c
    h.limits_model = types.SimpleNamespace(predict_classes=predict_classes)
    env.agents = [env.robot, env.human]
    env.cloth = 0
    env.cloth_attachment = types.SimpleNamespace(set_base_pos_orient=lambda pos, orient: sim.cloth_set_anchor(np.asarray(pos, dtype=np.float64)[None]))
    env.triangle1_point_indices, env.triangle2_point_indices = [1180, 2819, 30], [1322, 13, 696]      # dressing.py:156-157
    env.iteration, env.task_success, env.last_sim_time, env.gui = 0, 0, None, False
    env.action_space = types.SimpleNamespace(low=-np.ones(17), high=np.ones(17))
    env.action_robot_len, env.action_human_len = 7, 10
    env.np_random = np.random.RandomState(0)
    if getattr(env, 'util', None) is None:
        env.util = Util(0, env.np_random)
    acts = actions()
    links = [fac.gl(hb, j) for j in LEFT_ARM_JOINTS]
    lo, hi = np.array([h.lower_limits[j] for j in LEFT_ARM_JOINTS]), np.array([h.upper_limits[j] for j in LEFT_ARM_JOINTS])
    obs_r, obs_h, rew, done, total, success, sleeve, arm_q, n_restore, at_limit = [], [], [], [], [], [], [], [], [], []
    for t in range(N_STEPS):
        o, r, d, info = env.step({'robot': acts[t, :7].copy(), 'human': acts[t, 7:].copy()})
        obs_r.append(np.asarray(o['robot'], dtype=np.float64)); obs_h.append(np.asarray(o['human'], dtype=np.float64))
        rew.append(float(r['robot'])); done.append(bool(d['__all__'])); total.append(float(info['robot']['total_force_on_human']))
        success.append(float(env.task_success)); sleeve.append(int(bool(env.forearm_in_sleeve)) + 2 * int(bool(env.upperarm_in_sleeve)))
        q = sim.get_joint_states(links)[0][0].copy()
        arm_q.append(q); n_restore.append(restores[0]); at_limit.append(bool(np.any(np.isclose(q, lo, atol=1e-6, rtol=0) | np.isclose(q, hi, atol=1e-6, rtol=0))))
    print('steps', N_STEPS, 'reward', np.round(rew, 3), 'cloth force sum', np.round([o_[23] for o_ in obs_r], 2), 'robot force', np.round([o_[27] for o_ in obs_h], 2),
          'sleeve state', sleeve, 'restores', n_restore, 'at limit', at_limit)
    assert n_restore[-1] >= 1, 'the classifier never sent the arm back'
    assert any(at_limit), 'no joint reached its limit'
    out = {('sample_' + k): np.asarray(v) for k, v in smp.items()}
    out.update(actions=acts, obs_robot=np.array(obs_r), obs_human=np.array(obs_h), reward=np.array(rew), done=np.array(done),
               total_force=np.array(total), task_success=np.array(success), sleeve=np.array(sleeve), arm_q=np.array(arm_q),
               restores=np.array(n_restore), at_limit=np.array(at_limit))
    np.savez_compressed(os.path.join(HERE, 'dressing_coop_semantics.npz'), **out)


if __name__ == '__main__':
    main()
