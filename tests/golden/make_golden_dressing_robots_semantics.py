"""Golden rollouts of the reference's OWN `DressingEnv.step` (envs/dressing.py:12-106, `update_targets` :199-210, env.py:174-274 and
util.sleeve_on_arm_reward, all unmodified) with Sawyer and with Jaco, and of its co-optimisation step with Sawyer, on the CPU oracle
(rigid bodies + cloth) through the pybullet facade of make_golden_dressing_semantics.py / make_golden_dressing_coop_semantics.py (the
same wiring, with the robot's reference class in place of PR2).

The start state: the robot's placement comes from this repo's reset (`DressingSawyerBatch`: the TOC search; `DressingJacoBatch`: the
mounted arm's IK) on the kernel bodies compiled for the host (the oracle has no batched IK); the oracle then replays that placement
and runs a short settle at half gravity, as the PR2 goldens do.  The reference's robot is given the joint limits its own
`Agent.update_joint_limits` derives from the URDF (+-1e10 for Jaco's continuous joints).  In the co-optimisation rollout the person
lifts the left arm sideways (shoulder y) inside the gown until the joint-limit classifier sends the arm back.

Output: tests/golden/dressing_sawyer_semantics.npz, dressing_jaco_semantics.npz and dressing_sawyer_coop_semantics.npz, replayed by
tests/test_dressing_robots_semantics.py.

usage: python tests/golden/make_golden_dressing_robots_semantics.py [/root/reference]   (needs tests/kernel_harness/libagphys_emu.so)"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_feeding_robots_semantics import reference_limits  # noqa: E402

N_STEPS, N_STEPS_COOP, SETTLE = 8, 16, 3
# key: (reference env class, batch class, asset, seed of the placement)
CASES = {'sawyer': ('DressingSawyerEnv', 'DressingSawyerBatch', 'sawyer', 1), 'jaco': ('DressingJacoEnv', 'DressingJacoBatch', 'jaco', 1),
         'sawyer_coop': ('DressingSawyerHumanEnv', 'DressingSawyerBatch', 'sawyer', 1)}


def coop_actions():
    """[N_STEPS_COOP, 17]: the robot's small random moves, then the person's shoulder y at full action"""
    a = np.zeros((N_STEPS_COOP, 17))
    a[:, :7] = np.random.default_rng(2).uniform(-0.5, 0.5, size=(N_STEPS_COOP, 7))
    a[:, 7 + 4] = 1.0
    return a


def start(batch_cls, seed, coop):
    """The placement on the host-compiled kernels (no impairment, no colliding env), then the oracle's own reset of it and the
    short settle; returns the batch, the oracle and the sample."""
    from assistive_gym_b200 import capi
    from assistive_gym_b200.sim import BatchSim
    from oracle.oracle_py import OracleSim
    db = batch_cls(controllable_person=coop)
    emu = BatchSim(db.scene, db.config(), 1, _lib=capi.load_library(os.path.join(ROOT, 'tests', 'kernel_harness', 'libagphys_emu.so')))
    rng = np.random.default_rng(seed)
    smp = db.sample(1, rng)
    smp['impairment'][:] = 0; smp['strength'] = np.ones(1); smp['tremors'] = np.zeros((1, 10))
    if coop:
        smp['limit_scale'] = np.ones(1)
    smp = db.reset(emu, rng, sample=smp, attempts=12, settle_steps=0)
    assert db.unresolved == 0 and int(smp['goals_reached'][0]) >= 1
    emu.close()
    sim = OracleSim(db.scene, db.config(), 1)
    db.reset(sim, np.random.default_rng(0), sample=smp, settle_steps=0)
    sim.cloth_set_gravity([0, 0, -9.81 / 2]); sim.step(SETTLE); sim.cloth_set_gravity([0, 0, -9.81])
    return db, sim, smp


def rollout(ref, key):
    env_name, batch_name, asset, seed = CASES[key]
    coop = key.endswith('_coop')
    from assistive_gym_b200 import dressing_robots_batch
    from assistive_gym_b200.dressing_batch import LEFT_ARM_JOINTS, RADII
    from assistive_gym_b200.limits_model import load_model
    db, sim, smp = start(getattr(dressing_robots_batch, batch_name), seed, coop)
    male = bool(smp['male'][0])
    hb = db.humans['male' if male else 'female']
    for k in [k for k in sys.modules if k.startswith('assistive_gym.') or k == 'assistive_gym']:
        del sys.modules[k]
    from make_golden_env_logic import install_stubs
    from make_golden_feeding_semantics import Facade
    install_stubs(ref)
    import importlib
    dressing_envs = importlib.import_module('assistive_gym.envs.dressing_envs')
    from assistive_gym.envs.util import Util
    env = getattr(dressing_envs, env_name)()
    p = sys.modules['pybullet']
    fac = Facade(sim, db.scene, f32_targets=True)            # float32 motor targets, as the per-call env and the fused step set them
    fac.install(p)
    if coop:
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
    lo, hi = reference_limits(asset, db.R['arm'])
    env.robot.controllable_joint_lower_limits, env.robot.controllable_joint_upper_limits = lo, hi
    env.robot.motor_gains = env.human.motor_gains = 0.01                 # dressing.py:121
    env.cloth = 0
    env.cloth_attachment = types.SimpleNamespace(set_base_pos_orient=lambda pos, orient: sim.cloth_set_anchor(np.asarray(pos, dtype=np.float64)[None]))
    env.triangle1_point_indices, env.triangle2_point_indices = [1180, 2819, 30], [1322, 13, 696]      # dressing.py:156-157
    env.iteration, env.task_success, env.last_sim_time, env.gui = 0, 0, None, False
    env.np_random = np.random.RandomState(0)
    if getattr(env, 'util', None) is None:
        env.util = Util(0, env.np_random)
    out = {('sample_' + k): np.asarray(v) for k, v in smp.items()}
    if not coop:
        env.agents = [env.robot]
        env.action_space = types.SimpleNamespace(low=-np.ones(7), high=np.ones(7))
        actions = np.random.default_rng(seed + 1).uniform(-1, 1, size=(N_STEPS, 7))
        obs, rew, done, total, success, sleeve = [], [], [], [], [], []
        for t in range(N_STEPS):
            o, r, d, info = env.step(actions[t].copy())
            obs.append(np.asarray(o, dtype=np.float64)); rew.append(float(r)); done.append(bool(d)); total.append(float(info['total_force_on_human']))
            success.append(float(env.task_success)); sleeve.append(int(bool(env.forearm_in_sleeve)) + 2 * int(bool(env.upperarm_in_sleeve)))
        print(key, 'reward', np.round(rew, 3), 'cloth force sum', np.round([o_[23] for o_ in obs], 2), 'sleeve state', sleeve)
        assert max(o_[23] for o_ in obs) > 0, 'the gown never pressed on the person'
        out.update(actions=actions, obs=np.array(obs), reward=np.array(rew), done=np.array(done), total_force=np.array(total),
                   task_success=np.array(success), sleeve=np.array(sleeve))
        return out
    sc = db.scene
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
    env.action_space = types.SimpleNamespace(low=-np.ones(17), high=np.ones(17))
    env.action_robot_len, env.action_human_len = 7, 10
    acts = coop_actions()
    links = [fac.gl(hb, j) for j in LEFT_ARM_JOINTS]
    alo, ahi = h.controllable_joint_lower_limits, h.controllable_joint_upper_limits
    obs_r, obs_h, rew, done, total, success, sleeve, arm_q, n_restore, at_limit = [], [], [], [], [], [], [], [], [], []
    for t in range(N_STEPS_COOP):
        o, r, d, info = env.step({'robot': acts[t, :7].copy(), 'human': acts[t, 7:].copy()})
        obs_r.append(np.asarray(o['robot'], dtype=np.float64)); obs_h.append(np.asarray(o['human'], dtype=np.float64))
        rew.append(float(r['robot'])); done.append(bool(d['__all__'])); total.append(float(info['robot']['total_force_on_human']))
        success.append(float(env.task_success)); sleeve.append(int(bool(env.forearm_in_sleeve)) + 2 * int(bool(env.upperarm_in_sleeve)))
        q = sim.get_joint_states(links)[0][0].copy()
        arm_q.append(q); n_restore.append(restores[0]); at_limit.append(bool(np.any(np.isclose(q, alo, atol=1e-6, rtol=0) | np.isclose(q, ahi, atol=1e-6, rtol=0))))
    print(key, 'reward', np.round(rew, 3), 'cloth force sum', np.round([o_[23] for o_ in obs_r], 2), 'sleeve state', sleeve, 'restores', n_restore)
    assert max(o_[23] for o_ in obs_r) > 0, 'the gown never pressed on the person'
    assert n_restore[-1] >= 1, 'the classifier never sent the arm back'
    out.update(actions=acts, obs_robot=np.array(obs_r), obs_human=np.array(obs_h), reward=np.array(rew), done=np.array(done),
               total_force=np.array(total), task_success=np.array(success), sleeve=np.array(sleeve), arm_q=np.array(arm_q),
               restores=np.array(n_restore), at_limit=np.array(at_limit))
    return out


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    keys = sys.argv[2].split(',') if len(sys.argv) > 2 else list(CASES)
    for key in keys:
        np.savez_compressed(os.path.join(HERE, 'dressing_%s_semantics.npz' % key), **rollout(ref, key))


if __name__ == '__main__':
    main()
