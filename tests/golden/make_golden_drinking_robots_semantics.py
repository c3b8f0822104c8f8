"""Golden rollouts of the reference's OWN `DrinkingEnv.step` (envs/drinking.py:10-117 + env.py:174-274, unmodified) with Sawyer and
with PR2, on the CPU oracle through the pybullet facade of make_golden_drinking_semantics.py (the same wiring, with the robot's
reference class in place of Jaco).

The start state: the robot's base pose and start angles come from this repo's TOC reset (`DrinkingSawyerBatch` / `DrinkingPR2Batch`)
on the kernel bodies compiled for the host (the oracle has no batched IK); the oracle then replays that placement, puts the water in
the cup and runs the 50-step settle, and its state is stored.  The reference's robot is given the joint limits its own
`Agent.update_joint_limits` derives from the URDF (+-1e10 for PR2's continuous joints; make_golden_feeding_robots_semantics.py).
As in drinking_semantics.npz the robot tips the cup with its last two joints, one particle is tossed up from just in front of the
mouth (swallowed) and one appears 30 cm beside the cup (spilled).

Output: tests/golden/drinking_sawyer_semantics.npz and drinking_pr2_semantics.npz, replayed by tests/test_drinking_robots_semantics.py.

usage: python tests/golden/make_golden_drinking_robots_semantics.py [/root/reference]   (needs tests/kernel_harness/libagphys_emu.so)"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_drinking_semantics import N_STEPS, SPILL_STEP, SWALLOW_STEP, SWALLOW_V0  # noqa: E402
from make_golden_feeding_robots_semantics import reference_limits  # noqa: E402

CASES = {'sawyer': ('DrinkingSawyerEnv', 'DrinkingSawyerBatch', 3), 'pr2': ('DrinkingPR2Env', 'DrinkingPR2Batch', 5)}


def start(batch_cls, seed):
    """TOC placement on the host-compiled kernels, then the oracle's own reset with that placement and its settle."""
    from assistive_gym_b200 import capi
    from assistive_gym_b200.sim import BatchSim
    from oracle.oracle_py import OracleSim
    db = batch_cls()
    emu = BatchSim(db.scene, db.config(), 1, _lib=capi.load_library(os.path.join(ROOT, 'tests', 'kernel_harness', 'libagphys_emu.so')))
    smp = db.reset(emu, np.random.default_rng(seed), settle_steps=0, impairment='none')
    assert db.unresolved == 0 and int(smp['goals_reached'][0]) >= 2
    emu.close()
    sim = OracleSim(db.scene, db.config(), 1)
    db.reset(sim, np.random.default_rng(seed), settle_steps=50, sample=smp)
    return db, sim, smp


def record(key, ref_envs):
    import assistive_gym_b200.drinking_robots_batch as drb
    from assistive_gym.envs.agents.agent import Agent
    from assistive_gym.envs.util import Util
    from make_golden_feeding_semantics import Facade
    env_name, batch_name, seed = CASES[key]
    db, sim, smp = start(getattr(drb, batch_name), seed)
    start_state = sim.state_get()
    male = bool(smp['male'][0])
    hb = db.humans['male' if male else 'female']
    env = getattr(ref_envs, env_name)()
    p = sys.modules['pybullet']
    Facade(sim, db.scene, f32_targets=True).install(p)

    def euler(q, physicsClientId=None):                                 # PyBullet's getEulerFromQuaternion: roll, pitch, yaw (fixed axes x, y, z)
        x, y, z, w = [float(v) for v in q]
        sinp = 2 * (w * y - z * x)
        return (np.arctan2(2 * (w * x + y * z), 1 - 2 * (x * x + y * y)), np.arcsin(np.clip(sinp, -1, 1)), np.arctan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z)))
    p.getEulerFromQuaternion = euler

    def quat(e, physicsClientId=None):
        r, pt, y = [float(v) for v in e]
        cr, sr, cp, sp, cy, sy = np.cos(r / 2), np.sin(r / 2), np.cos(pt / 2), np.sin(pt / 2), np.cos(y / 2), np.sin(y / 2)
        return [sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy]
    p.getQuaternionFromEuler = quat
    env.robot.body, env.tool.body, env.human.body = db.robot, db.tool, hb
    env.human.gender = 'male' if male else 'female'
    for a in (env.robot, env.tool, env.human):
        a.id = 0
    lo, hi = reference_limits(db.R['asset'], env.robot.controllable_joint_indices)
    env.robot.controllable_joint_lower_limits, env.robot.controllable_joint_upper_limits = lo, hi
    env.robot.motor_gains = env.human.motor_gains = 0.005               # drinking.py:130
    env.agents = [env.robot]
    env.waters = []
    for w in db.waters:
        a = Agent(); a.body, a.id = w, 0
        env.waters.append(a)
    env.waters_active = list(env.waters)
    env.total_water_count = len(env.waters)
    env.cup_top_center_offset, env.cup_bottom_center_offset = np.array([0, 0, -0.055]), np.array([0, 0, 0.07])
    env.mouth_pos = [0, -0.11, 0.03] if male else [0, -0.1, 0.03]
    env.target = types.SimpleNamespace(set_base_pos_orient=lambda *a, **k: None)
    env.iteration, env.task_success, env.last_sim_time, env.gui = 0, 0, None, False
    env.action_space = types.SimpleNamespace(low=-np.ones(7), high=np.ones(7))
    env.np_random = np.random.RandomState(0)
    if getattr(env, 'util', None) is None:
        env.util = Util(0, env.np_random)
    env.update_targets()
    actions = np.zeros((N_STEPS, 7))
    actions[:, 5] = 1.0                                                 # tip the cup with the last two joints ...
    actions[:, 6] = 1.0
    actions[:, :5] = np.random.default_rng(seed + 1).uniform(-1, 1, size=(N_STEPS, 5)) * 0.2
    obs, rew, done, total, success, n_w, n_a = [], [], [], [], [], [], []
    swallow, swallow_pos, spill, spill_pos = -1, np.zeros(3), -1, np.zeros(3)
    for t in range(N_STEPS):
        if t == SWALLOW_STEP:
            swallow = db.waters.index(env.waters[0].body)
            head = sim.get_link_states([db.gl(hb, 23)])['pos'][0, 0]
            swallow_pos = env.target_pos + 0.015 * (env.target_pos - head) / np.linalg.norm(env.target_pos - head)      # 1.5 cm in front of the mouth
            sim.set_base_pose(db.waters[swallow], swallow_pos[None], np.array([[0, 0, 0, 1.0]]))
            sim.set_base_velocity(db.waters[swallow], np.array([[0, 0, SWALLOW_V0]]), np.zeros((1, 3)))
        if t == SPILL_STEP:                                                # a particle appears 30 cm beside the cup (out of it, farther than 0.1 m)
            spill = db.waters.index(env.waters[0].body)
            spill_pos = sim.get_link_states([int(db.scene['body_link0'][db.tool])])['com_pos'][0, 0] + np.array([0.3, 0.0, 0.0])
            sim.set_base_pose(db.waters[spill], spill_pos[None], np.array([[0, 0, 0, 1.0]]))
            sim.set_base_velocity(db.waters[spill], np.zeros((1, 3)), np.zeros((1, 3)))
        o, r, d, info = env.step(actions[t].copy())
        obs.append(np.asarray(o, dtype=np.float64)); rew.append(float(r)); done.append(bool(d)); total.append(float(info['total_force_on_human']))
        success.append(int(env.task_success)); n_w.append(len(env.waters)); n_a.append(len(env.waters_active))
    out = {('sample_' + k): np.asarray(v) for k, v in smp.items()}
    out.update(start_state=start_state, actions=actions, obs=np.array(obs), reward=np.array(rew), done=np.array(done), total_force=np.array(total),
               task_success=np.array(success), n_waters=np.array(n_w), n_waters_active=np.array(n_a), swallow_step=np.array(SWALLOW_STEP),
               swallow_water=np.array(swallow), swallow_v0=np.array(SWALLOW_V0), swallow_pos=np.array(swallow_pos), spill_step=np.array(SPILL_STEP),
               spill_water=np.array(spill), spill_pos=np.array(spill_pos), seed=np.array(seed), robot_lower=lo, robot_upper=hi)
    np.savez_compressed(os.path.join(HERE, 'drinking_%s_semantics.npz' % key), **out)
    print(key, 'waters left', n_w, 'active', n_a[-1], 'swallowed', success[-1], 'reward', np.round(rew, 2))


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    from make_golden_env_logic import install_stubs
    install_stubs(ref)
    import assistive_gym  # noqa: F401  (the reference package)
    from assistive_gym.envs import drinking_envs
    for key in CASES:
        record(key, drinking_envs)


if __name__ == '__main__':
    main()
