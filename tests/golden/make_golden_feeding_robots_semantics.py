"""Golden rollouts of the reference's OWN `FeedingEnv.step` with Sawyer and with PR2, and of `FeedingSawyerHumanEnv.step`, on the CPU
oracle through the pybullet facade of make_golden_feeding_semantics.py (the same wiring as make_golden_feeding_semantics.py and
make_golden_feeding_coop_semantics.py, with the robot's reference class in place of Jaco).

The start state: the robot's base pose and start angles come from this repo's TOC reset (`FeedingSawyerBatch` / `FeedingPR2Batch`) on the
kernel bodies compiled for the host (the oracle has no batched IK); the oracle then replays that placement, puts the bowl and the food in
place and runs the 25-step settle, and its state is stored.  The reference's robot is given the joint limits its own
`Agent.update_joint_limits` derives from the URDF (agent.py:209-230: a joint reported as (0, -1) is +-1e10), read from the compiled
model, so PR2's two continuous arm joints go through the reference's unlimited action clamp.

Output: tests/golden/feeding_sawyer_semantics.npz, feeding_pr2_semantics.npz (a particle tossed up from the mouth at EAT_STEP, as in
feeding_semantics.npz) and feeding_sawyer_coop_semantics.npz.  tests/test_feeding_robots_semantics.py replays them.

usage: python tests/golden/make_golden_feeding_robots_semantics.py [/root/reference]   (needs tests/kernel_harness/libagphys_emu.so)"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

N_STEPS, EAT_STEP, EAT_V0 = 30, 12, 0.5886
N_COOP = 24
HEAD = [20, 21, 22, 23]
CASES = {'sawyer': ('FeedingSawyerEnv', 'FeedingSawyerBatch', 3, False), 'pr2': ('FeedingPR2Env', 'FeedingPR2Batch', 5, False),
         'sawyer_coop': ('FeedingSawyerHumanEnv', 'FeedingSawyerBatch', 7, True)}


def reference_limits(asset, joints):
    """Agent.update_joint_limits of the reference for `joints`, from the compiled URDF model (getJointInfo[8:10])."""
    m = json.load(open(os.path.join(ROOT, 'assistive_gym_b200', 'assets', asset + '.agmodel.json')))
    lo, hi = [], []
    for j in joints:
        jt = m['links'][j + 1]['joint']
        l, u = (0.0, -1.0) if jt['type'] in ('continuous', 'fixed') else (jt['lower'], jt['upper'])
        if l == 0 and u == -1:
            l, u = -1e10, 1e10
        lo.append(l); hi.append(u)
    return np.array(lo, dtype=np.float64), np.array(hi, dtype=np.float64)


def start(batch_cls, seed, coop):
    """TOC placement on the host-compiled kernels, then the oracle's own reset with that placement and its settle."""
    from assistive_gym_b200 import capi
    from assistive_gym_b200.sim import BatchSim
    from oracle.oracle_py import OracleSim
    fb = batch_cls()
    emu = BatchSim(fb.scene, fb.config(), 1, _lib=capi.load_library(os.path.join(ROOT, 'tests', 'kernel_harness', 'libagphys_emu.so')))
    smp = fb.reset(emu, np.random.default_rng(seed), settle_steps=0, impairment='none', simulate_head=coop)
    assert fb.unresolved == 0 and int(smp['goals_reached'][0]) >= 2
    emu.close()
    sim = OracleSim(fb.scene, capi.default_config(), 1)
    fb.reset(sim, np.random.default_rng(seed), settle_steps=25, sample=smp, simulate_head=coop)
    return fb, sim, smp


def wire(env, fb, sim, smp, coop):
    from assistive_gym.envs.agents.agent import Agent
    from make_golden_feeding_semantics import Facade
    p = sys.modules['pybullet']
    fac = Facade(sim, fb.scene, f32_targets=True)           # motor targets reach the physics in fp32, as through the repo's `Agent.control`
    fac.install(p)
    male = bool(smp['male'][0])
    hb = fb.humans['male' if male else 'female']
    env.robot.body, env.tool.body, env.human.body = fb.robot, fb.tool, hb
    env.human.gender = 'male' if male else 'female'
    for a in (env.robot, env.tool, env.human):
        a.id = 0
    lo, hi = reference_limits(fb.R['asset'], env.robot.controllable_joint_indices)
    env.robot.controllable_joint_lower_limits, env.robot.controllable_joint_upper_limits = lo, hi
    env.robot.motor_gains = env.human.motor_gains = 0.025               # feeding.py:122
    env.agents = [env.robot]
    if coop:
        def resetJointState(body, jointIndex=None, targetValue=0.0, targetVelocity=0.0, physicsClientId=None):
            sim.set_joint_state([fac.gl(body, jointIndex)], q=np.array([[float(targetValue)]]), qd=np.array([[float(targetVelocity)]]))
            sim.forward_kinematics()
        p.resetJointState = resetJointState
        sc, h = fb.scene, env.human
        assert list(h.controllable_joint_indices) == HEAD
        h.all_joint_indices = list(range(int(sc['body_nlinks'][hb]) - 1))
        h.lower_limits = {j: float(sc['link_lower'][fac.gl(hb, j)]) for j in h.all_joint_indices}
        h.upper_limits = {j: float(sc['link_upper'][fac.gl(hb, j)]) for j in h.all_joint_indices}
        h.controllable_joint_lower_limits = np.array([h.lower_limits[j] for j in HEAD])
        h.controllable_joint_upper_limits = np.array([h.upper_limits[j] for j in HEAD])
        h.impairment, h.tremors, h.strength = 'none', np.zeros(4), 1.0
        h.arm_previous_valid_pose = {True: None, False: None}
        env.agents.append(h)
        env.action_robot_len, env.action_human_len = 7, 4
    env.foods = []
    for f in fb.foods:
        a = Agent(); a.body, a.id = f, 0
        env.foods.append(a)
    env.foods_active = list(env.foods)
    env.total_food_count = len(env.foods)
    env.mouth_pos = [0, -0.11, 0.03] if male else [0, -0.1, 0.03]       # feeding.py:186
    env.target = types.SimpleNamespace(set_base_pos_orient=lambda *a, **k: None)
    env.iteration, env.task_success, env.last_sim_time, env.gui = 0, 0, None, False
    k = 11 if coop else 7
    env.action_space = types.SimpleNamespace(low=-np.ones(k), high=np.ones(k))
    env.np_random = np.random.RandomState(0)
    env.update_targets()
    return fac, hb


def record(key, ref_envs):
    import assistive_gym_b200.feeding_robots_batch as frb
    env_name, batch_name, seed, coop = CASES[key]
    fb, sim, smp = start(getattr(frb, batch_name), seed, coop)
    env = getattr(ref_envs, env_name)()
    fac, hb = wire(env, fb, sim, smp, coop)
    start_state = sim.state_get()
    arng = np.random.default_rng(seed + 1)
    n = N_COOP if coop else N_STEPS
    a_r = arng.uniform(-1, 1, size=(n, 7)) * 0.3                       # gentle, so that the food stays on the spoon for a while
    out = {('sample_' + k): np.asarray(v) for k, v in smp.items()}
    if coop:
        a_h = np.concatenate([np.tile([0.0, 1.0, -1.0, 1.0], (n // 2, 1)), np.tile([0.0, -1.0, 1.0, -1.0], (n - n // 2, 1))])
        obs_r, obs_h, rew, head = [], [], [], []
        for t in range(n):
            o, r, d, info = env.step({'robot': a_r[t].copy(), 'human': a_h[t].copy()})
            obs_r.append(np.asarray(o['robot'], dtype=np.float64)); obs_h.append(np.asarray(o['human'], dtype=np.float64)); rew.append(float(r['robot']))
            head.append(sim.get_joint_states([fac.gl(hb, j) for j in HEAD])[0][0].copy())
        out.update(robot_actions=a_r, human_actions=a_h, obs_robot=np.array(obs_r), obs_human=np.array(obs_h), reward=np.array(rew), head_q=np.array(head))
        print(key, 'head (deg) at steps 0, 11, 23', np.round(np.rad2deg(np.array(head)[[0, 11, n - 1]]), 1))
    else:
        obs, rew, done, total, success, n_foods, n_active = [], [], [], [], [], [], []
        eat_food = -1
        for t in range(n):
            if t == EAT_STEP and env.foods:                             # forced event: a particle still on the spoon is tossed up from the mouth target
                eat_food = fb.foods.index(env.foods[0].body)
                sim.set_base_pose(fb.foods[eat_food], env.target_pos[None], np.array([[0, 0, 0, 1.0]]))
                sim.set_base_velocity(fb.foods[eat_food], np.array([[0, 0, EAT_V0]]), np.zeros((1, 3)))
            o, r, d, info = env.step(a_r[t].copy())
            obs.append(np.asarray(o, dtype=np.float64)); rew.append(float(r)); done.append(bool(d)); total.append(float(info['total_force_on_human']))
            success.append(int(env.task_success)); n_foods.append(len(env.foods)); n_active.append(len(env.foods_active))
        out.update(actions=a_r, obs=np.array(obs), reward=np.array(rew), done=np.array(done), total_force=np.array(total), task_success=np.array(success),
                   n_foods=np.array(n_foods), n_foods_active=np.array(n_active), eat_step=np.array(EAT_STEP), eat_v0=np.array(EAT_V0), eat_food=np.array(eat_food))
        print(key, 'steps', n, 'foods left', n_foods[-1], 'active', n_active[-1], 'task_success', success[-1], 'reward range', min(rew), max(rew))
    out['seed'] = np.array(seed)
    out['robot_lower'], out['robot_upper'] = env.robot.controllable_joint_lower_limits, env.robot.controllable_joint_upper_limits
    out['start_state'] = start_state
    name = {'sawyer': 'feeding_sawyer_semantics.npz', 'pr2': 'feeding_pr2_semantics.npz', 'sawyer_coop': 'feeding_sawyer_coop_semantics.npz'}[key]
    np.savez_compressed(os.path.join(HERE, name), **out)


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    from make_golden_env_logic import install_stubs
    install_stubs(ref)
    import assistive_gym  # noqa: F401  (the reference package)
    from assistive_gym.envs import feeding_envs
    for key in CASES:
        record(key, feeding_envs)


if __name__ == '__main__':
    main()
