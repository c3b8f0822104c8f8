"""Golden rollout of the reference's OWN co-optimisation Feeding step with a `tremor` person (`FeedingJacoHumanEnv`: envs/feeding.py:12-112,
`take_step` env.py:174-235 with the controllable tremor branch :205-215: the person's action accumulates into target_joint_angles, the
head is driven to target +- tremors), executed on the CPU oracle through the pybullet facade of make_golden_feeding_semantics.py.  The
person nods and turns into a joint limit, where the clamp zeroes part of the action.  Output:
tests/golden/feeding_coop_tremor_semantics.npz, replayed by tests/test_coop_tremor.py on the per-call env (oracle) and on the fused
step (kernel bodies compiled for the host).

usage: python tests/golden/make_golden_feeding_coop_tremor_semantics.py [reference checkout]"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

N_STEPS, SEED = 16, 5
HEAD = [20, 21, 22, 23]


def main():
    ref = sys.argv[1] if len(sys.argv) > 1 else '/root/reference'
    from assistive_gym_b200 import capi
    from assistive_gym_b200.feeding_batch import FeedingBatch
    from oracle.oracle_py import OracleSim
    fb = FeedingBatch()
    sim = OracleSim(fb.scene, capi.default_config(), 1)
    smp = fb.reset(sim, np.random.default_rng(SEED), settle_steps=25, impairment='none', simulate_head=True)
    male = bool(smp['male'][0])
    hb = fb.humans['male' if male else 'female']
    from make_golden_env_logic import install_stubs
    from make_golden_feeding_semantics import Facade
    install_stubs(ref)
    import assistive_gym  # noqa: F401  (the reference package)
    from assistive_gym.envs.agents.agent import Agent
    from assistive_gym.envs.feeding_envs import FeedingJacoHumanEnv
    env = FeedingJacoHumanEnv()
    p = sys.modules['pybullet']
    fac = Facade(sim, fb.scene, f32_targets=True)
    fac.install(p)

    def resetJointState(body, jointIndex=None, targetValue=0.0, targetVelocity=0.0, physicsClientId=None):
        sim.set_joint_state([fac.gl(body, jointIndex)], q=np.array([[float(targetValue)]]), qd=np.array([[float(targetVelocity)]]))
        sim.forward_kinematics()
    p.resetJointState = resetJointState
    env.robot.body, env.tool.body, env.human.body = fb.robot, fb.tool, hb
    env.human.gender = 'male' if male else 'female'
    for a in (env.robot, env.tool, env.human):
        a.id = 0
    sc = fb.scene
    env.robot.controllable_joint_lower_limits = np.array(fb.arm_lower, dtype=np.float64)
    env.robot.controllable_joint_upper_limits = np.array(fb.arm_upper, dtype=np.float64)
    h = env.human
    assert list(h.controllable_joint_indices) == HEAD
    h.all_joint_indices = list(range(int(sc['body_nlinks'][hb]) - 1))
    h.lower_limits = {j: float(sc['link_lower'][fac.gl(hb, j)]) for j in h.all_joint_indices}
    h.upper_limits = {j: float(sc['link_upper'][fac.gl(hb, j)]) for j in h.all_joint_indices}
    h.controllable_joint_lower_limits = np.array([h.lower_limits[j] for j in HEAD])
    h.controllable_joint_upper_limits = np.array([h.upper_limits[j] for j in HEAD])
    # the tremor person of human.py:87-90 (amplitudes stored at fp32, as the batched env draws them) and its target_joint_angles
    # as setup_joints takes them (human.py:123): the sampled head pose, limit-clipped
    tremors = np.random.default_rng(SEED + 2).uniform(np.deg2rad(-20), np.deg2rad(20), size=4).astype(np.float32).astype(np.float64)
    target0 = fb.tremor_rest_of(smp)[0].copy()
    h.impairment, h.tremors, h.strength, h.target_joint_angles = 'tremor', tremors.copy(), 1.0, target0.copy()
    h.arm_previous_valid_pose = {True: None, False: None}
    env.robot.motor_gains = env.human.motor_gains = 0.025               # feeding.py:122
    env.agents = [env.robot, env.human]
    env.foods = []
    for f in fb.foods:
        a = Agent(); a.body, a.id = f, 0
        env.foods.append(a)
    env.foods_active = list(env.foods)
    env.total_food_count = len(env.foods)
    env.mouth_pos = [0, -0.11, 0.03] if male else [0, -0.1, 0.03]
    env.target = types.SimpleNamespace(set_base_pos_orient=lambda *a, **k: None)
    env.iteration, env.task_success, env.last_sim_time, env.gui = 0, 0, None, False
    env.action_space = types.SimpleNamespace(low=-np.ones(11), high=np.ones(11))
    env.action_robot_len, env.action_human_len = 7, 4
    env.np_random = np.random.RandomState(0)
    env.update_targets()
    start_state = sim.state_get()                                       # stored: the replay does not depend on the IK of the reset being bit-reproducible
    arng = np.random.default_rng(SEED + 1)
    a_r = arng.uniform(-1, 1, size=(N_STEPS, 7)) * 0.3
    a_h = np.tile([0.0, 0.5, -0.5, 0.5], (N_STEPS, 1))                   # nod / turn into the limits and stay there, trembling
    obs_r, obs_h, rew, head, target = [], [], [], [], []
    for t in range(N_STEPS):
        o, r, d, info = env.step({'robot': a_r[t].copy(), 'human': a_h[t].copy()})
        obs_r.append(np.asarray(o['robot'], dtype=np.float64)); obs_h.append(np.asarray(o['human'], dtype=np.float64)); rew.append(float(r['robot']))
        head.append(sim.get_joint_states([fac.gl(hb, j) for j in HEAD])[0][0].copy())
        target.append(np.array(h.target_joint_angles, dtype=np.float64))
    head = np.array(head)
    out = {('sample_' + k): np.asarray(v) for k, v in smp.items()}
    out.update(robot_actions=a_r, human_actions=a_h, obs_robot=np.array(obs_r), obs_human=np.array(obs_h), reward=np.array(rew), head_q=head, seed=np.array(SEED),
               tremors=tremors, target0=target0, target_q=np.array(target),
               head_lower=np.array([h.lower_limits[j] for j in HEAD]), head_upper=np.array([h.upper_limits[j] for j in HEAD]))
    out['start_state'] = start_state
    np.savez_compressed(os.path.join(HERE, 'feeding_coop_tremor_semantics.npz'), **out)
    step = np.abs(np.diff(np.vstack([target0, np.array(target)]), axis=0)).max(axis=1)
    print('target travel per step (rad)', np.round(step, 3))
    print('steps', N_STEPS, 'head (deg) at the first, middle and last step', np.round(np.rad2deg(head[[0, N_STEPS // 2, -1]]), 1), 'limits', np.round(np.rad2deg(out['head_lower']), 0), np.round(np.rad2deg(out['head_upper']), 0))


if __name__ == '__main__':
    main()
