"""Co-optimisation step of BedBathing (reference envs/bed_bathing.py:12-111 with dict actions, :190-203 `update_targets`, env.py:174-235
incl. `Human.enforce_realistic_joint_limits`, agents/human.py:134-152): `BedBathingSawyerHumanEnv` of this repo, run on the CPU oracle,
replays the rollout of tests/golden/bathing_coop_semantics.npz, produced by the reference's OWN step code on the same oracle through
a pybullet facade (tests/golden/make_golden_bathing_coop_semantics.py).  The pad is pressed onto the forearm while the person rolls
it, so targets are wiped where the moving arm has carried them; then the person turns the upper arm until the joint-limit
classifier sends it back.  Both dict observations, the reward, the wiped targets and the arm's joint angles must agree."""
import os

import numpy as np

from assistive_gym_b200 import envs
from assistive_gym_b200.bed_bathing_batch import RIGHT_ARM_JOINTS, BedBathingBatch
from oracle.oracle_py import OracleSim
from tests.test_bed_bathing import _pressed_pair

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'bathing_coop_semantics.npz'))


def test_golden_wipes_moved_targets_and_the_classifier_acts():
    moved = np.linalg.norm(G['wiped_pos'] - G['targets_reset'][G['wiped_target']], axis=1)
    assert int((moved >= 0.01).sum()) >= 3                                     # wiped where the arm carried them, not where they started
    assert int(G['restores'][-1]) >= 1                                         # the classifier sent the arm back at least once
    assert int(G['new_contact_points'].sum()) == len(G['wiped_target']) == int(G['task_success'][-1])


def test_cooptimisation_bathing_step_reproduces_the_reference_s_rollout():
    bb = BedBathingBatch(controllable_person=True)
    sim, _other, smp, _ik = _pressed_pair(bb, lambda sc, cfg, n: OracleSim(sc, cfg, n), 1, seed=8)
    assert np.allclose(sim.state_get(), G['start_state'], atol=1e-9)            # the generator's start state ...
    sim.state_set(G['start_state']); sim.forward_kinematics()                  # ... to the last bit
    env = envs.make('BedBathingSawyerHuman-v1', n_envs=1)
    env._bb = bb
    env.id = sim                                                               # the env's per-call path on the oracle instead of the CUDA library
    env.plane.init(bb.plane, sim, env.np_random, indices=-1)
    env.robot.init(bb.robot, sim, env.np_random)
    env.tool.init(bb.tool, sim, env.np_random, indices=-1)
    env.furniture.init(bb.bed, sim, env.np_random, indices=-1)
    env.robot.motor_gains, env.robot.motor_forces = float(G['motor_gain']), float(G['motor_force'])
    env.male = G['sample_male'].astype(bool)
    env.humans = {}
    env.agents = [env.robot]
    for g, hb in bb.humans.items():
        h = type(env.human)(env.human.controllable_joint_indices, controllable=True)
        h.init(hb, sim, env.np_random, env.human.controllable_joint_indices)
        h.env_mask = env.male if g == 'male' else ~env.male
        h.set_limit_scale(np.ones(1))
        env.humans[g] = h
        env.agents.append(h)
    env.targets_pos_world, env.targets_alive = bb.targets_world(sim, {'male': env.male})
    env.total_target_count = env.targets_alive.sum(axis=1)
    assert int(env.total_target_count[0]) == int(G['total_target_count'])
    env.task_success = np.zeros(1, dtype=int)
    env.iteration = 0
    hb = bb.humans['male' if env.male[0] else 'female']
    links = [bb.gl(hb, j) for j in RIGHT_ARM_JOINTS]
    for t, a in enumerate(G['actions']):
        o, r, d, info = env.step({'robot': a[:7], 'human': a[7:]})
        assert sorted(o) == ['human', 'robot'] and sorted(d) == ['__all__', 'human', 'robot'] and sorted(info) == ['human', 'robot']
        arm = sim.get_joint_states(links)[0][0]
        assert np.allclose(arm, G['arm_q'][t], rtol=0, atol=1e-7), (t, np.abs(arm - G['arm_q'][t]).max())
        # forces: the reference sums the fp32 contact records, the restatement asks the oracle for the fp64 sum
        assert np.allclose(o['robot'][:23], G['obs_robot'][t][:23], rtol=0, atol=1e-6), (t, np.abs(o['robot'][:23] - G['obs_robot'][t][:23]).max())
        assert abs(o['robot'][23] - G['obs_robot'][t][23]) < 1e-4 * (1 + abs(G['obs_robot'][t][23]))
        assert np.allclose(o['human'][:26], G['obs_human'][t][:26], rtol=0, atol=1e-6), (t, np.abs(o['human'][:26] - G['obs_human'][t][:26]).max())
        assert np.allclose(o['human'][26:], G['obs_human'][t][26:], rtol=1e-4, atol=1e-4)
        assert abs(r['robot'] - G['reward'][t]) < 1e-5 and r['robot'] == r['human']
        assert bool(d['__all__']) == bool(G['done'][t])
        assert int(env.new_contact_points[0]) == int(G['new_contact_points'][t]) and int(env.task_success[0]) == int(G['task_success'][t]), t
        assert int(info['robot']['task_success']) == int(G['task_success'][t] >= G['total_target_count'] * 0.3)
