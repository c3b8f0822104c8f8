"""Co-optimisation step of Dressing (reference envs/dressing.py:12-106 with dict actions, :199-210 `update_targets`, env.py:174-235
incl. `Human.enforce_realistic_joint_limits`, agents/human.py:134-152, util.sleeve_on_arm_reward): `DressingPR2HumanEnv` of this repo,
run on the CPU oracle, replays the rollout of tests/golden/dressing_coop_semantics.npz, produced by the reference's OWN step code
on the same oracle, cloth included, through a pybullet facade (tests/golden/make_golden_dressing_coop_semantics.py).  The person
lifts the left arm inside the gown until a joint reaches its limit and the joint-limit classifier sends the arm back.  Both dict
observations, the reward, the sleeve state and the arm's joint angles must agree."""
import os

import numpy as np

from assistive_gym_b200 import envs
from assistive_gym_b200.dressing_batch import LEFT_ARM_JOINTS, DressingBatch
from oracle.oracle_py import OracleSim

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'dressing_coop_semantics.npz'))
SETTLE = 3                   # the generator's settle at half gravity


def golden_sample():
    return {k[len('sample_'):]: G[k] for k in G.files if k.startswith('sample_')}


def settled_start(db, sim):
    """The generator's start: the co-optimisation reset of the stored sample, then the short settle."""
    db.reset(sim, np.random.default_rng(0), sample=golden_sample(), settle_steps=0)
    sim.cloth_set_gravity([0, 0, -9.81 / 2]); sim.step(SETTLE); sim.cloth_set_gravity([0, 0, -9.81])


def test_golden_moves_the_arm_into_a_limit_and_the_classifier_acts():
    assert G['at_limit'].any()                                                 # some joint reached its limit
    assert int(G['restores'][-1]) >= 1                                         # the classifier sent the arm back at least once
    assert np.abs(G['arm_q'][-1] - G['arm_q'][0]).max() > 0.3                  # the arm moved
    assert G['obs_robot'][:, 23].max() > 5                                     # inside the gown: the cloth presses on the person


def test_cooptimisation_dressing_step_reproduces_the_reference_s_rollout():
    db = DressingBatch(controllable_person=True)
    sim = OracleSim(db.scene, DressingBatch.config(), 1)
    settled_start(db, sim)
    env = envs.make('DressingPR2Human-v1', n_envs=1)
    env._db = db
    env.id = sim                                                               # the env's per-call path on the oracle instead of the CUDA library
    env.plane.init(db.plane, sim, env.np_random, indices=-1)
    env.robot.init(db.robot, sim, env.np_random)
    env.furniture.init(db.wheelchair, sim, env.np_random, indices=-1)
    env.robot.motor_gains = 0.01
    env.male = G['sample_male'].astype(bool)
    env.humans = {}
    env.agents = [env.robot]
    for g, hb in db.humans.items():
        h = type(env.human)(env.human.controllable_joint_indices, controllable=True)
        h.init(hb, sim, env.np_random, env.human.controllable_joint_indices)
        h.env_mask = env.male if g == 'male' else ~env.male
        h.motor_gains = 0.01
        h.set_limit_scale(np.ones(1))
        env.humans[g] = h
        env.agents.append(h)
    env.task_success = np.zeros(1)
    env.iteration = 0
    links = [db.gl(db.humans['male' if env.male[0] else 'female'], j) for j in LEFT_ARM_JOINTS]
    for t, a in enumerate(G['actions']):
        o, r, d, info = env.step({'robot': a[:7], 'human': a[7:]})
        assert sorted(o) == ['human', 'robot'] and sorted(d) == ['__all__', 'human', 'robot'] and sorted(info) == ['human', 'robot']
        arm = sim.get_joint_states(links)[0][0]
        assert np.allclose(arm, G['arm_q'][t], rtol=0, atol=1e-7), (t, np.abs(arm - G['arm_q'][t]).max())
        assert np.allclose(o['robot'][:23], G['obs_robot'][t][:23], rtol=0, atol=1e-6), (t, np.abs(o['robot'][:23] - G['obs_robot'][t][:23]).max())
        assert np.allclose(o['human'][:26], G['obs_human'][t][:26], rtol=0, atol=1e-6), (t, np.abs(o['human'][:26] - G['obs_human'][t][:26]).max())
        # forces: the same contacts under both, summed in a different order
        assert np.allclose(o['robot'][23:], G['obs_robot'][t][23:], rtol=1e-6, atol=1e-6)
        assert np.allclose(o['human'][26:], G['obs_human'][t][26:], rtol=1e-6, atol=1e-6)
        assert abs(r['robot'] - G['reward'][t]) < 1e-6 and r['robot'] == r['human']
        assert bool(d['__all__']) == bool(G['done'][t])
        assert int(env.forearm_in_sleeve[0]) + 2 * int(env.upperarm_in_sleeve[0]) == int(G['sleeve'][t])
        assert abs(env.task_success[0] - G['task_success'][t]) < 1e-6
        assert int(info['robot']['task_success']) == int(G['task_success'][t] >= 0.4)
