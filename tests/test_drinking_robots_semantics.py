"""DrinkingSawyer-v1 and DrinkingPR2-v1 against the reference's OWN `DrinkingEnv.step` with those robots
(tests/golden/drinking_{sawyer,pr2}_semantics.npz, recorded on the CPU oracle by make_golden_drinking_robots_semantics.py: the cup
tipped by the last two joints, one particle swallowed (+10), one spilled (-1)).  These pin what is robot-specific in the step: the end
effector of the velocity term, the robot base frame of the observation and PR2's continuous arm joints under the unlimited action
clamp and the [-pi, pi) observation wrap.

- the env's own per-call step on the oracle reproduces each rollout to rounding;
- the fused kernel bodies compiled for the host (`ag_drinking_step_host`) replay them from the golden start at DrinkingJaco-v1's bounds;
- on the H100, `drinking_step_dev` with torch tensors replays them at the same bounds."""
import os

import numpy as np
import pytest

from assistive_gym_b200 import envs
from assistive_gym_b200.drinking_robots_batch import DrinkingPR2Batch, DrinkingSawyerBatch
from assistive_gym_b200.sim import BatchSim

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CASES = {'sawyer': ('DrinkingSawyer-v1', DrinkingSawyerBatch), 'pr2': ('DrinkingPR2-v1', DrinkingPR2Batch)}


def _load(robot):
    G = np.load(os.path.join(GOLDEN, 'drinking_%s_semantics.npz' % robot))
    return G, {k[len('sample_'):]: G[k] for k in G.files if k.startswith('sample_')}


def _inject(db, sim, G, t):
    """the golden's swallowed / spilled particle, placed before step t"""
    for key in ('swallow', 'spill'):
        if t == int(G[key + '_step']):
            w = db.waters[int(G[key + '_water'])]
            sim.set_base_pose(w, G[key + '_pos'][None], np.array([[0, 0, 0, 1.0]]))
            sim.set_base_velocity(w, np.array([[0, 0, float(G['swallow_v0']) if key == 'swallow' else 0.0]]), np.zeros((1, 3)))


def _count(mask):
    return np.array([bin(int(m)).count('1') for m in np.atleast_1d(mask)])


def _per_call_replay(robot, sim, state, check):
    """`DrinkingEnv.step` (per call, through the Agent getters) on `sim` from the golden start; `check(t, env, out)` per step."""
    G, smp = _load(robot)
    env = envs.make(CASES[robot][0], n_envs=1)
    db = env._db
    assert np.array_equal(G['robot_lower'], db.arm_lower) and np.array_equal(G['robot_upper'], db.arm_upper)     # the reference's own limits
    db.reset(sim, np.random.default_rng(0), settle_steps=0, sample=smp)
    sim.state_set(state); sim.forward_kinematics()
    env.attach(sim)
    env.start_episode(smp)
    for t, a in enumerate(G['actions']):
        _inject(db, sim, G, t)
        if not check(t, env, env.step(a)):
            break
    return G


@pytest.mark.parametrize('robot', list(CASES))
def test_per_call_step_reproduces_the_reference_s_rollout(robot):
    from oracle.oracle_py import OracleSim
    G, _ = _load(robot)
    sim = OracleSim(CASES[robot][1]().scene, DrinkingSawyerBatch.config(), 1)

    def check(t, env, out):
        obs, rew, done, info = out
        assert np.allclose(obs[:24], G['obs'][t][:24], rtol=0, atol=1e-9), (t, np.abs(obs - G['obs'][t]).max())
        assert abs(obs[24] - G['obs'][t][24]) < 1e-6 and abs(info['total_force_on_human'] - G['total_force'][t]) < 1e-6      # forces
        assert abs(rew - G['reward'][t]) < 1e-9, (t, rew, G['reward'][t])
        assert bool(done) == bool(G['done'][t])
        assert int(env.waters.sum()) == int(G['n_waters'][t]) and int(env.waters_active.sum()) == int(G['n_waters_active'][t])
        assert int(env.task_success[0]) == int(G['task_success'][t])
        return True
    _per_call_replay(robot, sim, G['start_state'], check)
    # one particle swallowed (+10) and one spilled (-1) in the recorded rollout
    assert G['task_success'][-1] == 1 and G['n_waters'][-1] == 62
    assert G['reward'][int(G['swallow_step'])] > 8 and G['reward'][int(G['spill_step'])] < G['reward'][int(G['spill_step']) - 1] - 0.9


def _replay_fused(lib, robot, step):
    """The fused step from the golden start, against what the reference's own `DrinkingEnv.step` returned, over the whole rollout:
    DrinkingJaco-v1's bounds (observation 1e-4, reward 1e-2), the same task success and particle counts."""
    G, smp = _load(robot)
    db = CASES[robot][1]()
    sim = BatchSim(db.scene, db.config(), 1, _lib=lib)
    db.reset(sim, np.random.default_rng(0), settle_steps=0, sample=smp)
    sim.state_set(G['start_state'].astype(np.float32)); sim.forward_kinematics()
    db.start_fused(sim, smp)
    d_obs, d_rew = [], []
    for t, a in enumerate(G['actions']):
        _inject(db, sim, G, t)
        obs, rew, done, info = step(sim, np.asarray(a, dtype=np.float32)[None])
        ts, w, wa = sim.drinking_get_state()
        d_obs.append(np.abs(obs[0, :24] - G['obs'][t][:24]).max()); d_rew.append(abs(rew[0] - G['reward'][t]))
        assert d_obs[-1] < 1e-4 and d_rew[-1] < 1e-2, (t, d_obs[-1], rew[0], G['reward'][t])
        assert bool(done[0] > 0.5) == bool(G['done'][t])
        assert int(ts[0]) == int(G['task_success'][t]), (t, ts, G['task_success'][t])
        assert _count(w)[0] == int(G['n_waters'][t]) and _count(wa)[0] == int(G['n_waters_active'][t]), (t, _count(w), _count(wa))
    assert sim.overflow_count() == 0
    sim.close()
    print('%s: fused replay over %d steps: obs max %.2e, reward max %.2e' % (robot, len(d_obs), max(d_obs), max(d_rew)))
    return np.array(d_obs), np.array(d_rew)


@pytest.mark.parametrize('robot', list(CASES))
def test_fused_replay_host_compiled(emu_lib, robot):
    _replay_fused(emu_lib, robot, lambda sim, a: sim.drinking_step_host(a))


@pytest.mark.parametrize('robot', list(CASES))
def test_per_call_step_on_the_kernel_bodies_parts_like_the_fused_step(emu_lib, robot):
    """The per-call step on the same fp32 kernels, from the same golden start, stays within the bounds the fused step holds against the
    fp64 oracle over the whole rollout: what separates either from the oracle is fp32 against fp64 physics, which grows through the
    water's contacts from a few 1e-7 at the first step (the per-call step accumulates its PD targets in fp64, the fused one in fp32)."""
    d_fused, r_fused = _replay_fused(emu_lib, robot, lambda sim, a: sim.drinking_step_host(a))
    G, _ = _load(robot)
    db = CASES[robot][1]()
    prod = BatchSim(db.scene, db.config(), 1, _lib=emu_lib)
    d_per, r_per = [], []

    def check(t, env, out):
        obs, rew, done, info = out
        d_per.append(np.abs(obs[:24] - G['obs'][t][:24]).max()); r_per.append(abs(rew - G['reward'][t]))
        assert int(env.waters.sum()) == int(G['n_waters'][t]) and int(env.task_success[0]) == int(G['task_success'][t])
        return True
    _per_call_replay(robot, prod, G['start_state'].astype(np.float32), check)
    prod.close()
    d_per, r_per = np.array(d_per), np.array(r_per)
    print('%s: |oracle - fp32| per step, fused %s\n per-call %s' % (robot, np.array2string(d_fused, precision=1), np.array2string(d_per, precision=1)))
    assert d_per.max() < 1e-4 and r_per.max() < 1e-2
    assert d_fused[0] < 1e-6 and d_per[0] < 1e-6


@pytest.mark.gpu
@pytest.mark.parametrize('robot', list(CASES))
def test_fused_replay_cuda(gpu_lib, robot):
    from tests.test_drinking_fused import _step_dev_torch
    _replay_fused(gpu_lib, robot, _step_dev_torch)
