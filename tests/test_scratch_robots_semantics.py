"""ScratchItchSawyer-v1, ScratchItchPR2-v1 and their co-optimisation ids against the reference's OWN `ScratchItchEnv.step` with those
robots (tests/golden/scratch_{sawyer,pr2}_semantics.npz and scratch_{sawyer,pr2}_coop_semantics.npz, recorded on the CPU oracle by
make_golden_scratch_robots_semantics.py).  These pin what is robot-specific in the step: the left end effector of the velocity term,
the robot base frame of the observation (PR2's base inertial frame) and the scratcher held at the left tool joint.  PR2's two
continuous arm joints stay inside (-pi, pi) in these rollouts, so they do not exercise the observation wrap or the unlimited action
clamp; `test_pr2_continuous_joint_wraps_past_pi_host_compiled` drives one past pi on the fused and the per-call step instead.  Each single-agent rollout starts with the scratcher's
tip on the itch target, so scratches are counted; in each co-optimisation rollout the classifier sends the raised arm back.

- the env's own per-call step on the oracle reproduces each rollout to rounding;
- the fused kernel bodies compiled for the host (`ag_scratch_step_host`, `ag_coop_step_host`) replay them from the golden start;
- on the H100, `scratch_step_dev` / `coop_step_dev` with torch tensors replay them."""
import os

import numpy as np
import pytest

from assistive_gym_b200 import capi, envs
from assistive_gym_b200.scratch_itch_batch import RIGHT_ARM_JOINTS
from assistive_gym_b200.scratch_itch_robots_batch import ScratchItchPR2Batch, ScratchItchSawyerBatch
from assistive_gym_b200.sim import BatchSim

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
CASES = {'sawyer': ScratchItchSawyerBatch, 'pr2': ScratchItchPR2Batch}
IDS = {'sawyer': 'ScratchItchSawyer-v1', 'pr2': 'ScratchItchPR2-v1', 'sawyer_coop': 'ScratchItchSawyerHuman-v1', 'pr2_coop': 'ScratchItchPR2Human-v1'}


def _load(name):
    G = np.load(os.path.join(GOLDEN, 'scratch_%s_semantics.npz' % name))
    return G, {k[len('sample_'):]: G[k] for k in G.files if k.startswith('sample_')}


def _env_on_oracle(key, monkeypatch):
    """The env's own reset on the CPU oracle, from the golden's draws and TOC placement, then the golden's start state."""
    import assistive_gym_b200.envs.scratch_itch as scratch_mod
    from oracle.oracle_py import OracleSim
    G, smp = _load(key)
    env = envs.make(IDS[key], n_envs=1)
    sb = env._sb
    assert np.array_equal(G['robot_lower'], sb.arm_lower) and np.array_equal(G['robot_upper'], sb.arm_upper)     # the reference's own limits
    sim = OracleSim(sb.scene, capi.default_config(residual_threshold=0.0), 1)
    monkeypatch.setattr(scratch_mod, 'BatchSim', lambda *a, **k: sim)
    monkeypatch.setattr(sb, 'sample', lambda *a, **k: dict(smp))     # the oracle has no batched IK: the placement is replayed
    monkeypatch.setattr(sb, 'start_fused', lambda *a, **k: None)     # the oracle has no fused step
    monkeypatch.setattr(sb, 'start_coop', lambda *a, **k: None)
    env.reset()
    sim.state_set(G['start_state']); sim.forward_kinematics()
    return env, sim, G, smp


@pytest.mark.parametrize('robot', list(CASES))
def test_per_call_step_reproduces_the_reference_s_rollout(robot, monkeypatch):
    """`ScratchItchEnv.step_reference_api` (take_step, _get_obs, get_total_force, human_preferences through the Agent getters)."""
    env, sim, G, smp = _env_on_oracle(robot, monkeypatch)
    for t, a in enumerate(G['actions']):
        obs, rew, done, info = env.step_reference_api(a[None])
        assert np.allclose(obs[:29], G['obs'][t][:29], rtol=0, atol=1e-9), (t, np.abs(obs[:29] - G['obs'][t][:29]).max())
        assert abs(obs[29] - G['obs'][t][29]) < 1e-6 and abs(info['total_force_on_human'][0] - G['total_force'][t]) < 1e-6      # forces
        assert abs(env.tool_force_at_target[0] - G['force_at_target'][t]) < 1e-6
        assert abs(rew - G['reward'][t]) < 1e-9, (t, rew, G['reward'][t])
        assert bool(done) == bool(G['done'][t]) and int(env.task_success[0]) == int(G['task_success'][t])
    assert G['task_success'][-1] >= 1 and G['reward'].max() > 4                     # the rollout contains counted scratches


@pytest.mark.parametrize('robot', list(CASES))
def test_coop_per_call_step_reproduces_the_reference_s_rollout(robot, monkeypatch):
    """The co-optimisation env's `step` (dict actions and observations, the person's arm inside the realistic joint limits)."""
    env, sim, G, smp = _env_on_oracle(robot + '_coop', monkeypatch)
    hb = env._sb.humans['male' if smp['male'][0] else 'female']
    links = [env._sb.gl(hb, j) for j in RIGHT_ARM_JOINTS]
    for t in range(len(G['reward'])):
        o, r, d, info = env.step({'robot': np.zeros(7), 'human': G['human_action']})
        arm = sim.get_joint_states(links)[0][0]
        assert np.allclose(arm, G['arm_q'][t], rtol=0, atol=1e-7), (t, np.abs(arm - G['arm_q'][t]).max())
        assert np.allclose(o['robot'][:29], G['obs_robot'][t][:29], rtol=0, atol=1e-6) and abs(o['robot'][29] - G['obs_robot'][t][29]) < 1e-4 * (1 + abs(G['obs_robot'][t][29]))
        assert np.allclose(o['human'][:32], G['obs_human'][t][:32], rtol=0, atol=1e-6) and np.allclose(o['human'][32:], G['obs_human'][t][32:], rtol=1e-4, atol=1e-4)
        assert abs(r['robot'] - G['reward'][t]) < 1e-5 and r['robot'] == r['human']
    assert G['sent_back'].any() and G['arm_q'][:, 3].max() < np.deg2rad(130)          # the classifier, not the joint range, ends the motion


def _replay_fused(lib, robot, step):
    G, smp = _load(robot)
    sb = CASES[robot]()
    prod = BatchSim(sb.scene, capi.default_config(residual_threshold=0.0), 1, _lib=lib)
    sb.reset(prod, np.random.default_rng(0), sample=dict(smp))
    prod.state_set(G['start_state'].astype(np.float32)); prod.forward_kinematics()
    sb.start_fused(prod, smp)
    err, rerr, succ, ferr = [], [], [], []
    for t, a in enumerate(G['actions']):
        obs, rew, info = step(prod, a[None].astype(np.float32))
        err.append(np.abs(obs[0, :29] - G['obs'][t][:29]).max()); rerr.append(abs(rew[0] - G['reward'][t])); succ.append(int(info[0, 3]))
        # the tool force (obs[29]) and the total force on the person (info[0]), relative to a 1 % + 1e-3 N bound
        ferr.append(max(abs(obs[0, 29] - G['obs'][t][29]) / (0.01 * abs(G['obs'][t][29]) + 1e-3),
                        abs(info[0, 0] - G['total_force'][t]) / (0.01 * abs(G['total_force'][t]) + 1e-3)))
    prod.close()
    err, rerr, ferr = np.array(err), np.array(rerr), np.array(ferr)
    print('%s fused replay: max |obs error| steps 0-3 %.2e, all %.2e; max |reward error| %.2e; force error / bound %.2f (peak force %.2f N)'
          % (robot, err[:4].max(), err.max(), rerr.max(), ferr.max(), G['total_force'].max()))
    # ScratchItchJaco's bounds (test_reference_scratch_semantics.py): 1e-5 on the observation, forces within 1 % + 1e-3, 1e-3 on the
    # reward, the same scratches.  These single-agent rollouts need no looser horizon: over their 16 steps the fp32 kernels stay within
    # 2e-6 of the fp64 oracle (host build; 1.2e-6 measured on an H100).
    assert np.array_equal(succ, G['task_success'].astype(int)), (succ, G['task_success'])
    assert G['total_force'].max() > 1 and ferr.max() < 1, ferr                      # the forces compared are not all zero
    assert err.max() < 1e-5 and rerr.max() < 1e-3, (err, rerr)


@pytest.mark.parametrize('robot', list(CASES))
def test_fused_kernel_bodies_replay_the_reference_s_rollout(emu_lib, robot):
    def step(sim, a):
        obs, rew, done, info = sim.scratch_step_host(a)
        return obs, rew, info
    _replay_fused(emu_lib, robot, step)


def _replay_coop(lib, robot, step):
    G, smp = _load(robot + '_coop')
    sb = CASES[robot]()
    sim = BatchSim(sb.scene, capi.default_config(residual_threshold=0.0), 1, _lib=lib)
    sb.reset(sim, np.random.default_rng(0), sample=dict(smp))
    sim.state_set(G['start_state'].astype(np.float32)); sim.forward_kinematics()
    sb.start_fused(sim, smp)
    sb.start_coop(sim, smp)
    links = [sb.gl(sb.humans['male' if smp['male'][0] else 'female'], j) for j in RIGHT_ARM_JOINTS]
    e = {k: [] for k in ('arm', 'obs_robot', 'obs_human', 'force', 'reward')}
    for t in range(len(G['reward'])):
        obs_r, obs_h, rew = step(sim, np.concatenate([np.zeros(7), G['human_action']])[None].astype(np.float32))
        arm = sim.get_joint_states(links)[0][0]
        e['arm'].append(np.abs(arm - G['arm_q'][t]).max()); e['obs_robot'].append(np.abs(obs_r[0, :29] - G['obs_robot'][t][:29]).max())
        e['obs_human'].append(np.abs(obs_h[0, :32] - G['obs_human'][t][:32]).max()); e['reward'].append(abs(rew[0] - G['reward'][t]))
        # forces: the tool force (obs_robot[29]), the total force on the person and the tool force at the target (obs_human[32:34])
        f = np.concatenate([obs_r[0, 29:30], obs_h[0, 32:34]]); fg = np.concatenate([G['obs_robot'][t][29:30], G['obs_human'][t][32:34]])
        e['force'].append((np.abs(f - fg) / (1 + np.abs(fg))).max())
    sim.close()
    e = {k: np.array(v) for k, v in e.items()}
    # the first step at which the person's raised arm touches the robot or the scratcher (the total force on the person turns non-zero)
    touch = G['obs_human'][:, 32] > 0
    k = int(np.argmax(touch)) if touch.any() else len(touch)
    print('%s coop replay, max |error| over steps 0-%d:' % (robot, k - 1), {n: '%.2e' % v[:k].max() for n, v in e.items()},
          'over all %d:' % len(touch), {n: '%.2e' % v.max() for n, v in e.items()}, 'peak force on the person %.2f N' % G['obs_human'][:, 32].max())
    # Until the person's arm touches the robot: test_coop_fused.py's bounds for ScratchItchJacoHuman-v1's golden (3e-6 on the arm and
    # the observations, 1e-4 on the forces, 1e-5 on the reward).  ScratchItchPR2Human-v1's arm never touches the robot and holds them
    # over all 45 steps.  In ScratchItchSawyerHuman-v1 the raised upper arm presses on Sawyer from step 14 (up to 5.6 N on the person),
    # and from then on the arm parts from the fp64 oracle by up to 4.5e-6 rad, the observations by 1.5e-5 and the forces by 1.3e-3 N on
    # the host build (H100: arm 3.8e-6, observations 1.8e-5, forces 1.1e-3 relative, reward 2.2e-5).  The per-call step run on the same fp32 kernels parts at
    # the same step by the same amounts, so the split is fp32 against fp64 contact physics, not the fused step's semantics.
    assert e['arm'][:k].max() < 3e-6 and e['obs_robot'][:k].max() < 3e-6 and e['obs_human'][:k].max() < 3e-6, e
    assert e['force'][:k].max() < 1e-4 and e['reward'][:k].max() < 1e-5, e
    assert e['arm'].max() < 1e-5 and e['obs_robot'].max() < 5e-5 and e['obs_human'].max() < 5e-5, e
    assert e['force'].max() < 5e-3 and e['reward'].max() < 1e-4, e
    assert k == {'sawyer': 14, 'pr2': len(touch)}[robot]


@pytest.mark.parametrize('robot', list(CASES))
def test_coop_kernel_bodies_replay_the_reference_s_rollout(emu_lib, robot):
    def step(sim, a):
        obs_r, obs_h, rew, done, info = sim.coop_step_host(a)
        return obs_r, obs_h, rew
    _replay_coop(emu_lib, robot, step)


@pytest.mark.gpu
@pytest.mark.parametrize('robot', list(CASES))
def test_step_dev_replays_the_reference_s_rollouts_cuda(gpu_lib, robot):
    import torch
    dev = torch.device('cuda:0')
    o, oh = torch.zeros(1, 30, device=dev), torch.zeros(1, 34, device=dev)
    r, d, i = torch.zeros(1, device=dev), torch.zeros(1, device=dev), torch.zeros(1, 4, device=dev)

    def step(sim, a):
        at = torch.as_tensor(a, device=dev).contiguous()
        torch.cuda.synchronize()
        sim.scratch_step_dev(at.data_ptr(), o.data_ptr(), r.data_ptr(), d.data_ptr(), i.data_ptr())
        torch.cuda.synchronize()
        return o.cpu().numpy().astype(np.float64), r.cpu().numpy().astype(np.float64), i.cpu().numpy()

    def coop_step(sim, a):
        at = torch.as_tensor(a, device=dev).contiguous()
        torch.cuda.synchronize()
        sim.coop_step_dev(at.data_ptr(), o.data_ptr(), oh.data_ptr(), r.data_ptr(), d.data_ptr(), i.data_ptr())
        torch.cuda.synchronize()
        return o.cpu().numpy().astype(np.float64), oh.cpu().numpy().astype(np.float64), r.cpu().numpy().astype(np.float64)
    _replay_fused(gpu_lib, robot, step)
    _replay_coop(gpu_lib, robot, coop_step)


def test_pr2_continuous_joint_wraps_past_pi_host_compiled(emu_lib):
    """PR2's left wrist roll (a continuous joint: limits +-1e10) turned past pi: the fused and the per-call step leave it unclamped
    and report it wrapped into [-pi, pi) (scratch_itch.py:64), and agree."""
    pair = [envs.make('ScratchItchPR2-v1', n_envs=2, seed=5) for _ in range(2)]
    for env in pair:
        env._sim_lib = emu_lib
        env.reset()
        sb = env._sb
        assert sb.arm_upper[6] == 1e10
        q = env.id.get_joint_states(sb.arm_links)[0].astype(np.float64)
        q[:, 6] = np.pi - 0.2
        env.id.set_joint_state(sb.arm_links, q=q, qd=np.zeros_like(q))
        env.id.set_motor_targets(sb.arm_links, q)
        env.id.forward_kinematics()
    fused, percall = pair
    a = np.zeros((2, 7), np.float32); a[:, 6] = 1.0
    wrapped = False
    for t in range(6):
        o1 = fused.step(a)[0]
        o2 = percall.step_reference_api(a)[0]
        q = fused.id.get_joint_states([fused._sb.arm_links[6]])[0][:, 0]
        assert np.abs(o1 - o2)[:, :29].max() < 1e-4, (t, np.abs(o1 - o2).max())
        assert np.allclose(o1[:, 19], (q + np.pi) % (2 * np.pi) - np.pi, atol=1e-5)
        wrapped |= bool(np.all(q > np.pi) and np.all(o1[:, 19] < 0))
    for env in pair:
        env.close()
    assert wrapped                                                           # the joint crossed pi and the observation wrapped
