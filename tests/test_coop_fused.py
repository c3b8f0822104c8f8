"""The fused co-optimisation step (ag_coop_*; FeedingJacoHuman-v1 and ScratchItchJacoHuman-v1): the person's half of
`take_step`, `enforce_joint_limits` + the realistic-arm-limit classifier after every substep and the person's observation run
as kernels next to the task's own fused step.

On the CPU (kernel bodies compiled for the host): the reference's own rollouts (tests/golden/*_coop_semantics.npz), the fused
step against the per-call `step` of the same env, and the device classifier against limits_model.  On the H100: the same at
benchmark scale, and the vector env with torch CUDA tensors."""
import os

import numpy as np
import pytest

from assistive_gym_b200 import capi, envs
from assistive_gym_b200.feeding_batch import FeedingBatch
from assistive_gym_b200.limits_model import load_model
from assistive_gym_b200.scratch_itch_batch import RIGHT_ARM_JOINTS, ScratchItchBatch
from assistive_gym_b200.sim import BatchSim

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
HEAD = [20, 21, 22, 23]


def _scratch_golden(lib):
    G = np.load(os.path.join(GOLDEN, 'scratch_coop_semantics.npz'))
    smp = {k[len('sample_'):]: G[k] for k in G.files if k.startswith('sample_')}
    sb = ScratchItchBatch()
    sim = BatchSim(sb.scene, capi.default_config(), 1, _lib=lib)
    sb.reset(sim, np.random.default_rng(0), sample=dict(smp))
    for hb in sb.humans.values():             # ScratchItchEnv.reset: the start pose is clipped to the person's limits
        links = [sb.gl(hb, j) for j in RIGHT_ARM_JOINTS]
        q = sim.get_joint_states(links)[0]
        sim.set_joint_state(links, q=np.clip(q, sb.scene['link_lower'][links], sb.scene['link_upper'][links]))
    sim.forward_kinematics()
    sb.start_fused(sim, smp)
    sb.start_coop(sim, smp)
    links = [sb.gl(sb.humans['male' if smp['male'][0] else 'female'], j) for j in RIGHT_ARM_JOINTS]
    a = np.concatenate([np.zeros(7), G['human_action']])[None]
    err = dict(arm=0.0, obs_robot=0.0, obs_human=0.0, force=0.0, reward=0.0)
    arm = []
    for t in range(len(G['reward'])):
        obs_r, obs_h, rew, done, info = sim.coop_step_host(a)
        arm.append(sim.get_joint_states(links)[0][0])
        err['arm'] = max(err['arm'], np.abs(arm[-1] - G['arm_q'][t]).max())
        err['obs_robot'] = max(err['obs_robot'], np.abs(obs_r[0, :29] - G['obs_robot'][t][:29]).max())
        err['obs_human'] = max(err['obs_human'], np.abs(obs_h[0, :32] - G['obs_human'][t][:32]).max())
        err['force'] = max(err['force'], abs(obs_r[0, 29] - G['obs_robot'][t][29]), np.abs(obs_h[0, 32:] - G['obs_human'][t][32:]).max())
        err['reward'] = max(err['reward'], abs(rew[0] - G['reward'][t]))
    sim.close()
    print('scratch coop golden, max |error| over 45 steps:', {k: '%.2e' % v for k, v in err.items()})
    arm = np.array(arm)
    # The golden comes from the fp64 CPU oracle; the kernel bodies integrate in fp32, which leaves ~1e-6 rad on the arm (the
    # per-call test on the oracle itself holds 1e-7).  Observations and reward keep the per-call test's bounds.
    assert err['arm'] < 3e-6 and err['obs_robot'] < 3e-6 and err['obs_human'] < 3e-6, err
    assert err['force'] < 1e-4 and err['reward'] < 1e-5, err
    assert abs(np.rad2deg(arm[-1, 3]) - 116.5) < 0.5 and np.rad2deg(arm[20, 3]) < 100        # the classifier stops the shoulder


def _feeding_golden(lib):
    G = np.load(os.path.join(GOLDEN, 'feeding_coop_semantics.npz'))
    fb = FeedingBatch()
    sim = BatchSim(fb.scene, capi.default_config(), 1, _lib=lib)
    smp = fb.reset(sim, np.random.default_rng(int(G['seed'])), settle_steps=0, impairment='none', simulate_head=True)
    assert all(np.array_equal(np.asarray(smp[k]), G['sample_' + k]) for k in smp if 'sample_' + k in G.files)
    sim.state_set(G['start_state'])
    fb.start_fused(sim, smp)
    fb.start_coop(sim, smp)
    links = [fb.gl(fb.humans['male' if smp['male'][0] else 'female'], j) for j in HEAD]
    err = dict(head=0.0, obs_robot=0.0, obs_human=0.0, reward=0.0)
    err5 = dict(err)
    head = []
    for t in range(len(G['reward'])):
        obs_r, obs_h, rew, done, info = sim.coop_step_host(np.concatenate([G['robot_actions'][t], G['human_actions'][t]])[None])
        head.append(sim.get_joint_states(links)[0][0])
        e = dict(head=np.abs(head[-1] - G['head_q'][t]).max(), obs_robot=np.abs(obs_r[0] - G['obs_robot'][t]).max(),
                 obs_human=np.abs(obs_h[0] - G['obs_human'][t]).max(), reward=abs(rew[0] - G['reward'][t]))
        for k in err:
            err[k] = max(err[k], e[k])
            if t < 5:
                err5[k] = max(err5[k], e[k])
    sim.close()
    print('feeding coop golden, max |error| over steps 0-4:', {k: '%.2e' % v for k, v in err5.items()},
          'over all 24:', {k: '%.2e' % v for k, v in err.items()})
    head = np.array(head)
    # Steps 0-4 hold the per-call test's bounds (1e-6 on the observations, 1e-5 on the reward).  From step 6 on, the robot's
    # wrist joint (obs_robot[16]) drifts by a few 1e-4 rad from the fp64 oracle: the robot's own fused step (k_feed_pre, the fp32
    # solver), which this path shares with FeedingJaco-v1.  The person's head joints stay within 2e-6 rad throughout.
    assert err5['obs_robot'] < 2e-6 and err5['obs_human'] < 1e-6 and err5['reward'] < 1e-5, err5
    assert err['head'] < 5e-6 and err['obs_robot'] < 2e-3 and err['obs_human'] < 1e-3 and err['reward'] < 1e-3, err
    assert np.abs(head[11] - head[0]).max() > 0.2                             # the head followed the person's action


def _make_env(env_id, n, lib, seed):
    env = envs.make(env_id, n_envs=n, seed=seed)
    env._sim_lib = lib
    batch = env._sb if hasattr(env, '_sb') else env._fb
    sample = batch.sample

    def sample_both_genders_half_limited(*a, **kw):
        s = sample(*a, **kw)
        s['male'][:] = np.arange(n) % 2
        lim = np.arange(n) % 4 < 2                    # the `limits` impairment at scale 0.5 in half of the envs
        s['impairment'] = np.where(lim, 1, s['impairment']).astype(np.int32)
        s['limit_scale'] = np.where(lim, 0.5, s['limit_scale'])
        return s
    batch.sample = sample_both_genders_half_limited
    return env


def _fused_vs_percall(lib, env_id, n, steps, seed=5):
    """Two envs from the same seed: one stepped by `step` (per-call), one by `step_fused`; the same float32 actions."""
    per, fus = _make_env(env_id, n, lib, seed), _make_env(env_id, n, lib, seed)
    o_p, o_f = per.reset(), fus.reset()
    assert all(np.array_equal(o_p[k], o_f[k]) for k in ('robot', 'human'))       # reset is deterministic
    k = fus.action_human_len
    rng = np.random.default_rng(seed)
    d_obs, d_rew = {'robot': [], 'human': []}, []
    for t in range(steps):
        act = {'robot': rng.uniform(-1, 1, size=(n, 7)).astype(np.float32), 'human': rng.uniform(-1, 1, size=(n, k)).astype(np.float32)}
        r_p, r_f = per.step(act), fus.step_fused(act)
        for a, b in zip(r_p, r_f):                    # the same dict shapes and keys
            assert a.keys() == b.keys()
            for key in a:
                if isinstance(a[key], dict):
                    assert a[key].keys() == b[key].keys()
                else:
                    assert np.shape(a[key]) == np.shape(b[key]), key
        assert r_p[2]['__all__'] == r_f[2]['__all__'] and np.array_equal(r_p[2]['robot'], r_f[2]['robot'])
        assert np.array_equal(r_p[3]['robot']['task_success'], r_f[3]['robot']['task_success'])
        for key in ('robot', 'human'):
            d_obs[key].append(np.abs(r_p[0][key] - r_f[0][key]).max(axis=1))
        d_rew.append(np.abs(r_p[1]['robot'] - r_f[1]['robot']))
        assert np.all(r_f[1]['robot'] == r_f[1]['human'])
    per.close(); fus.close()
    d = {k_: np.array(v) for k_, v in d_obs.items()}
    d['reward'] = np.array(d_rew)
    for k_, v in d.items():
        print('%s %s fused - per-call |diff| per env-step: median %.2e  p90 %.2e  max %.2e' % (env_id, k_, np.median(v), np.quantile(v, 0.9), v.max()))
    return d


def _classify(lib, n_env=1):
    env = envs.make('ScratchItchJacoHuman-v1', n_envs=n_env, seed=3)
    env._sim_lib = lib
    env.reset()
    rng = np.random.default_rng(0)
    m = 65536
    two_pi = 2 * np.pi
    x = np.stack([rng.uniform(0, two_pi, m), rng.uniform(0, two_pi, m), rng.uniform(-np.pi, np.pi, m), rng.uniform(0, two_pi, m)], axis=1).astype(np.float32)
    p_dev = env.id.coop_classify(x)
    env.close()
    p_ref = load_model().predict(x)[:, 0]
    dp = np.abs(p_dev.astype(np.float64) - p_ref)
    sure = np.abs(p_ref - 0.5) > 1e-4
    print('classifier: max |dp| %.2e, %d of %d reachable, %d within 1e-4 of 0.5' % (dp.max(), int((p_ref > 0.5).sum()), m, int((~sure).sum())))
    assert dp.max() < 1e-5
    assert np.array_equal((p_dev > 0.5)[sure], (p_ref > 0.5)[sure])
    assert 0.05 < (p_ref > 0.5).mean() < 0.95                                 # the inputs span both classes


def test_coop_scratch_golden_host_compiled(emu_lib):
    _scratch_golden(emu_lib)


def test_coop_feeding_golden_host_compiled(emu_lib):
    _feeding_golden(emu_lib)


@pytest.mark.parametrize('env_id', ['ScratchItchJacoHuman-v1', 'FeedingJacoHuman-v1'])
def test_coop_fused_matches_per_call_host_compiled(emu_lib, env_id):
    d = _fused_vs_percall(emu_lib, env_id, n=8, steps=10)
    assert d['human'].max() < 1e-3 and d['robot'].max() < 1e-3 and d['reward'].max() < 1e-3


def test_coop_classifier_host_compiled(emu_lib):
    _classify(emu_lib)


def test_coop_init_rejects_bad_input(emu_lib):
    sb = ScratchItchBatch()
    sim = BatchSim(sb.scene, capi.default_config(), 2, _lib=emu_lib)
    from assistive_gym_b200.feeding_batch import coop_params, pack_mlp
    P = coop_params(sb.scene, sb.humans, 1, RIGHT_ARM_JOINTS, 0.05)
    with pytest.raises(RuntimeError, match='ag_scratch_init first'):
        sim.coop_init(P)
    sb.start_fused(sim, sb.sample(2, np.random.default_rng(0)))
    w = pack_mlp(P, load_model(), [3, 4, 5, 6], -1.0)
    P.mlp_sizes[2] = 32
    with pytest.raises(RuntimeError, match='4-64-64-64-1'):
        sim.coop_init(P, mlp=w)
    P.mlp_sizes[2] = 64
    P.joint_links_m[0] = P.joint_links_f[0]
    with pytest.raises(RuntimeError, match='bad joint link'):
        sim.coop_init(P, mlp=w)
    P.joint_links_m[0] = P.joint_links_m[1] - 1
    with pytest.raises(RuntimeError, match='limit_scale'):
        sim.coop_init(P, limit_scale=[0.5, 0.0], mlp=w)
    sim.coop_init(P, limit_scale=[0.5, 1.0], mlp=w)
    sim.close()


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', ['ScratchItchJacoHuman-v1', 'FeedingJacoHuman-v1'])
def test_coop_fused_matches_per_call_cuda(gpu_lib, env_id):
    d = _fused_vs_percall(gpu_lib, env_id, n=1024, steps=10)
    # free-running fp32 with contacts: a few envs may part ways; the population must not
    for k in ('robot', 'human'):
        assert np.median(d[k]) < 1e-4 and np.quantile(d[k], 0.9) < 1e-2, k
    assert np.median(d['reward']) < 1e-4 and np.quantile(d['reward'], 0.9) < 1e-2


@pytest.mark.gpu
def test_coop_classifier_cuda(gpu_lib):
    _classify(gpu_lib)


@pytest.mark.gpu
@pytest.mark.parametrize('env_id,obs_dims,q_slice', [('FeedingJacoHuman-v1', (25, 23), slice(10, 14)),
                                                     ('ScratchItchJacoHuman-v1', (30, 34), slice(13, 23))])
def test_coop_vec_env_torch_episode(gpu_lib, env_id, obs_dims, q_slice):
    import torch
    from assistive_gym_b200.vec_env import AssistiveVecEnv
    n = 256
    vec = AssistiveVecEnv('assistive_gym:' + env_id, n_envs=n, device=0, _lib=gpu_lib, double_buffer=True)
    obs = vec.reset()
    assert obs['robot'].shape == (n, obs_dims[0]) and obs['human'].shape == (n, obs_dims[1])
    k = vec.env.action_human_len
    dev = torch.device('cuda:0')
    act = {'robot': torch.zeros(n, 7, device=dev), 'human': torch.ones(n, k, device=dev)}
    q0 = torch.as_tensor(obs['human'][:, q_slice], device=dev)
    for t in range(200):
        o, r, d, info = vec.step(act)
        assert isinstance(o['human'], torch.Tensor) and o['human'].is_cuda and o['robot'].shape == (n, obs_dims[0])
        assert o['human'].shape == (n, obs_dims[1]) and r['robot'].shape == (n,) and r['robot'] is r['human']
        if t == 19:
            moved = (o['human'][:, q_slice] - q0).abs().max(dim=1).values
            print(env_id, 'person joint travel after 20 steps: median %.3f rad' % moved.median().item())
            assert (moved > 0.05).float().mean().item() > 0.9                 # the person's action moves the person
        if t < 199:
            assert not d['__all__'] and 'terminal_observation' not in info['robot']
            assert torch.isfinite(o['robot']).all() and torch.isfinite(o['human']).all() and torch.isfinite(r['robot']).all()
    assert d['__all__'] and bool(d['robot'].all())
    term = info['human']['terminal_observation']
    assert term.shape == (n, obs_dims[1]) and torch.isfinite(term).all() and torch.isfinite(info['robot']['terminal_observation']).all()
    assert o['human'].shape == (n, obs_dims[1]) and not torch.equal(o['human'], term)          # the fresh episode's observation
    o, r, d, info = vec.step(act)                                                                # the swapped-in copy steps
    assert not d['__all__'] and torch.isfinite(o['human']).all()
    vec.close()
