"""The fused DrinkingJaco-v1 step (ag_drinking.cuh, `ag_drinking_step_*`, `DrinkingEnv.step_fused`, `AssistiveVecEnv`).

On the CPU (kernel bodies compiled for the host): the fused step replays the rollout the reference's own `DrinkingEnv.step` returned
(tests/golden/drinking_semantics.npz: one particle swallowed, one spilled) at the tolerances the per-call path meets on the same
physics; `step_fused` returns what the per-call `step` returns; the device-pointer step equals the host-buffer one; bad input
fails with a message; ASan / UBSan are clean over reset and a few fused steps.
On the H100: the golden replay through `drinking_step_dev`, graph replay against direct launches, and a 4096-env double-buffered
vector-env episode with torch actions."""
import ctypes as C
import glob
import os
import subprocess
import sys

import numpy as np
import pytest

from assistive_gym_b200 import envs
from assistive_gym_b200.drinking_batch import N_WATER, DrinkingBatch
from assistive_gym_b200.feeding_batch import TREMOR_JOINTS, coop_params
from assistive_gym_b200.sim import BatchSim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = np.load(os.path.join(ROOT, 'tests', 'golden', 'drinking_semantics.npz'))
N_GOLDEN_STEPS = 16          # the steps the per-call kernel-body replay checks


def _count(mask):
    return np.array([bin(int(m)).count('1') for m in np.atleast_1d(mask)])


def _golden_sim(lib):
    """one env at the golden start state, the fused step armed"""
    db = DrinkingBatch()
    sim = BatchSim(db.scene, DrinkingBatch.config(), 1, _lib=lib)
    smp = {k[len('sample_'):]: G[k] for k in G.files if k.startswith('sample_')}
    db.reset(sim, np.random.default_rng(0), settle_steps=0, sample=smp)
    sim.state_set(G['start_state'].astype(np.float32)); sim.forward_kinematics()
    db.start_fused(sim, smp)
    return db, sim


def _inject(db, sim, t):
    """the golden's swallowed / spilled particle, placed before step t"""
    for key in ('swallow', 'spill'):
        if t == int(G[key + '_step']):
            w = db.waters[int(G[key + '_water'])]
            sim.set_base_pose(w, G[key + '_pos'][None], np.array([[0, 0, 0, 1.0]]))
            sim.set_base_velocity(w, np.array([[0, 0, float(G['swallow_v0']) if key == 'swallow' else 0.0]]), np.zeros((1, 3)))


def _step_dev_host_buffers(sim, a):
    """`drinking_step_dev` with host buffers (the host-compiled library reads them directly)"""
    n = sim.n
    obs, rew, done, info = np.zeros((n, 25), np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros((n, 4), np.float32)
    a = np.ascontiguousarray(a, dtype=np.float32)
    sim.drinking_step_dev(a.ctypes.data, obs.ctypes.data, rew.ctypes.data, done.ctypes.data, info.ctypes.data)
    return obs, rew, done, info


def _step_dev_torch(sim, a):
    """`drinking_step_dev` with CUDA tensors"""
    import torch
    n = sim.n
    ta = torch.as_tensor(np.ascontiguousarray(a, dtype=np.float32), device='cuda')
    out = (torch.zeros((n, 25), device='cuda'), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda'), torch.zeros((n, 4), device='cuda'))
    torch.cuda.synchronize()
    sim.drinking_step_dev(ta.data_ptr(), *[o.data_ptr() for o in out])
    torch.cuda.synchronize()
    return tuple(o.cpu().numpy() for o in out)


def _golden_replay(lib, step):
    db, sim = _golden_sim(lib)
    for t, a in enumerate(G['actions'][:N_GOLDEN_STEPS]):
        _inject(db, sim, t)
        obs, rew, done, info = step(sim, np.asarray(a, dtype=np.float32)[None])
        ts, w, wa = sim.drinking_get_state()
        assert np.abs(obs[0, :24] - G['obs'][t][:24]).max() < 1e-4 and abs(rew[0] - G['reward'][t]) < 1e-2, (t, rew[0], G['reward'][t])
        assert bool(done[0] > 0.5) == bool(G['done'][t])
        assert int(ts[0]) == int(G['task_success'][t]), (t, ts, G['task_success'][t])
        assert _count(w)[0] == int(G['n_waters'][t]) and _count(wa)[0] == int(G['n_waters_active'][t]), (t, _count(w), _count(wa))
    assert sim.overflow_count() == 0
    sim.close()


def test_golden_replay_host_compiled(emu_lib):
    """the fused step from the golden start, against what the reference's own `DrinkingEnv.step` returned (+10 and -1 steps included)"""
    assert int(G['task_success'][N_GOLDEN_STEPS - 1]) == 1 and G['n_waters'][N_GOLDEN_STEPS - 1] < N_WATER - 1       # both events are covered
    _golden_replay(emu_lib, lambda sim, a: sim.drinking_step_host(a))


def _make_env(lib, n, seed):
    env = envs.make('DrinkingJaco-v1', n_envs=n, seed=seed)
    env._sim_lib = lib
    sample = env._db.sample

    def both_genders(*a, **kw):
        s = sample(*a, **kw)
        s['male'][:] = np.arange(len(s['male'])) % 2
        return s
    env._db.sample = both_genders
    return env


def _fused_vs_percall(lib, n, steps=10, seed=7, inject=True):
    """Two envs from the same seed, one stepped by `step` (per-call), one by `step_fused`, with the same float32 actions.  The
    per-call step accumulates the PD targets in fp64, the fused one in fp32 (as Feeding's does); the last-bit differences grow
    through the water's contacts, so the horizon is the ten steps over which they stay below 1e-5 here."""
    per, fus = _make_env(lib, n, seed), _make_env(lib, n, seed)
    o_p, o_f = per.reset(), fus.reset()
    assert np.array_equal(o_p, o_f)                                   # reset is deterministic
    db = fus._db
    # per env the two topmost particles leave the cup (what stays in it hardly moves): one is put at the mouth moving up against
    # gravity (swallowed), one far from the cup (spilled)
    sc = fus.id.scene
    z = fus.id.get_link_states([int(sc['body_link0'][w]) for w in db.waters])['pos'][:, :, 2]
    top2 = np.argsort(-z, axis=1, kind='stable')[:, :2]
    v0 = 9.81 * 5 * 0.02 / 2
    for env in (per, fus) if inject else ():
        for k in np.unique(top2):
            for col, pos, vz in ((0, np.atleast_2d(env.target_pos), v0), (1, np.ones((n, 3)), 0.0)):
                m = (top2[:, col] == k).astype(np.int32)
                if m.any():
                    env.id.set_base_pose(db.waters[k], pos, np.array([[0, 0, 0, 1.0]] * n), mask=m)
                    env.id.set_base_velocity(db.waters[k], np.array([[0, 0, vz]] * n), np.zeros((n, 3)), mask=m)
    rng = np.random.default_rng(seed)
    d_obs, d_rew = [], []
    for t in range(steps):
        act = rng.uniform(-1, 1, size=(n, 7)).astype(np.float32)
        r_p, r_f = per.step(act), fus.step_fused(act)
        for a, b in zip(r_p, r_f):
            assert type(a) is type(b) and np.shape(a) == np.shape(b)
        assert r_p[3].keys() == r_f[3].keys()
        for k in r_p[3]:
            assert np.shape(r_p[3][k]) == np.shape(r_f[3][k]), k
            if k == 'total_force_on_human':
                assert np.allclose(r_p[3][k], r_f[3][k], rtol=1e-5, atol=1e-4)
            else:
                assert np.array_equal(r_p[3][k], r_f[3][k]), k
        assert np.array_equal(r_p[2], r_f[2])
        assert np.array_equal(per.waters, fus.waters) and np.array_equal(per.waters_active, fus.waters_active), t
        assert np.array_equal(per.task_success, fus.task_success), t
        d_obs.append(np.abs(np.atleast_2d(r_p[0]) - np.atleast_2d(r_f[0])).max())
        d_rew.append(np.abs(np.asarray(r_p[1]) - np.asarray(r_f[1])).max())
    swallowed, spilled = int(fus.task_success.sum()), int((~fus.waters).sum()) - int(fus.task_success.sum())
    per.close(); fus.close()
    print('n=%d fused - per-call: obs max %.2e, reward max %.2e; %d swallowed, %d spilled' % (n, max(d_obs), max(d_rew), swallowed, spilled))
    return np.array(d_obs), np.array(d_rew), swallowed, spilled


def test_fused_step_matches_per_call_step_host_compiled(emu_lib):
    d_obs, d_rew, swallowed, spilled = _fused_vs_percall(emu_lib, 4)
    assert swallowed >= 1 and spilled >= 1
    assert d_obs.max() < 1e-5 and d_rew.max() < 1e-4, (d_obs.max(), d_rew.max())


def test_fused_step_matches_per_call_step_single_env_host_compiled(emu_lib):
    """n_envs == 1: the same squeezed shapes, scalar reward and done, scalar info entries"""
    d_obs, d_rew, _, _ = _fused_vs_percall(emu_lib, 1, inject=False)
    assert d_obs.max() < 1e-5 and d_rew.max() < 1e-4, (d_obs.max(), d_rew.max())


def test_dev_step_matches_host_step_and_null_info_host_compiled(emu_lib):
    outs = {}
    for mode in ('host', 'dev'):
        db, sim = _golden_sim(emu_lib)
        rows = []
        for t, a in enumerate(G['actions'][:6]):
            _inject(db, sim, t)
            a = np.asarray(a, dtype=np.float32)[None]
            rows.append(sim.drinking_step_host(a) if mode == 'host' else _step_dev_host_buffers(sim, a))
        outs[mode] = [np.stack(x) for x in zip(*rows)] + list(sim.drinking_get_state()) + [sim.state_get()]
        sim.close()
    for h, d in zip(outs['host'], outs['dev']):
        assert np.array_equal(h, d)
    db, sim = _golden_sim(emu_lib)
    a = np.ascontiguousarray(G['actions'][0][None], dtype=np.float32)
    obs, rew, done = np.zeros((1, 25), np.float32), np.zeros(1, np.float32), np.zeros(1, np.float32)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    assert emu_lib.ag_drinking_step_host(sim.h, p(a), p(obs), p(rew), p(done), None) == 0, emu_lib.ag_last_error()
    assert np.array_equal(obs, outs['host'][0][0]) and np.array_equal(rew, outs['host'][1][0])
    sim.close()


def test_bad_input_fails_with_a_message_host_compiled(emu_lib):
    db = DrinkingBatch()
    sim = BatchSim(db.scene, DrinkingBatch.config(), 1, _lib=emu_lib)
    with pytest.raises(RuntimeError, match='ag_drinking_init not called'):
        sim.drinking_step_host(np.zeros((1, 7), np.float32))
    with pytest.raises(RuntimeError, match='ag_drinking_init not called'):
        sim.drinking_get_state()
    P = db.drinking_params()
    P.n_water = 65
    with pytest.raises(RuntimeError, match='1..64 water particles'):
        sim.drinking_init(P, [1])
    P = db.drinking_params()
    P.tool_body = db.scene.n_bodies
    with pytest.raises(RuntimeError, match='bad body'):
        sim.drinking_init(P, [1])
    P = db.drinking_params()
    P.water_body0 = db.scene.n_bodies - 3
    with pytest.raises(RuntimeError, match='bad body'):
        sim.drinking_init(P, [1])
    db.start_fused(sim, {'male': np.array([1])})
    with pytest.raises(RuntimeError, match='drinking co-optimisation id .*is not built'):
        sim.coop_init(coop_params(db.scene, db.humans, 4, TREMOR_JOINTS, 0.025))
    sim.close()


WORKLOAD = r'''
import sys
import numpy as np
sys.path.insert(0, sys.argv[2])
from assistive_gym_b200 import capi
from assistive_gym_b200.drinking_batch import DrinkingBatch
from assistive_gym_b200.sim import BatchSim
lib = capi.load_library(sys.argv[1])
db = DrinkingBatch()
n = 3
sim = BatchSim(db.scene, DrinkingBatch.config(), n, _lib=lib)
rng = np.random.default_rng(3)
s = db.reset(sim, rng, settle_steps=4)
db.start_fused(sim, s)
w = db.waters[0]
sim.set_base_pose(w, np.array([[1.0, 1.0, 1.0]] * n), None)            # a spilled particle
for _ in range(3):
    sim.drinking_step_host(rng.uniform(-1, 1, size=(n, 7)).astype(np.float32))
print(sim.drinking_get_state())
db.start_fused(sim, s)                                                   # re-armed episode
sim.drinking_step_host(np.zeros((n, 7), np.float32))
sim.close()
print('ASAN-WORKLOAD-OK')
'''


def test_fused_drinking_step_is_asan_clean(tmp_path):
    asan = sorted(glob.glob('/usr/lib/gcc/x86_64-linux-gnu/*/libasan.so'))
    if not asan:
        pytest.skip('libasan not installed')
    so = str(tmp_path / 'libagphys_asan.so')
    subprocess.check_call(['/usr/bin/g++', '-x', 'c++', '-std=c++17', '-O1', '-g', '-fPIC', '-shared', '-DAG_CPU_EMU', '-fsanitize=address,undefined', '-fno-sanitize-recover=undefined',
                           '-fno-omit-frame-pointer', '-Wno-unused-function', '-o', so, os.path.join(ROOT, 'assistive_gym_b200', 'csrc', 'agphys.cu')])
    script = tmp_path / 'drinking_workload.py'
    script.write_text(WORKLOAD)
    ubsan = sorted(glob.glob('/usr/lib/gcc/x86_64-linux-gnu/*/libubsan.so'))
    env = dict(os.environ, LD_PRELOAD=' '.join([asan[-1]] + ubsan[-1:]), ASAN_OPTIONS='detect_leaks=0')
    r = subprocess.run([sys.executable, str(script), so, ROOT], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and 'ASAN-WORKLOAD-OK' in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
    assert 'AddressSanitizer' not in r.stderr and 'runtime error' not in r.stderr


# ------------------------------------------------------------------ H100
@pytest.mark.gpu
def test_golden_replay_cuda(gpu_lib):
    _golden_replay(gpu_lib, _step_dev_torch)


def _graph_rollout(lib, steps=6, n=4, seed=17):
    env = _make_env(lib, n, seed)
    env.reset()
    sim = env.id
    rng = np.random.default_rng(seed)
    out = {'obs': [], 'reward': [], 'done': [], 'info': [], 'launches': []}
    for _ in range(steps):
        l0 = sim.kernel_launches()
        r = sim.drinking_step_host(rng.uniform(-1, 1, size=(n, 7)).astype(np.float32))
        out['launches'].append(sim.kernel_launches() - l0)
        for k, v in zip(('obs', 'reward', 'done', 'info'), r):
            out[k].append(v)
    out = {k: np.asarray(v) for k, v in out.items()}
    ts, w, wa = sim.drinking_get_state()
    out.update(task_success=ts, waters=w, waters_active=wa, state=sim.state_get())
    env.close()
    return out


@pytest.mark.gpu
def test_graph_replay_matches_direct_launches_cuda(gpu_lib, emu_lib, monkeypatch):
    graph = _graph_rollout(gpu_lib)
    monkeypatch.setenv('AG_GRAPH', '0')             # read by ag_create
    direct = _graph_rollout(gpu_lib)
    for k in graph:
        assert np.array_equal(graph[k], direct[k]), k
    assert np.array_equal(graph['launches'], _graph_rollout(emu_lib, steps=2)['launches'][[0] * 6])


@pytest.mark.gpu
def test_vec_env_episode_4096_double_buffered_cuda(gpu_lib):
    import torch
    from assistive_gym_b200.envs.drinking import points_in_cylinder
    from assistive_gym_b200.vec_env import AssistiveVecEnv
    n = 4096

    def in_cup(env):
        top, bottom, _ = env._cup_centres()
        sc = env.id.scene
        wp = env.id.get_link_states([int(sc['body_link0'][w.body]) for w in env.water_agents])['pos'].astype(np.float64)
        c = points_in_cylinder(top, bottom, 0.05, wp).sum(axis=1)
        print('in-cup particles after the reset settle: min %d, p1 %d, median %d; envs with >= 56: %d of %d; histogram %s'
              % (c.min(), np.quantile(c, 0.01), np.median(c), int((c >= 56).sum()), len(c), np.bincount(c, minlength=N_WATER + 1)[40:].tolist()))
        return c

    vec = AssistiveVecEnv('assistive_gym:DrinkingJaco-v1', n_envs=n, double_buffer=True)
    obs = vec.reset()
    assert obs.shape == (n, 25) and np.all(np.isfinite(obs))
    counts = [in_cup(vec.env)]
    assert vec.env.id.overflow_count() == 0
    first = vec.env
    g = torch.Generator(device='cuda').manual_seed(0)
    for t in range(200):
        if t == 199:                                  # the last step auto-resets onto the standby copy
            assert first.id.overflow_count() == 0
        a = torch.rand((n, 7), device='cuda', generator=g) * 2 - 1
        o, r, d, info = vec.step(a)
        assert bool(torch.isfinite(o).all()) and bool(torch.isfinite(r).all())
    assert bool(d.all()) and 'terminal_observation' in info and bool(torch.isfinite(info['terminal_observation']).all())
    assert vec.env is not first
    counts.append(in_cup(vec.env))
    assert vec.env.id.overflow_count() == 0
    o, r, d, info = vec.step(torch.zeros((n, 7), device='cuda'))
    assert bool(torch.isfinite(o).all()) and bool(torch.isfinite(r).all())
    vec.close()
    for c in counts:
        assert (c >= 56).mean() >= 0.99, np.bincount(c, minlength=N_WATER + 1)
