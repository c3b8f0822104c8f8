"""The co-optimisation person's `tremor` impairment (human_impairment=...; human.py:80-92, env.py:205-215): the per-call
`take_step` and the fused step's k_coop_pre (ag_coop_set_tremor) accumulate the person's action into each env's
target_joint_angles and drive the controllable joints to target +- amplitude, the sign flipping every env step.

On the CPU (kernel bodies compiled for the host): the reference's own tremor rollouts (tests/golden/*_coop_tremor_semantics.npz) on
the per-call env and on the fused step, the fused step against the per-call `step` with half the envs trembling in each of the
four tasks, the default ids against a pin taken before the keyword existed, the draw statistics, the C ABI's rules and the
sanitizer build on a small tremor workload.  On the H100: the same comparison at 1024 envs, graph replay against direct launches
and a double-buffered vector-env episode with `human_impairment='random'` for one id per task."""
import os
import subprocess
import sys

import numpy as np
import pytest

from assistive_gym_b200 import capi, envs
from assistive_gym_b200.scratch_itch_batch import RIGHT_ARM_JOINTS, ScratchItchBatch
from assistive_gym_b200.sim import BatchSim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden')
ONE_PER_TASK = ['FeedingJacoHuman-v1', 'ScratchItchJacoHuman-v1', 'BedBathingSawyerHuman-v1', 'DressingPR2Human-v1']
KW = {'DressingPR2Human-v1': dict(toc_attempts=6)}


def _make(env_id, n, lib, seed):
    """`env_id` with human_impairment='tremor', then the draw narrowed to half the envs (the rest 'none'); the genders alternate,
    so both trembling genders are covered."""
    env = envs.make(env_id, n_envs=n, seed=seed, human_impairment='tremor', **KW.get(env_id, {}))
    env._sim_lib = lib
    draw = env._person_sample

    def half_trembling(*a):
        s = draw(*a)
        s['male'][:] = np.arange(n) % 2
        on = np.arange(n) % 4 < 2
        s['impairment'] = np.where(on, 3, 0).astype(np.int32)
        s['tremors'] = np.where(on[:, None], s['tremors'], 0.0)
        return s
    env._person_sample = half_trembling
    return env


def _count_restorations(env):
    """per env, how often the per-call classifier put the person's arm back (enforce_realistic_joint_limits)"""
    env.restored = np.zeros(env.n_envs, dtype=int)
    for g, h in env.humans.items():
        call = h.enforce_realistic_joint_limits

        def counted(mask=None, h=h, call=call):
            q0 = np.atleast_2d(h.get_joint_angles(h.controllable_joint_indices)).copy()
            call(mask)
            q1 = np.atleast_2d(h.get_joint_angles(h.controllable_joint_indices))
            env.restored += (np.abs(q1 - q0).max(axis=1) > 0) & np.asarray(mask, dtype=bool)
        h.enforce_realistic_joint_limits = counted


def _fused_vs_percall(lib, env_id, n, steps, seed=5):
    """Two envs from the same seed, half the envs trembling: one stepped by `step` (per-call), one by `step_fused`; the same
    float32 actions.  The person's action is small noise with four joints pushed at full speed (the shoulder and the elbow of an
    arm, the head), in a direction that reaches a pose the classifier rejects within a few steps."""
    per, fus = _make(env_id, n, lib, seed), _make(env_id, n, lib, seed)
    o_p, o_f = per.reset(), fus.reset()
    assert all(np.array_equal(o_p[k], o_f[k]) for k in ('robot', 'human'))
    _count_restorations(per)
    target0 = {g: h.target_joint_angles.copy() for g, h in per.humans.items()}
    k = fus.action_human_len
    rng = np.random.default_rng(seed)
    # the last entry of the robot's observation and the last two of the person's are forces (N), the rest poses and angles
    pose = {'robot': fus.obs_robot_len - 1, 'human': fus.obs_human_len - 2}
    d = {'robot': [], 'human': [], 'force_rel': [], 'reward': []}
    push = np.where((np.arange(n) % 2 == 0)[:, None], [-1.0, -1.0, -1.0, -1.0], [1.0, -1.0, 1.0, -1.0])
    cols = slice(3, 7) if k == 10 else slice(0, 4)
    for t in range(steps):
        human = rng.uniform(-0.2, 0.2, size=(n, k))
        human[:, cols] = push
        act = {'robot': rng.uniform(-1, 1, size=(n, 7)).astype(np.float32), 'human': human.astype(np.float32)}
        r_p, r_f = per.step(act), fus.step_fused(act)
        assert r_p[2]['__all__'] == r_f[2]['__all__'] and np.array_equal(r_p[2]['robot'], r_f[2]['robot'])
        for key, m in pose.items():
            d[key].append(np.abs(r_p[0][key][:, :m] - r_f[0][key][:, :m]).max(axis=1))
        d['force_rel'].append(np.max([(np.abs(r_p[0][key][:, m:] - r_f[0][key][:, m:]) / (1 + np.abs(r_p[0][key][:, m:]))).max(axis=1)
                                      for key, m in pose.items()], axis=0))
        d['reward'].append(np.abs(r_p[1]['robot'] - r_f[1]['robot']))
    trembling = per.humans['male'].tremor_mask | per.humans['female'].tremor_mask
    # the action accumulated into the trembling envs' targets, and only there
    moved = sum(np.abs(h.target_joint_angles - target0[g]).max(axis=1) * h.tremor_mask for g, h in per.humans.items())
    restored = per.restored.copy()
    per.close(); fus.close()
    d = {k_: np.array(v) for k_, v in d.items()}
    for k_, v in d.items():
        print('%s tremor %s fused - per-call |diff| per env-step: median %.2e  p90 %.2e  max %.2e' % (env_id, k_, np.median(v), np.quantile(v, 0.9), v.max()))
    return d, trembling, restored, moved


@pytest.mark.parametrize('env_id', ONE_PER_TASK)
def test_tremor_fused_matches_per_call_host_compiled(emu_lib, env_id):
    n = 8
    d, trembling, restored, moved = _fused_vs_percall(emu_lib, env_id, n=n, steps=10)
    assert trembling.sum() == n // 2 and set(np.arange(n)[trembling] % 2) == {0, 1}          # both genders tremble
    # a pose the classifier puts back while the arm is in contact parts the two paths by a few 1e-3 at most; the gown's
    # contacts at their margin move a force by a fraction (test_dressing_coop.py); the reward carries forces at weight 0.01
    for k in ('robot', 'human'):
        assert np.median(d[k]) < 1e-5 and d[k].max() < 5e-3, k
    assert d['force_rel'].max() < (0.35 if env_id.startswith('Dressing') else 0.2) and d['reward'].max() < 0.02
    if not env_id.startswith('Feeding'):       # a trembling arm the classifier put back
        print(env_id, 'restorations per env', restored.tolist())
        assert (restored[trembling] > 0).any()
    assert (moved[trembling] > 0.05).all() and not moved[~trembling].any()


# ---------------------------------------------------------------------------------------------------------------- the keyword
def _batch(env):
    return getattr(env, next(a for a in ('_fb', '_sb', '_bb', '_db') if hasattr(env, a)))


@pytest.mark.parametrize('env_id', ONE_PER_TASK)
def test_random_draw_statistics(env_id):
    """'random' at 4096 envs: a quarter of the persons tremble, amplitudes inside +-20 deg (the head) or +-10 deg (an arm), a
    tremor person keeps limit_scale = 1 and strength = 1.  The default draw has no tremor, and the keyword leaves every other
    field of the sample as the default draw has it."""
    n = 4096
    env = envs.make(env_id, n_envs=n, human_impairment='random')
    args = ('no_tremor',) if env_id.startswith('Feeding') else ()
    s = env._person_sample(_batch(env), np.random.default_rng(7), *args)
    base = envs.make(env_id, n_envs=n)
    assert base._person_sample(_batch(base), np.random.default_rng(7), *args) is None
    s0 = _batch(base).sample(n, np.random.default_rng(7), *args)
    assert not np.any(s0['impairment'] == 3)
    for k in s0:
        if k not in ('impairment', 'limit_scale', 'strength', 'tremors'):
            assert np.array_equal(s[k], s0[k]), k
    imp = s['impairment']
    counts = np.bincount(imp, minlength=4)
    se = np.sqrt(0.25 * 0.75 / n)
    assert all(abs(c / n - 0.25) < 4 * se for c in counts), counts
    t = imp == 3
    amp = np.deg2rad(20 if env_id.startswith('Feeding') else 10)
    assert s['tremors'].shape == (n, env.action_human_len)
    assert np.all(np.abs(s['tremors'][t]) <= amp) and np.abs(s['tremors'][t]).max() > 0.9 * amp and not s['tremors'][~t].any()
    assert np.all(s['limit_scale'][t] == 1.0) and np.all(s['strength'][t] == 1.0)
    assert np.all((s['limit_scale'][imp == 1] >= 0.5) & (s['limit_scale'][imp == 1] < 1.0))
    assert np.all((s['strength'][imp == 2] >= 0.25) & (s['strength'][imp == 2] < 1.0))


def test_keyword_reaches_every_coop_id_and_is_checked():
    coop = [i for i in envs.ENV_REGISTRY if i.endswith('Human-v1')]
    assert len(coop) == 11
    for env_id in coop:
        assert envs.make(env_id, human_impairment='tremor').human_impairment_coop == 'tremor'
        assert envs.make(env_id).human_impairment_coop is None
    import assistive_gym
    assert assistive_gym.make('assistive_gym:ScratchItchPR2Human-v1', human_impairment='none').human_impairment_coop == 'none'
    with pytest.raises(ValueError, match='must be None'):
        envs.make('FeedingJacoHuman-v1', human_impairment='shaky')
    with pytest.raises(TypeError):
        envs.make('FeedingJaco-v1', human_impairment='tremor')


# ---------------------------------------------------------------------------------------------------------------- the C ABI
def test_coop_set_tremor_rules_host_compiled(emu_lib):
    from assistive_gym_b200.feeding_batch import FeedingBatch, TREMOR_JOINTS, coop_params
    n = 2
    fb = FeedingBatch()
    sim = BatchSim(fb.scene, capi.default_config(), n, _lib=emu_lib)
    s = fb.reset(sim, np.random.default_rng(0), settle_steps=0, impairment='none', simulate_head=True)
    fb.start_fused(sim, s)
    with pytest.raises(RuntimeError, match='ag_coop_init first'):
        sim._ck(sim.lib.ag_coop_set_tremor(sim.h, None, None, None))
    P = coop_params(fb.scene, fb.humans, 0, TREMOR_JOINTS, 0.025)
    sim.coop_init(P)
    on, tgt, amp = np.array([1, 0]), np.zeros((n, 4)), np.full((n, 4), 0.1)
    sim.feeding_set_tremor(on, tgt, amp)                       # the single-agent person's tremor
    with pytest.raises(RuntimeError, match="task's own tremor"):
        sim.coop_set_tremor(on, tgt, amp)
    sim.feeding_set_tremor(np.zeros(n), tgt, amp)
    sim.coop_set_tremor(on, tgt, amp)
    sim.feeding_set_tremor(on, tgt, amp)                       # switched on afterwards: the step refuses
    with pytest.raises(RuntimeError, match='only one of them'):
        sim.coop_step_host(np.zeros((n, 11), np.float32))
    sim.feeding_set_tremor(np.zeros(n), tgt, amp)
    with pytest.raises(RuntimeError, match='bad arguments'):
        sim.coop_set_tremor(on)
    with pytest.raises(RuntimeError, match='finite'):
        sim.coop_set_tremor(on, tgt, np.full((n, 4), np.nan))
    sim.coop_set_tremor(None)                                  # off
    sim.close()


def test_coop_init_switches_tremor_off_host_compiled(emu_lib):
    """a re-armed batch does not inherit the last episode's tremor: after ag_coop_init the step is the one without tremor"""
    from assistive_gym_b200.feeding_batch import FeedingBatch, TREMOR_JOINTS, coop_params
    n = 2
    fb = FeedingBatch()
    out = []
    for arm_tremor in (False, True):
        sim = BatchSim(fb.scene, capi.default_config(), n, _lib=emu_lib)
        s = fb.reset(sim, np.random.default_rng(0), settle_steps=0, impairment='none', simulate_head=True)
        fb.start_fused(sim, s)
        P = coop_params(fb.scene, fb.humans, 0, TREMOR_JOINTS, 0.025)
        sim.coop_init(P)
        if arm_tremor:
            sim.coop_set_tremor([1, 1], fb.tremor_rest_of(s), np.full((n, 4), 0.3))
            sim.coop_init(P)
        out.append(sim.coop_step_host(np.full((n, 11), 0.5, np.float32)))
        sim.close()
    assert all(np.array_equal(a, b) for a, b in zip(*out))


# ---------------------------------------------------------------------------------------------------------------- the default
def test_default_coop_ids_match_the_pin_host_compiled(emu_lib):
    """reset + 10 fused steps of one co-optimisation id per task with default arguments, bit for bit as before the keyword
    existed (tests/golden/make_golden_coop_default_pin.py)"""
    sys.path.insert(0, GOLDEN)
    from make_golden_coop_default_pin import IDS, rollout
    G = np.load(os.path.join(GOLDEN, 'coop_default_pin.npz'))
    for env_id in IDS:
        got = rollout(emu_lib, env_id)
        assert len(got) == sum(k.startswith(env_id + '_') for k in G.files)
        for i, a in enumerate(got):
            assert np.array_equal(np.asarray(a), G['%s_%03d' % (env_id, i)]), (env_id, i)


# ---------------------------------------------------------------------------------------------------------------- sanitizers
ASAN_WORKLOAD = r'''
import sys
import numpy as np
sys.path.insert(0, sys.argv[2])
from assistive_gym_b200 import capi
from tests.test_coop_tremor import _make
lib = capi.load_library(sys.argv[1])
for env_id in ('FeedingJacoHuman-v1', 'ScratchItchJacoHuman-v1'):
    env = _make(env_id, 3, lib, 2)
    env.reset()
    a = {'robot': np.full((3, 7), 0.3, np.float32), 'human': np.full((3, env.action_human_len), 0.7, np.float32)}
    for _ in range(3):
        env.step_fused(a)
    env.id.coop_set_tremor(None)
    env.step_fused(a)
    env.close()
print('ASAN-TREMOR-OK')
'''


def test_tremor_workload_is_asan_clean(tmp_path):
    """the kernel bodies compiled with AddressSanitizer + UBSan (as tests/test_sanitizer.py builds them) on a small tremor
    co-optimisation workload: odd batch, trembling and still envs, the tremor switched off mid-episode"""
    import glob
    asan = sorted(glob.glob('/usr/lib/gcc/x86_64-linux-gnu/*/libasan.so'))
    if not asan:
        pytest.skip('libasan not installed')
    so = str(tmp_path / 'libagphys_asan.so')
    subprocess.check_call(['/usr/bin/g++', '-x', 'c++', '-std=c++17', '-O1', '-g', '-fPIC', '-shared', '-DAG_CPU_EMU', '-fsanitize=address,undefined',
                           '-fno-sanitize-recover=undefined', '-fno-omit-frame-pointer', '-Wno-unused-function', '-o', so,
                           os.path.join(ROOT, 'assistive_gym_b200', 'csrc', 'agphys.cu')])
    ubsan = sorted(glob.glob('/usr/lib/gcc/x86_64-linux-gnu/*/libubsan.so'))
    env = dict(os.environ, LD_PRELOAD=' '.join([asan[-1]] + ubsan[-1:]), ASAN_OPTIONS='detect_leaks=0')
    r = subprocess.run([sys.executable, '-c', ASAN_WORKLOAD, so, ROOT], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and 'ASAN-TREMOR-OK' in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
    assert 'AddressSanitizer' not in r.stderr and 'runtime error' not in r.stderr


# ---------------------------------------------------------------------------------------------------------------- H100
@pytest.mark.gpu
@pytest.mark.parametrize('env_id', ONE_PER_TASK)
def test_tremor_fused_matches_per_call_cuda(gpu_lib, env_id):
    n, steps = (256, 3) if env_id.startswith('Dressing') else (1024, 10)
    d, trembling, restored, moved = _fused_vs_percall(gpu_lib, env_id, n=n, steps=steps)
    assert trembling.sum() == n // 2 and (moved[trembling] > 0.05).all() and not moved[~trembling].any()
    # free-running fp32 with contacts: a few envs may part ways; the population must not
    for k in ('robot', 'human'):
        assert np.median(d[k]) < 1e-4 and np.quantile(d[k], 0.9) < 1e-2, k
        assert np.median(d[k][:, trembling]) < 1e-4, k
    if env_id.startswith('Dressing'):          # the bounds of test_dressing_coop.py: cloth forces enter the reward
        assert np.median(d['force_rel']) < 0.05 and np.median(d['reward']) < 1e-3
    else:
        assert np.median(d['reward']) < 1e-4 and np.quantile(d['reward'], 0.9) < 2e-2


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', ['FeedingJacoHuman-v1', 'ScratchItchJacoHuman-v1'])
def test_tremor_graph_replay_equals_direct_launches_cuda(gpu_lib, env_id, monkeypatch):
    n = 256
    out = []
    for graph in ('1', '0'):
        monkeypatch.setenv('AG_GRAPH', graph)             # read by ag_create
        env = _make(env_id, n, gpu_lib, 9)
        env.reset()
        rng = np.random.default_rng(4)
        res = []
        for _ in range(6):
            r = env.step_fused({'robot': rng.uniform(-1, 1, size=(n, 7)).astype(np.float32),
                                'human': rng.uniform(-1, 1, size=(n, env.action_human_len)).astype(np.float32)})
            res += [r[0]['robot'], r[0]['human'], r[1]['robot']]
        res.append(env.id.state_get())
        env.close()
        out.append(res)
    assert all(np.array_equal(a, b) for a, b in zip(*out))


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', ONE_PER_TASK)
def test_tremor_vec_env_torch_episode_cuda(gpu_lib, env_id):
    """a 200-step double-buffered episode with human_impairment='random', torch tensors in and out"""
    import torch
    from assistive_gym_b200.vec_env import AssistiveVecEnv
    n = 64 if env_id.startswith('Dressing') else 256
    vec = AssistiveVecEnv('assistive_gym:' + env_id, n_envs=n, device=0, _lib=gpu_lib, double_buffer=True, human_impairment='random',
                          **KW.get(env_id, {}))
    vec.reset()
    trembling = vec.env.humans['male'].tremor_mask | vec.env.humans['female'].tremor_mask
    assert 0 < trembling.sum() < n
    dev = torch.device('cuda:0')
    k = vec.env.action_human_len
    act = {'robot': torch.zeros(n, 7, device=dev), 'human': torch.full((n, k), 0.3, device=dev)}
    for t in range(200):
        o, r, d, info = vec.step(act)
        assert isinstance(o['human'], torch.Tensor) and o['human'].is_cuda
        if t < 199:
            assert not d['__all__'] and torch.isfinite(o['robot']).all() and torch.isfinite(o['human']).all() and torch.isfinite(r['robot']).all()
    assert d['__all__'] and torch.isfinite(info['human']['terminal_observation']).all()
    o, r, d, info = vec.step(act)                     # the swapped-in copy steps
    assert not d['__all__'] and torch.isfinite(o['human']).all()
    vec.close()


# ---------------------------------------------------------------------------------------------------------------- the reference's own rollouts
def _clamped(G, actions):
    """per step and joint: the target moved less than frame_skip x 0.05 x the action, i.e. the limit clamp zeroed the action"""
    travel = np.abs(np.diff(np.vstack([G['target0'], G['target_q']]), axis=0))
    return travel < 5 * 0.05 * np.abs(actions) - 1e-9


def _tremor_person(env, G):
    env._person_tremor({'impairment': np.array([3]), 'tremors': G['tremors'][None]}, G['target0'][None])


def _feeding_percall_on_oracle(G):
    from assistive_gym_b200.envs.agents.agent import Agent
    from assistive_gym_b200.envs.agents.furniture import Furniture
    from assistive_gym_b200.feeding_batch import FeedingBatch
    from oracle.oracle_py import OracleSim
    fb = FeedingBatch()
    sim = OracleSim(fb.scene, capi.default_config(), 1)
    smp = fb.reset(sim, np.random.default_rng(int(G['seed'])), settle_steps=25, impairment='none', simulate_head=True)
    assert all(np.array_equal(np.asarray(smp[k]), G['sample_' + k]) for k in smp if 'sample_' + k in G.files)
    sim.state_set(G['start_state']); sim.forward_kinematics()
    env = envs.make('FeedingJacoHuman-v1', n_envs=1)
    env._fb, env.id = fb, sim
    env.plane.init(fb.plane, sim, env.np_random, indices=-1)
    env.robot.init(fb.robot, sim, env.np_random)
    env.tool.init(fb.tool, sim, env.np_random, indices=-1)
    env.furniture.init(fb.wheelchair, sim, env.np_random, indices=-1)
    env.table, env.bowl = Furniture(), Furniture()
    env.table.init(fb.table, sim, env.np_random, indices=-1)
    env.bowl.init(fb.bowl, sim, env.np_random, indices=-1)
    env.male = smp['male'].astype(bool)
    env.robot.motor_gains = env.human.motor_gains = 0.025
    env.humans, env.agents = {}, [env.robot]
    for g, hb in fb.humans.items():
        h = type(env.human)(env.human.controllable_joint_indices, controllable=True)
        h.init(hb, sim, env.np_random, env.human.controllable_joint_indices)
        h.motor_gains, h.motor_forces = 0.025, 1.0
        env.humans[g] = h
        env.agents.append(h)
    _tremor_person(env, G)
    env.foods_agents = []
    for f in fb.foods:
        a = Agent()
        a.init(f, sim, env.np_random, indices=-1)
        env.foods_agents.append(a)
    env.mouth_pos = np.where(env.male[:, None], fb.mouth['male'], fb.mouth['female'])
    env.foods = np.ones((1, 8), dtype=bool); env.foods_active = np.ones((1, 8), dtype=bool)
    env.task_success = np.zeros(1, dtype=int)
    env.iteration = 0
    env.update_targets()
    return env, fb, sim


def test_feeding_tremor_per_call_reproduces_the_reference_s_rollout():
    G = np.load(os.path.join(GOLDEN, 'feeding_coop_tremor_semantics.npz'))
    env, fb, sim = _feeding_percall_on_oracle(G)
    h = env.humans['male' if env.male[0] else 'female']
    links = [fb.gl(h.body, j) for j in h.controllable_joint_indices]
    for t in range(len(G['reward'])):
        o, r, d, info = env.step({'robot': G['robot_actions'][t], 'human': G['human_actions'][t]})
        head = sim.get_joint_states(links)[0][0]
        assert np.allclose(head, G['head_q'][t], rtol=0, atol=1e-7), (t, np.abs(head - G['head_q'][t]).max())
        assert np.allclose(h.target_joint_angles[0], G['target_q'][t], rtol=0, atol=1e-12), t
        assert np.allclose(o['robot'], G['obs_robot'][t], rtol=0, atol=1e-6), (t, np.abs(o['robot'] - G['obs_robot'][t]).max())
        assert np.allclose(o['human'], G['obs_human'][t], rtol=0, atol=1e-6), (t, np.abs(o['human'] - G['obs_human'][t]).max())
        assert abs(r['robot'] - G['reward'][t]) < 1e-5
    assert _clamped(G, G['human_actions']).any()                   # the limit clamp zeroed part of the action
    sim.close()


def test_feeding_tremor_fused_reproduces_the_reference_s_rollout_host_compiled(emu_lib):
    from assistive_gym_b200.feeding_batch import FeedingBatch
    G = np.load(os.path.join(GOLDEN, 'feeding_coop_tremor_semantics.npz'))
    fb = FeedingBatch()
    sim = BatchSim(fb.scene, capi.default_config(), 1, _lib=emu_lib)
    smp = fb.reset(sim, np.random.default_rng(int(G['seed'])), settle_steps=0, impairment='none', simulate_head=True)
    sim.state_set(G['start_state'])
    smp = dict(smp, impairment=np.array([3], np.int32), tremors=G['tremors'][None])
    assert np.array_equal(fb.coop_tremor_target(smp)[0], G['target0'])
    fb.start_fused(sim, smp)
    fb.start_coop(sim, smp)
    links = [fb.gl(fb.humans['male' if smp['male'][0] else 'female'], j) for j in (20, 21, 22, 23)]
    err = dict(head=0.0, obs_robot=0.0, obs_human=0.0, reward=0.0)
    err5 = dict(err)
    for t in range(len(G['reward'])):
        obs_r, obs_h, rew, done, info = sim.coop_step_host(np.concatenate([G['robot_actions'][t], G['human_actions'][t]])[None])
        e = dict(head=np.abs(sim.get_joint_states(links)[0][0] - G['head_q'][t]).max(), obs_robot=np.abs(obs_r[0] - G['obs_robot'][t]).max(),
                 obs_human=np.abs(obs_h[0] - G['obs_human'][t]).max(), reward=abs(rew[0] - G['reward'][t]))
        for k in err:
            err[k] = max(err[k], e[k])
            if t < 5:
                err5[k] = max(err5[k], e[k])
    sim.close()
    print('feeding tremor golden, max |error| over steps 0-4:', {k: '%.2e' % v for k, v in err5.items()}, 'over all:', {k: '%.2e' % v for k, v in err.items()})
    # the bounds of test_coop_fused.py's Feeding replay
    assert err5['obs_robot'] < 2e-6 and err5['obs_human'] < 1e-6 and err5['reward'] < 1e-5, err5
    assert err['head'] < 5e-6 and err['obs_robot'] < 2e-3 and err['obs_human'] < 1e-3 and err['reward'] < 1e-3, err


def _scratch_golden_sample(G):
    return {k[len('sample_'):]: G[k] for k in G.files if k.startswith('sample_')}


def test_scratch_tremor_per_call_reproduces_the_reference_s_rollout():
    from oracle.oracle_py import OracleSim
    G = np.load(os.path.join(GOLDEN, 'scratch_coop_tremor_semantics.npz'))
    sb = ScratchItchBatch()
    sim = OracleSim(sb.scene, capi.default_config(), 1)
    smp = _scratch_golden_sample(G)
    sb.reset(sim, np.random.default_rng(0), sample=smp)
    env = envs.make('ScratchItchJacoHuman-v1', n_envs=1)
    env._sb, env.id = sb, sim
    env.plane.init(sb.plane, sim, env.np_random, indices=-1)
    env.robot.init(sb.robot, sim, env.np_random)
    env.tool.init(sb.tool, sim, env.np_random, indices=-1)
    env.furniture.init(sb.wheelchair, sim, env.np_random, indices=-1)
    env.male = smp['male'].astype(bool)
    env.humans, env.agents = {}, [env.robot]
    for g, hb in sb.humans.items():
        h = type(env.human)(env.human.controllable_joint_indices, controllable=True)
        h.init(hb, sim, env.np_random, env.human.controllable_joint_indices)
        h.env_mask = env.male if g == 'male' else ~env.male
        h.set_limit_scale(np.ones(1))
        env.humans[g] = h
        env.agents.append(h)
    _tremor_person(env, G)
    assert np.array_equal(sb.coop_tremor_target(smp)[0], G['target0'])
    env._limb_links, env._target_local = sb.limb_links(smp), smp['target_local']
    env.prev_target_contact_pos = np.zeros((1, 3))
    env.task_success = np.zeros(1, dtype=int)
    env.iteration = 0
    h = env.humans['male' if env.male[0] else 'female']
    links = [sb.gl(h.body, j) for j in RIGHT_ARM_JOINTS]
    for t in range(len(G['reward'])):
        o, r, d, info = env.step({'robot': np.zeros(7), 'human': G['human_action']})
        arm = sim.get_joint_states(links)[0][0]
        assert np.allclose(arm, G['arm_q'][t], rtol=0, atol=1e-7), (t, np.abs(arm - G['arm_q'][t]).max())
        assert np.allclose(h.target_joint_angles[0], G['target_q'][t], rtol=0, atol=1e-12), t
        assert np.allclose(o['robot'][:29], G['obs_robot'][t][:29], rtol=0, atol=1e-6) and abs(o['robot'][29] - G['obs_robot'][t][29]) < 1e-4 * (1 + abs(G['obs_robot'][t][29]))
        assert np.allclose(o['human'][:32], G['obs_human'][t][:32], rtol=0, atol=1e-6) and np.allclose(o['human'][32:], G['obs_human'][t][32:], rtol=1e-4, atol=1e-4)
        assert abs(r['robot'] - G['reward'][t]) < 1e-5
    assert G['restores'][-1] > 0                                                # the classifier put the trembling arm back
    assert _clamped(G, G['human_action']).any()                                 # the limit clamp zeroed part of the action
    sim.close()


def test_scratch_tremor_fused_reproduces_the_reference_s_rollout_host_compiled(emu_lib):
    G = np.load(os.path.join(GOLDEN, 'scratch_coop_tremor_semantics.npz'))
    smp = _scratch_golden_sample(G)
    sb = ScratchItchBatch()
    sim = BatchSim(sb.scene, capi.default_config(), 1, _lib=emu_lib)
    sb.reset(sim, np.random.default_rng(0), sample=dict(smp))
    sim.forward_kinematics()
    smp = dict(smp, impairment=np.array([3], np.int32), tremors=G['tremors'][None])
    sb.start_fused(sim, smp)
    sb.start_coop(sim, smp)
    links = [sb.gl(sb.humans['male' if smp['male'][0] else 'female'], j) for j in RIGHT_ARM_JOINTS]
    a = np.concatenate([np.zeros(7), G['human_action']])[None]
    err = dict(arm=0.0, obs_robot=0.0, obs_human=0.0, force=0.0, reward=0.0)
    for t in range(len(G['reward'])):
        obs_r, obs_h, rew, done, info = sim.coop_step_host(a)
        err['arm'] = max(err['arm'], np.abs(sim.get_joint_states(links)[0][0] - G['arm_q'][t]).max())
        err['obs_robot'] = max(err['obs_robot'], np.abs(obs_r[0, :29] - G['obs_robot'][t][:29]).max())
        err['obs_human'] = max(err['obs_human'], np.abs(obs_h[0, :32] - G['obs_human'][t][:32]).max())
        err['force'] = max(err['force'], abs(obs_r[0, 29] - G['obs_robot'][t][29]), np.abs(obs_h[0, 32:] - G['obs_human'][t][32:]).max())
        err['reward'] = max(err['reward'], abs(rew[0] - G['reward'][t]))
    sim.close()
    print('scratch tremor golden, max |error| over %d steps:' % len(G['reward']), {k: '%.2e' % v for k, v in err.items()})
    # the bounds of test_coop_fused.py's ScratchItch replay
    assert err['arm'] < 3e-6 and err['obs_robot'] < 3e-6 and err['obs_human'] < 3e-6, err
    assert err['force'] < 1e-4 and err['reward'] < 1e-5, err
