"""ScratchItchSawyer-v1, ScratchItchPR2-v1, ScratchItchSawyerHuman-v1 and ScratchItchPR2Human-v1: ScratchItch with the robots that are
not wheelchair-mounted, placed by TOC (scratch_itch_robots_batch.py), on the fused device step of ScratchItchJaco.

On the CPU: the templates and the reset against the reference's own recorded `reset()` (tests/golden/scratch_robots_reset_recipes.json),
the registry, reset quality, the fused step against the per-call step on the kernel bodies compiled for the host, and ASan/UBSan over a
ScratchItchPR2Human-v1 reset (31 of the 32 DoFs an env may have) and a few fused steps.  On the H100: the same comparison at 1024 envs,
graph replay against direct launches, 4096-env double-buffered vector-env episodes and torch dict episodes for the co-optimisation ids."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from assistive_gym_b200 import capi, envs
from assistive_gym_b200.kinematics import q_from_rpy
from assistive_gym_b200.scene import JOINT_FIXED
from assistive_gym_b200.scratch_itch_robots_batch import PR2, SAWYER, TARGET_EE_POS, ScratchItchPR2Batch, ScratchItchSawyerBatch
from assistive_gym_b200.sim import BatchSim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECIPES = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'scratch_robots_reset_recipes.json')))
SINGLE = ['ScratchItchSawyer-v1', 'ScratchItchPR2-v1']
COOP = ['ScratchItchSawyerHuman-v1', 'ScratchItchPR2Human-v1']
BATCH = {'scratch_sawyer': (ScratchItchSawyerBatch, SAWYER, 'sawyer.urdf'), 'scratch_pr2': (ScratchItchPR2Batch, PR2, 'pr2_no_torso_lift_tall.urdf')}
_TEMPLATES = {}


def _template(key):
    if key not in _TEMPLATES:
        _TEMPLATES[key] = BATCH[key][0]()
    return _TEMPLATES[key]


def _calls(rec, fn):
    return [c for c in rec['calls'] if c['fn'] == fn]


def _quat_close(a, b, tol=1e-9):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return min(np.abs(a - b).max(), np.abs(a + b).max()) < tol


# ------------------------------------------------------------------ registry
def test_registry_resolves_the_four_ids():
    import assistive_gym
    import assistive_gym.envs as shim_envs
    from assistive_gym_b200.envs import scratch_itch_envs
    for env_id in SINGLE + COOP:
        cls = getattr(scratch_itch_envs, env_id.split('-')[0] + 'Env')
        assert envs.ENV_REGISTRY[env_id] is cls and assistive_gym.ENV_REGISTRY[env_id] is cls
        assert getattr(shim_envs, env_id.split('-')[0] + 'Env') is cls
    env = envs.make('assistive_gym:ScratchItchPR2-v1', n_envs=2)
    assert env.action_space.shape == (7,) and env.observation_space.shape == (30,)       # scratch_itch.py:8: 23 + 7
    assert env.robot.controllable_joint_indices == PR2['arm'] and env.robot.left_end_effector == 76
    assert env.robot.gripper_pos['scratch_itch'] == [0.25] * 4 and env.robot.toc_base_pos_offset['scratch_itch'] == [0.1, 0, 0]
    env = envs.make('ScratchItchSawyerHuman-v1', n_envs=2)
    assert env.action_human_len == 10 and env.obs_human_len == 34 and env.obs_robot_len == 30
    from assistive_gym_b200.envs.agents.robot import Robot
    from assistive_gym_b200.envs.scratch_itch import ScratchItchEnv
    from assistive_gym_b200.envs.agents.human import Human
    with pytest.raises(KeyError):                      # robots without a ScratchItch scene raise instead of falling back
        ScratchItchEnv(robot=Robot('left', [0] * 7, [0] * 7, [], 0, 0, [], [], {}, 0, 0, {}, {}, [], [], {}, {}, False), human=Human([]))
    with pytest.raises(KeyError):
        envs.make('ScratchItchBaxter-v1')


# ------------------------------------------------------------------ templates against the reference's recorded reset()
@pytest.mark.parametrize('key', list(BATCH))
def test_template_matches_reference_reset_recipe(key):
    rec = RECIPES[key]
    sb = _template(key)
    _, R, urdf = BATCH[key]
    sc = sb.scene
    loads = {c['args'][0]: c['kw'] for c in _calls(rec, 'loadURDF')}
    # bodies: the robot fixed at its load pose, the plain wheelchair (not mounted) where this scene puts it
    assert loads[urdf]['useFixedBase'] == 1 and np.allclose(loads[urdf]['basePosition'], R['base_pos'])
    assert np.allclose(sc['base_pos0'][sb.robot], R['base_pos'])
    assert 'wheelchair.urdf' in loads and 'wheelchair_jaco.urdf' not in loads
    assert np.allclose(sc['base_pos0'][sb.wheelchair], loads['wheelchair.urdf']['basePosition']) and loads['wheelchair.urdf']['useFixedBase'] == 0
    assert 'tool_scratch.urdf' in loads
    # the scratcher on a fixed constraint at the LEFT tool joint, with the task's offsets, max force 500
    (con,) = _calls(rec, 'createConstraint')
    assert con['args'][1] == R['tool_joint'] and con['args'][4] == 4
    assert np.allclose(con['kw']['parentFramePosition'], sb.tool_pos_offset)
    assert _quat_close(con['kw']['parentFrameOrientation'], sb.tool_quat_offset)
    assert np.array_equal(sc['con_link'][0], [sb.gl(sb.robot, R['tool_joint']), int(sc['body_link0'][sb.tool])])
    assert _calls(rec, 'changeConstraint')[0]['kw']['maxForce'] == sc['con_maxforce'][0] == 500
    # gripper: joints, open position, gain and force
    (grip,) = [c for c in _calls(rec, 'setJointMotorControlArray') if c['args'][0] == rec['robot_body']]
    assert grip['kw']['jointIndices'] == R['gripper'] and np.allclose(grip['kw']['targetPositions'], R['gripper_pos'])
    assert np.allclose(grip['kw']['positionGains'], 0.05) and np.allclose(grip['kw']['forces'], 500)
    for j, v in zip(R['gripper'], R['gripper_pos']):
        assert rec['robot_joint_resets'][str(j)] == pytest.approx(v)                       # set_instantly=True
    # the robot's default motor gains, gravity off for robot, person and scratcher (scratch_itch.py:123-126)
    assert rec['motor_gains'] == {'robot': 0.05, 'human': 0.05}
    grav = {c['kw'].get('body') for c in _calls(rec, 'setGravity') if c['args'] == [0, 0, 0]}
    assert grav == {rec['robot_body'], rec['human_body'], rec['tool_body']}
    for body in [sb.robot, sb.tool] + list(sb.humans.values()):
        assert np.all(sc['body_gravity'][body] == 0)
    # IK goals (scratch_itch.py:114-116): the randomised end-effector pose with the task orientation, then shoulder, elbow, wrist by position
    ik = _calls(rec, 'calculateInverseKinematics')
    tq = q_from_rpy(R['ee_orient_rpy'])
    assert all(c['args'][1] == R['ee'] for c in ik) and len(ik) == 4
    assert np.abs(np.asarray(ik[0]['kw']['targetPosition']) - TARGET_EE_POS).max() <= 0.05 + 1e-12
    assert _quat_close(ik[0]['kw']['targetOrientation'], tq) and all(c['kw']['targetOrientation'] is None for c in ik[1:])
    # the base-pose sampling box and yaw range (robot.py:140-144 with right_side=True, base yaw 0 +- 30 degrees)
    poses = [c['kw'] for c in _calls(rec, 'resetBasePositionAndOrientation') if c['args'][0] == rec['robot_body']]
    assert len(poses) >= 50
    base0 = np.array([-0.85, -0.4, 0]) + np.array(R['toc_base_pos_offset'])
    d = np.array([p['pos'] for p in poses]) - base0
    assert np.all(d[:, 0] <= 0) and np.all(d[:, 0] >= -0.5) and np.all(np.abs(d[:, 1]) <= 0.5) and np.all(d[:, 2] == 0)
    yaw = np.rad2deg(2 * np.arctan2([p['orn'][2] for p in poses], [p['orn'][3] for p in poses]))
    assert np.all(np.abs(yaw) <= 30 + 1e-9) and yaw.std() > 5
    # simulated joints: the left arm and the left gripper; every other joint welded at the angle reset_joints gives it
    l0, nl = int(sc['body_link0'][sb.robot]), int(sc['body_nlinks'][sb.robot])
    live = [j for j in range(nl - 1) if sc['link_jtype'][l0 + 1 + j] != JOINT_FIXED]
    assert sorted(live) == sorted(R['arm'] + R['gripper'])
    welded = {int(j): v for j, v in rec['robot_joint_resets'].items() if int(j) not in R['arm'] + R['gripper'] and abs(v) > 0}
    assert welded == pytest.approx({j: v for j, v in R['weld_preset'].items() if v != 0})
    # DoFs per env: the robot's simulated joints and both genders' right arms
    assert len(live) + 2 * 10 == {'scratch_sawyer': 29, 'scratch_pr2': 31}[key]


@pytest.mark.parametrize('key', list(BATCH))
def test_welded_pose_matches_reset_joints(key):
    """The welded template's forward kinematics equal the unwelded model's at the reference's reset angles."""
    from assistive_gym_b200.kinematics import BodyKinematics
    from assistive_gym_b200.scene import SceneBuilder
    sb = _template(key)
    _, R, _ = BATCH[key]
    b = SceneBuilder()
    body = b.load_urdf(R['asset'], base_pos=R['base_pos'], fixed_base=True, **R['load'])
    kin0 = BodyKinematics(b.finalize(), body)
    q = np.zeros((1, kin0.nl))
    for j, v in R['weld_preset'].items():
        q[0, j + 1] = v
    q[0, np.array(R['arm']) + 1] = np.linspace(-0.5, 0.5, 7)
    q1 = np.zeros((1, sb.kin.nl))
    q1[0, np.array(R['arm']) + 1] = np.linspace(-0.5, 0.5, 7)
    bp, bq = np.array([R['base_pos']], dtype=np.float64), np.array([[0, 0, 0, 1.0]])
    assert np.abs(kin0.fk(bp, bq, q)[0] - sb.kin.fk(bp, bq, q1)[0]).max() < 1e-12


# ------------------------------------------------------------------ reset quality
@pytest.mark.parametrize('key', list(BATCH))
def test_toc_reset_quality(emu_lib, key):
    sb = _template(key)
    n = 64
    sim = BatchSim(sb.scene, capi.default_config(), n, _lib=emu_lib)
    s = sb.reset(sim, np.random.default_rng(11))
    start = float((sb.goals_reached >= 1).mean())
    hit = sb.colliding(sim)
    print('%s: TOC reached the start goal in %.3f of %d envs, all four goals in %.3f; collision-free starts %.3f'
          % (key, start, n, float((sb.goals_reached == 4).mean()), 1 - float(hit.mean())))
    # the reference, too, keeps a colliding pose after its three rounds (env.py:282-309); `unresolved` reports them
    assert start >= 0.95 and 1 - float(hit.mean()) >= 0.95 and sb.unresolved == int(hit.sum())
    # the start pose puts the end effector at the randomised goal (IK threshold 0.03 of position_robot_toc)
    ok = sb.goals_reached >= 1
    ee = sim.get_link_states([sb.ee_link])['pos'][:, 0]
    assert np.linalg.norm(ee - (TARGET_EE_POS + s['ee_offset']), axis=1)[ok].max() < 0.03
    # a replayed sample puts every env back where the search left it
    q7 = sim.get_joint_states(sb.arm_links)[0]
    sim2 = BatchSim(sb.scene, sim.cfg, n, _lib=emu_lib)
    sb.reset(sim2, np.random.default_rng(0), sample=s)
    assert np.array_equal(sim2.get_joint_states(sb.arm_links)[0], q7) and sb.unresolved == int(hit.sum())
    sim2.close()
    sim.step(25)
    cnt, _ = sim.solver_stats()
    print('%s: contacts per env after 25 steps: median %d, max %d of %d' % (key, int(np.median(cnt)), int(cnt.max()), sim.cfg.max_contacts))
    assert sim.overflow_count() == 0
    sim.close()


def test_feeding_toc_search_unchanged_by_the_shared_placement(emu_lib):
    """FeedingTocBatch now places its robot through the same `TocPlacement` as ScratchItch: its searched placement is what the
    reference's recorded FeedingPR2 rollout was replayed from (tests/golden/feeding_pr2_semantics.npz, seed 5)."""
    from assistive_gym_b200.feeding_robots_batch import FeedingPR2Batch
    G = np.load(os.path.join(ROOT, 'tests', 'golden', 'feeding_pr2_semantics.npz'))
    fb = FeedingPR2Batch()
    sim = BatchSim(fb.scene, fb.config(), 1, _lib=emu_lib)
    s = fb.reset(sim, np.random.default_rng(int(G['seed'])), settle_steps=0, impairment='none')
    sim.close()
    for k in ('base_pos', 'base_quat', 'q7', 'goals_reached'):
        assert np.array_equal(s[k], G['sample_' + k]), k


# ------------------------------------------------------------------ fused step against the per-call step
def _single_fused_vs_percall(lib, env_id, n, steps=10, seed=7):
    a, b = envs.make(env_id, n_envs=n, seed=seed), envs.make(env_id, n_envs=n, seed=seed)
    a._sim_lib = b._sim_lib = lib
    oa, ob = a.reset(), b.reset()
    assert np.array_equal(oa, ob) and len(set(a.male.tolist())) == 2
    rng = np.random.default_rng(seed)
    d_obs, d_rew = [], []
    for t in range(steps):
        act = rng.uniform(-1, 1, size=(n, 7)).astype(np.float32)
        o1, r1, d1, i1 = a.step(act)
        o2, r2, d2, i2 = b.step_reference_api(act)
        assert np.array_equal(d1, d2) and set(i1) >= {'total_force_on_human', 'task_success'}
        assert np.array_equal(i1['task_success'], i2['task_success'])
        d_obs.append(np.abs(o1 - o2).max(axis=1))
        d_rew.append(np.abs(r1 - r2))
    a.close(); b.close()
    d = {'obs': np.array(d_obs), 'reward': np.array(d_rew)}
    for k, v in d.items():
        print('%s %s fused - per-call |diff| per env-step: median %.2e  p90 %.2e  max %.2e' % (env_id, k, np.median(v), np.quantile(v, 0.9), v.max()))
    return d


@pytest.mark.parametrize('env_id', SINGLE)
def test_single_agent_fused_matches_per_call_host_compiled(emu_lib, env_id):
    d = _single_fused_vs_percall(emu_lib, env_id, n=8)
    assert np.median(d['obs']) < 1e-6 and np.median(d['reward']) < 1e-6              # test_coop_fused.py's bounds over ten steps
    assert d['obs'].max() < 1e-3 and d['reward'].max() < 1e-3


@pytest.mark.parametrize('env_id', COOP)
def test_coop_fused_matches_per_call_host_compiled(emu_lib, env_id):
    from tests.test_coop_fused import _fused_vs_percall
    d = _fused_vs_percall(emu_lib, env_id, n=8, steps=10)
    assert d['human'].max() < 1e-3 and d['robot'].max() < 1e-3 and d['reward'].max() < 1e-3      # test_coop_fused.py's bounds


@pytest.mark.parametrize('env_id', COOP)
def test_coop_person_moves_the_arm_host_compiled(emu_lib, env_id):
    env = envs.make(env_id, n_envs=4, seed=2)
    env._sim_lib = emu_lib
    obs = env.reset()
    q0 = obs['human'][:, 13:23].copy()
    for t in range(15):
        obs, r, d, info = env.step_fused({'robot': np.zeros((4, 7), np.float32), 'human': np.ones((4, 10), np.float32)})
    travel = np.abs(obs['human'][:, 13:23] - q0).max(axis=1)
    print(env_id, 'arm travel after 15 steps:', travel)
    assert np.all(travel > 0.05) and np.all(np.isfinite(obs['robot']))
    env.close()


# ------------------------------------------------------------------ sanitizers
ASAN_WORKLOAD = r'''
import sys
import numpy as np
sys.path.insert(0, sys.argv[2])
from assistive_gym_b200 import capi, envs
lib = capi.load_library(sys.argv[1])
env = envs.make('ScratchItchPR2Human-v1', n_envs=3, seed=4)
env._sim_lib = lib
obs = env.reset()
rng = np.random.default_rng(0)
for t in range(3):
    o, r, d, i = env.step_fused({'robot': rng.uniform(-1, 1, (3, 7)).astype(np.float32), 'human': rng.uniform(-1, 1, (3, 10)).astype(np.float32)})
    assert np.all(np.isfinite(o['robot'])) and np.all(np.isfinite(o['human']))
o, r, d, i = env.id.scratch_step_host(rng.uniform(-1, 1, (3, 7)).astype(np.float32))
env.close()
print('ASAN-WORKLOAD-OK')
'''


def test_scratch_pr2_human_is_asan_clean(tmp_path):
    asan = sorted(glob.glob('/usr/lib/gcc/x86_64-linux-gnu/*/libasan.so'))
    if not asan:
        pytest.skip('libasan not installed')
    so = str(tmp_path / 'libagphys_asan.so')
    subprocess.check_call(['/usr/bin/g++', '-x', 'c++', '-std=c++17', '-O1', '-g', '-fPIC', '-shared', '-DAG_CPU_EMU', '-fsanitize=address,undefined', '-fno-sanitize-recover=undefined',
                           '-fno-omit-frame-pointer', '-Wno-unused-function', '-o', so, os.path.join(ROOT, 'assistive_gym_b200', 'csrc', 'agphys.cu')])
    ubsan = sorted(glob.glob('/usr/lib/gcc/x86_64-linux-gnu/*/libubsan.so'))
    script = tmp_path / 'workload.py'
    script.write_text(ASAN_WORKLOAD)
    env = dict(os.environ, LD_PRELOAD=' '.join([asan[-1]] + ubsan[-1:]), ASAN_OPTIONS='detect_leaks=0')
    r = subprocess.run([sys.executable, str(script), so, ROOT], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and 'ASAN-WORKLOAD-OK' in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
    assert 'AddressSanitizer' not in r.stderr and 'runtime error' not in r.stderr


# ------------------------------------------------------------------ H100
@pytest.mark.gpu
@pytest.mark.parametrize('env_id', SINGLE)
def test_single_agent_fused_matches_per_call_cuda(gpu_lib, env_id):
    d = _single_fused_vs_percall(gpu_lib, env_id, n=1024)
    for k in ('obs', 'reward'):                      # free-running fp32 with contacts: a few envs may part ways; the population must not
        assert np.median(d[k]) < 1e-4 and np.quantile(d[k], 0.9) < 1e-2, k


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', COOP)
def test_coop_fused_matches_per_call_cuda(gpu_lib, env_id):
    from tests.test_coop_fused import _fused_vs_percall
    d = _fused_vs_percall(gpu_lib, env_id, n=1024, steps=10)
    for k in ('robot', 'human', 'reward'):
        assert np.median(d[k]) < 1e-4 and np.quantile(d[k], 0.9) < 1e-2, k


def _rollout_dev(env_id, n=64, steps=6):
    import torch
    env = envs.make(env_id, n_envs=n, seed=21)
    env.reset()
    sim = env.id
    dev = torch.device('cuda:0')
    g = torch.Generator(device='cuda').manual_seed(0)
    coop = env.human.controllable
    k = 7 + (10 if coop else 0)
    o, oh = torch.zeros(n, 30, device=dev), torch.zeros(n, 34, device=dev)
    r, d, info = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, 4, device=dev)
    out = []
    for t in range(steps):
        a = (torch.rand((n, k), device=dev, generator=g) * 2 - 1).contiguous()
        torch.cuda.synchronize()
        if coop:
            sim.coop_step_dev(a.data_ptr(), o.data_ptr(), oh.data_ptr(), r.data_ptr(), d.data_ptr(), info.data_ptr())
        else:
            sim.scratch_step_dev(a.data_ptr(), o.data_ptr(), r.data_ptr(), d.data_ptr(), info.data_ptr())
        torch.cuda.synchronize()
        out.append(torch.cat([o, oh, r[:, None], d[:, None], info], dim=1).cpu().numpy())
    env.close()
    return np.array(out)


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', SINGLE + COOP)
def test_graph_replay_matches_direct_launches_cuda(gpu_lib, env_id, monkeypatch):
    graph = _rollout_dev(env_id)
    monkeypatch.setenv('AG_GRAPH', '0')             # read by ag_create
    direct = _rollout_dev(env_id)
    assert np.all(np.isfinite(graph)) and np.array_equal(graph, direct)


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', SINGLE)
def test_vec_env_episode_4096_double_buffered_cuda(gpu_lib, env_id):
    import time
    import torch
    from assistive_gym_b200.vec_env import AssistiveVecEnv
    n = 4096
    vec = AssistiveVecEnv('assistive_gym:' + env_id, n_envs=n, double_buffer=True)
    t0 = time.perf_counter()
    obs = vec.reset()
    sb = vec.env._sb
    print('%s: first reset %.2f s; TOC reached the start goal in %.4f of envs, %d envs left colliding'
          % (env_id, time.perf_counter() - t0, float((sb.goals_reached >= 1).mean()), sb.unresolved))
    assert obs.shape == (n, 30) and np.all(np.isfinite(obs))
    assert vec.env.id.overflow_count() == 0
    first = vec.env
    g = torch.Generator(device='cuda').manual_seed(0)
    for t in range(200):
        if t == 199:                                  # the last step auto-resets onto the standby copy
            cnt, it = first.id.solver_stats()
            print('%s: contacts per env at step 199: median %d, max %d; overflowed envs %d' % (env_id, int(np.median(cnt)), int(cnt.max()), first.id.overflow_count()))
            assert first.id.overflow_count() == 0
        a = torch.rand((n, 7), device='cuda', generator=g) * 2 - 1
        o, r, d, info = vec.step(a)
        assert bool(torch.isfinite(o).all()) and bool(torch.isfinite(r).all())
    assert bool(d.all()) and 'terminal_observation' in info and bool(torch.isfinite(info['terminal_observation']).all())
    assert vec.env is not first and vec.env.id.overflow_count() == 0
    o, r, d, info = vec.step(torch.zeros((n, 7), device='cuda'))
    assert bool(torch.isfinite(o).all()) and bool(torch.isfinite(r).all()) and not bool(d.any())
    vec.close()


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', COOP)
def test_coop_vec_env_torch_episode_cuda(gpu_lib, env_id):
    import torch
    from assistive_gym_b200.vec_env import AssistiveVecEnv
    n = 1024
    vec = AssistiveVecEnv('assistive_gym:' + env_id, n_envs=n, device=0, _lib=gpu_lib)
    obs = vec.reset()
    assert obs['robot'].shape == (n, 30) and obs['human'].shape == (n, 34)
    dev = torch.device('cuda:0')
    g = torch.Generator(device='cuda').manual_seed(0)
    q0 = torch.as_tensor(obs['human'][:, 13:23], device=dev)
    sim = vec.env.id
    for t in range(200):
        act = {'robot': torch.rand((n, 7), device=dev, generator=g) * 2 - 1, 'human': torch.ones(n, 10, device=dev)}
        if t == 199:
            print('%s: overflowed envs at step 199: %d' % (env_id, sim.overflow_count()))
            assert sim.overflow_count() == 0
        o, r, d, info = vec.step(act)
        assert isinstance(o['human'], torch.Tensor) and o['human'].is_cuda and r['robot'] is r['human']
        if t == 19:
            moved = (o['human'][:, 13:23] - q0).abs().max(dim=1).values
            print(env_id, 'person joint travel after 20 steps: median %.3f rad' % moved.median().item())
            assert (moved > 0.05).float().mean().item() > 0.9
        if t < 199:
            assert not d['__all__'] and torch.isfinite(o['robot']).all() and torch.isfinite(o['human']).all() and torch.isfinite(r['robot']).all()
    assert d['__all__'] and torch.isfinite(info['human']['terminal_observation']).all()
    vec.close()
