"""DrinkingSawyer-v1 and DrinkingPR2-v1: Drinking with the robots that are not wheelchair-mounted, placed by TOC
(drinking_robots_batch.py), on the fused device step of DrinkingJaco (ag_drinking.cuh).

On the CPU: the templates and the reset against the reference's own recorded `reset()` (tests/golden/drinking_robots_reset_recipes.json),
the registry, TOC reset quality and replay, the fused step against the per-call step on the kernel bodies compiled for the host, and
ASan/UBSan over a DrinkingPR2-v1 reset and a few fused steps.  On the H100: graph replay against direct launches and a 4096-env
double-buffered vector-env episode per id."""
import glob
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from assistive_gym_b200 import envs
from assistive_gym_b200.drinking_batch import N_WATER, WATER_RADIUS
from assistive_gym_b200.drinking_robots_batch import PR2, SAWYER, TARGET_EE_POS, DrinkingPR2Batch, DrinkingSawyerBatch
from assistive_gym_b200.envs.drinking import points_in_cylinder
from assistive_gym_b200.kinematics import q_from_rpy
from assistive_gym_b200.scene import JOINT_FIXED
from assistive_gym_b200.sim import BatchSim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECIPES = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'drinking_robots_reset_recipes.json')))
IDS = ['DrinkingSawyer-v1', 'DrinkingPR2-v1']
BATCH = {'drinking_sawyer': (DrinkingSawyerBatch, SAWYER, 'sawyer.urdf'), 'drinking_pr2': (DrinkingPR2Batch, PR2, 'pr2_no_torso_lift_tall.urdf')}
GRID = np.array([[i * 2 * WATER_RADIUS - 0.02, j * 2 * WATER_RADIUS - 0.02, k * 2 * WATER_RADIUS + 0.075]
                 for i in range(4) for j in range(4) for k in range(4)])          # drinking.py:159-168
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


def _in_cup(env):
    top, bottom, _ = env._cup_centres()
    sc = env.id.scene
    wp = env.id.get_link_states([int(sc['body_link0'][w.body]) for w in env.water_agents])['pos'].astype(np.float64)
    return points_in_cylinder(top, bottom, 0.05, wp).sum(axis=1)


# ------------------------------------------------------------------ registry
def test_registry_resolves_the_two_ids():
    import assistive_gym
    import assistive_gym.envs as shim_envs
    from assistive_gym_b200.envs import drinking_envs
    for env_id in IDS:
        cls = getattr(drinking_envs, env_id.split('-')[0] + 'Env')
        assert envs.ENV_REGISTRY[env_id] is cls and assistive_gym.ENV_REGISTRY[env_id] is cls
        assert getattr(shim_envs, env_id.split('-')[0] + 'Env') is cls
    env = envs.make('assistive_gym:DrinkingPR2-v1', n_envs=2)
    assert env.action_space.shape == (7,) and env.observation_space.shape == (25,)       # drinking.py:8: 18 + 7
    assert env.robot.controllable_joint_indices == PR2['arm'] and env.robot.right_end_effector == 54
    assert env.robot.gripper_pos['drinking'] == [0.45] * 4 and env.robot.toc_base_pos_offset['drinking'] == [0.2, 0.2, 0]
    assert env.robot.tool_pos_offset['drinking'] == [-0.01, 0, -0.05] and env.robot.toc_ee_orient_rpy['drinking'] == [0, 0, 0]
    env = envs.make('DrinkingSawyer-v1', n_envs=2)
    assert env.robot.right_end_effector == 19 and env.obs_robot_len == 25
    from assistive_gym_b200.envs.agents.human import Human
    from assistive_gym_b200.envs.agents.robot import Robot
    from assistive_gym_b200.envs.drinking import DrinkingEnv
    with pytest.raises(KeyError):                      # robots without a Drinking scene raise instead of falling back
        DrinkingEnv(robot=Robot('right', [0] * 7, [0] * 7, [], 0, 0, [], [], {}, 0, 0, {}, {}, [], [], {}, {}, False), human=Human([]))
    for unbuilt in ('DrinkingJacoHuman-v1', 'DrinkingSawyerHuman-v1', 'DrinkingPR2Human-v1', 'DrinkingBaxter-v1', 'DrinkingStretch-v1', 'DrinkingPanda-v1'):
        with pytest.raises(KeyError):
            envs.make(unbuilt)
        assert unbuilt not in assistive_gym.ENV_REGISTRY


# ------------------------------------------------------------------ templates against the reference's recorded reset()
@pytest.mark.parametrize('key', list(BATCH))
def test_template_matches_reference_reset_recipe(key, emu_lib):
    rec = RECIPES[key]
    db = _template(key)
    _, R, urdf = BATCH[key]
    sc = db.scene
    loads = {c['args'][0]: c['kw'] for c in _calls(rec, 'loadURDF')}
    # bodies: the robot fixed at its load pose, the plain wheelchair (not mounted), no table and no bowl
    assert loads[urdf]['useFixedBase'] == 1 and np.allclose(loads[urdf]['basePosition'], R['base_pos'])
    assert np.allclose(sc['base_pos0'][db.robot], R['base_pos'])
    assert 'wheelchair.urdf' in loads and 'wheelchair_jaco.urdf' not in loads and 'table_tall.urdf' not in loads and 'bowl.urdf' not in loads
    assert np.allclose(sc['base_pos0'][db.wheelchair], loads['wheelchair.urdf']['basePosition']) and loads['wheelchair.urdf']['useFixedBase'] == 0
    # the cup: the coffee cup mesh at scale 0.045, mass 1, on a fixed constraint at the RIGHT tool joint with the task's offsets
    (cup_shape,) = [c for c in _calls(rec, 'createCollisionShape') if 'cup' in str(c['kw'].get('fileName', ''))]
    assert cup_shape['kw']['meshScale'] == [0.045] * 3
    (cup,) = [c for c in _calls(rec, 'createMultiBody') if c['kw'].get('baseCollisionShapeIndex') == cup_shape['kw']['shape']]
    assert cup['kw']['baseMass'] == 1 and cup['kw']['bodies'] == [rec['tool_body']]
    (con,) = _calls(rec, 'createConstraint')
    assert con['args'][0] == rec['robot_body'] and con['args'][1] == R['tool_joint'] and con['args'][4] == 4
    assert np.allclose(con['kw']['parentFramePosition'], db.tool_pos_offset)
    assert _quat_close(con['kw']['parentFrameOrientation'], db.tool_quat_offset)
    assert np.array_equal(sc['con_link'][0], [db.gl(db.robot, R['tool_joint']), int(sc['body_link0'][db.tool])])
    assert _calls(rec, 'changeConstraint')[0]['kw']['maxForce'] == sc['con_maxforce'][0] == 500
    # gripper: joints, open position, gain and force
    (grip,) = [c for c in _calls(rec, 'setJointMotorControlArray') if c['args'][0] == rec['robot_body']]
    assert grip['kw']['jointIndices'] == R['gripper'] and np.allclose(grip['kw']['targetPositions'], R['gripper_pos'])
    assert np.allclose(grip['kw']['positionGains'], 0.05) and np.allclose(grip['kw']['forces'], 500)
    opened = np.clip(R['gripper_pos'], sc['link_lower'][db.gripper_links], sc['link_upper'][db.gripper_links])
    for j, v in zip(R['gripper'], opened):
        assert rec['robot_joint_resets'][str(j)] == pytest.approx(v)                       # set_instantly=True, clipped to the limits
    # motor gains of drinking.py:130, gravity off for robot, person and cup (drinking.py:152-155)
    assert rec['motor_gains'] == {'robot': 0.005, 'human': 0.005}
    grav = {c['kw'].get('body') for c in _calls(rec, 'setGravity') if c['args'] == [0, 0, 0]}
    assert grav == {rec['robot_body'], rec['human_body'], rec['tool_body']}
    for body in [db.robot, db.tool] + list(db.humans.values()):
        assert np.all(sc['body_gravity'][body] == 0)
    # IK goals (drinking.py:145-147): the cup pose with the task orientation, then the mouth by position, then the mouth with it
    ik = _calls(rec, 'calculateInverseKinematics')
    tq = q_from_rpy(R['ee_orient_rpy'])
    assert all(c['args'][1] == R['ee'] for c in ik) and len(ik) >= 3
    assert np.abs(np.asarray(ik[0]['kw']['targetPosition']) - TARGET_EE_POS).max() <= 0.05 + 1e-12
    assert _quat_close(ik[0]['kw']['targetOrientation'], tq) and ik[1]['kw']['targetOrientation'] is None
    assert np.allclose(ik[2]['kw']['targetPosition'], ik[1]['kw']['targetPosition']) and _quat_close(ik[2]['kw']['targetOrientation'], tq)
    # the base-pose sampling box and yaw range (robot.py:140-144 with right_side=True, base yaw 0 +- 30 degrees)
    poses = [c['kw'] for c in _calls(rec, 'resetBasePositionAndOrientation') if c['args'][0] == rec['robot_body']]
    assert len(poses) >= 50
    base0 = np.array([-0.85, -0.4, 0]) + np.array(R['toc_base_pos_offset'])
    d = np.array([p['pos'] for p in poses]) - base0
    assert np.all(d[:, 0] <= 0) and np.all(d[:, 0] >= -0.5) and np.all(np.abs(d[:, 1]) <= 0.5) and np.all(d[:, 2] == 0)
    # simulated joints: the right arm and the right gripper; every other joint welded at the angle reset_joints gives it
    l0, nl = int(sc['body_link0'][db.robot]), int(sc['body_nlinks'][db.robot])
    live = [j for j in range(nl - 1) if sc['link_jtype'][l0 + 1 + j] != JOINT_FIXED]
    assert sorted(live) == sorted(R['arm'] + R['gripper'])
    welded = {int(j): v for j, v in rec['robot_joint_resets'].items() if int(j) not in R['arm'] + R['gripper'] and abs(v) > 0}
    assert welded == pytest.approx({j: v for j, v in R['weld_preset'].items() if v != 0})
    # 64 water spheres (radius 5 mm, 1 g) on the 4 x 4 x 4 grid over the cup's position, then the 50-step settle
    (water,) = [c for c in _calls(rec, 'createMultiBody') if 'batchPositions' in c['kw']]
    cup_pos = [c['kw']['pos'] for c in _calls(rec, 'resetBasePositionAndOrientation') if c['args'][0] == rec['tool_body']][-1]
    assert water['kw']['baseMass'] == 0.001 and len(water['kw']['bodies']) == N_WATER
    assert np.allclose(np.array(water['kw']['batchPositions']) - cup_pos, GRID, atol=1e-12)
    assert rec['n_step_simulation'] == 50
    # ... which this template puts over the cup's centre of mass
    sim = BatchSim(sc, db.config(), 2, _lib=emu_lib)
    db.reset(sim, np.random.default_rng(3), settle_steps=0)
    sim.forward_kinematics()
    com = sim.get_link_states([int(sc['body_link0'][db.tool])])['com_pos'][:, 0].astype(np.float64)
    wp = sim.get_link_states([int(sc['body_link0'][w]) for w in db.waters])['pos'].astype(np.float64)
    assert np.abs(wp - com[:, None, :] - GRID[None]).max() < 1e-5
    assert np.allclose(sim.get_joint_states(db.gripper_links)[0], opened[None], atol=1e-7)
    sim.close()


@pytest.mark.parametrize('key', list(BATCH))
def test_welded_pose_matches_reset_joints(key):
    """The welded template's forward kinematics equal the unwelded model's at the reference's reset angles."""
    from assistive_gym_b200.kinematics import BodyKinematics
    from assistive_gym_b200.scene import SceneBuilder
    db = _template(key)
    _, R, _ = BATCH[key]
    b = SceneBuilder()
    body = b.load_urdf(R['asset'], base_pos=R['base_pos'], fixed_base=True, **R['load'])
    kin0 = BodyKinematics(b.finalize(), body)
    q = np.zeros((1, kin0.nl))
    for j, v in R['weld_preset'].items():
        q[0, j + 1] = v
    q[0, np.array(R['arm']) + 1] = np.linspace(-0.5, 0.5, 7)
    q1 = np.zeros((1, db.kin.nl))
    q1[0, np.array(R['arm']) + 1] = np.linspace(-0.5, 0.5, 7)
    bp, bq = np.array([R['base_pos']], dtype=np.float64), np.array([[0, 0, 0, 1.0]])
    assert np.abs(kin0.fk(bp, bq, q)[0] - db.kin.fk(bp, bq, q1)[0]).max() < 1e-12


# ------------------------------------------------------------------ reset quality
@pytest.mark.parametrize('env_id', IDS)
def test_toc_reset_quality(emu_lib, env_id):
    n = 64
    env = envs.make(env_id, n_envs=n, seed=11)
    env._sim_lib = emu_lib
    env.reset()
    db, sim = env._db, env.id
    s = db.last_sample
    hit = db.colliding(sim)
    c = _in_cup(env)
    cnt, _ = sim.solver_stats()
    print('%s: TOC reached both start goals in %d of %d envs, all three in %d; %d envs still colliding after three rounds; '
          'in-cup particles after the settle: min %d over the envs not colliding; contacts per env max %d of %d'
          % (env_id, int((db.goals_reached >= 2).sum()), n, int((db.goals_reached == 3).sum()), db.unresolved,
             c[~hit].min(), int(cnt.max()), sim.cfg.max_contacts))
    assert np.all(db.goals_reached >= 2)
    assert db.unresolved == int(hit.sum()) and hit.mean() <= 0.5
    # In a few Sawyer envs the water misses the cup during the settle (3 of 64 at this seed); the share is reported, not hidden
    print('%s: envs not colliding with all 64 particles in the cup: %d of %d' % (env_id, int((c[~hit] == N_WATER).sum()), int((~hit).sum())))
    assert (c[~hit] == N_WATER).mean() >= 0.9
    assert sim.overflow_count() == 0
    env.close()


@pytest.mark.parametrize('key', list(BATCH))
def test_replayed_placement_reproduces_the_search(emu_lib, key):
    """A sample that holds `base_pos`, `base_quat` and `q7` is replayed: the same start state as the search that produced it, without
    drawing from the generator.  The searched start pose puts the end effector at the randomised goal (IK threshold 0.03)."""
    db = _template(key)
    n = 16
    a, b = BatchSim(db.scene, db.config(), n, _lib=emu_lib), BatchSim(db.scene, db.config(), n, _lib=emu_lib)
    s = db.reset(a, np.random.default_rng(5), settle_steps=0)
    ok = s['goals_reached'] >= 2
    ee = a.get_link_states([db.ee_link])['pos'][:, 0]
    assert ok.all() and np.linalg.norm(ee - (TARGET_EE_POS + s['ee_offset']), axis=1).max() < 0.03
    unresolved = db.unresolved
    rng = np.random.default_rng(6)
    s2 = db.reset(b, rng, settle_steps=0, sample=s)
    assert np.array_equal(a.state_get(), b.state_get()) and db.unresolved == unresolved
    assert rng.integers(0, 2 ** 31) == np.random.default_rng(6).integers(0, 2 ** 31)
    for k in ('base_pos', 'base_quat', 'q7'):
        assert np.array_equal(s2[k], s[k])
    a.close(); b.close()


# ------------------------------------------------------------------ fused step against the per-call step
def _make_env(lib, env_id, n, seed):
    env = envs.make(env_id, n_envs=n, seed=seed)
    env._sim_lib = lib
    sample = env._db.sample

    def both_genders(*a, **kw):
        s = sample(*a, **kw)
        s['male'][:] = np.arange(len(s['male'])) % 2
        return s
    env._db.sample = both_genders
    return env


def _fused_vs_percall(lib, env_id, n, steps=10, seed=7, inject=True):
    """Two envs from the same seed, one stepped by `step` (per call), one by `step_fused`, with the same float32 actions; per env the
    two topmost particles are put at the mouth moving up (swallowed) and far from the cup (spilled), as in test_drinking_fused.py."""
    per, fus = _make_env(lib, env_id, n, seed), _make_env(lib, env_id, n, seed)
    o_p, o_f = per.reset(), fus.reset()
    assert np.array_equal(o_p, o_f)
    db = fus._db
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
    print('%s n=%d fused - per-call: obs max %.2e, reward max %.2e; %d swallowed, %d spilled' % (env_id, n, max(d_obs), max(d_rew), swallowed, spilled))
    return np.array(d_obs), np.array(d_rew), swallowed, spilled


@pytest.mark.parametrize('env_id', IDS)
def test_fused_step_matches_per_call_step_host_compiled(emu_lib, env_id):
    d_obs, d_rew, swallowed, spilled = _fused_vs_percall(emu_lib, env_id, 4)
    assert swallowed >= 1 and spilled >= 1
    assert d_obs.max() < 1e-5 and d_rew.max() < 1e-4, (d_obs.max(), d_rew.max())


@pytest.mark.parametrize('env_id', IDS)
def test_fused_step_matches_per_call_step_single_env_host_compiled(emu_lib, env_id):
    """n_envs == 1: the same squeezed shapes, scalar reward and done, scalar info entries"""
    d_obs, d_rew, _, _ = _fused_vs_percall(emu_lib, env_id, 1, inject=False)
    assert d_obs.max() < 1e-5 and d_rew.max() < 1e-4, (d_obs.max(), d_rew.max())


@pytest.mark.parametrize('env_id', IDS)
def test_vector_envs_host_compiled(emu_lib, env_id):
    """`AssistiveVecEnv` (host path, episode end with the in-step reset) and `AssistiveRLlibVectorEnv` dispatch on the task, so the
    new ids run through them unchanged."""
    from assistive_gym_b200.vec_env import AssistiveRLlibVectorEnv
    from tests.test_vec_env import _check_host_path
    _check_host_path(emu_lib, 'assistive_gym:' + env_id, 25)
    v = AssistiveRLlibVectorEnv('assistive_gym:' + env_id, n_envs=2, seed=5, _lib=emu_lib)
    obs = v.vector_reset()
    assert len(obs) == 2 and obs[0].shape == (25,) and v.num_envs == 2
    o, r, d, infos = v.vector_step([v.action_space.sample() for _ in range(2)])
    assert len(o) == 2 and isinstance(r[0], float) and d == [False] * 2 and set(infos[0]) == {'total_force_on_human', 'task_success'}
    v.vec.close()


# ------------------------------------------------------------------ sanitizers
ASAN_WORKLOAD = r'''
import sys
import numpy as np
sys.path.insert(0, sys.argv[2])
from assistive_gym_b200 import capi, envs
lib = capi.load_library(sys.argv[1])
env = envs.make('DrinkingPR2-v1', n_envs=3, seed=4)
env._sim_lib = lib
obs = env.reset()
rng = np.random.default_rng(0)
for t in range(2):
    o, r, d, i = env.step(rng.uniform(-1, 1, (3, 7)).astype(np.float32))
    assert np.all(np.isfinite(o))
for t in range(2):
    o, r, d, i = env.step_fused(rng.uniform(-1, 1, (3, 7)).astype(np.float32))
    assert np.all(np.isfinite(o))
env.close()
print('ASAN-WORKLOAD-OK')
'''


def test_drinking_pr2_is_asan_clean(tmp_path):
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
    r = subprocess.run([sys.executable, str(script), so, ROOT], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and 'ASAN-WORKLOAD-OK' in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
    assert 'AddressSanitizer' not in r.stderr and 'runtime error' not in r.stderr


# ------------------------------------------------------------------ H100
def _graph_rollout(lib, env_id, steps=6, n=4, seed=17):
    env = _make_env(lib, env_id, n, seed)
    env.reset()
    sim = env.id
    rng = np.random.default_rng(seed)
    out = {'obs': [], 'reward': [], 'done': [], 'info': []}
    for _ in range(steps):
        for k, v in zip(('obs', 'reward', 'done', 'info'), sim.drinking_step_host(rng.uniform(-1, 1, size=(n, 7)).astype(np.float32))):
            out[k].append(v)
    out = {k: np.asarray(v) for k, v in out.items()}
    ts, w, wa = sim.drinking_get_state()
    out.update(task_success=ts, waters=w, waters_active=wa, state=sim.state_get())
    env.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', IDS)
def test_graph_replay_matches_direct_launches_cuda(gpu_lib, env_id, monkeypatch):
    graph = _graph_rollout(gpu_lib, env_id)
    monkeypatch.setenv('AG_GRAPH', '0')             # read by ag_create
    direct = _graph_rollout(gpu_lib, env_id)
    for k in graph:
        assert np.all(np.isfinite(graph[k].astype(np.float64))) and np.array_equal(graph[k], direct[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', IDS)
def test_vec_env_episode_4096_double_buffered_cuda(gpu_lib, env_id):
    import time
    import torch
    from assistive_gym_b200.vec_env import AssistiveVecEnv
    n = 4096

    def report(env, label):
        db = env._db
        hit = db.colliding(env.id)
        c = _in_cup(env)
        print('%s %s: TOC reached both start goals in %d of %d envs; %d envs left colliding; in-cup particles after the settle, envs not '
              'colliding: min %d, envs with all 64: %d of %d' % (env_id, label, int((db.goals_reached >= 2).sum()), n, int(hit.sum()),
                                                                c[~hit].min(), int((c[~hit] == N_WATER).sum()), int((~hit).sum())))
        return c, hit

    vec = AssistiveVecEnv('assistive_gym:' + env_id, n_envs=n, double_buffer=True)
    t0 = time.perf_counter()
    obs = vec.reset()
    print('%s: first reset %.2f s' % (env_id, time.perf_counter() - t0))
    assert obs.shape == (n, 25) and np.all(np.isfinite(obs))
    resets = [report(vec.env, 'first reset')]
    assert vec.env.id.overflow_count() == 0
    first = vec.env
    g = torch.Generator(device='cuda').manual_seed(0)
    for t in range(200):
        if t == 199:                                  # the last step auto-resets onto the standby copy
            cnt, it = first.id.solver_stats()
            print('%s: contacts per env at step 199: mean %.1f, max %d of %d; overflowed envs %d'
                  % (env_id, float(cnt.mean()), int(cnt.max()), first.id.cfg.max_contacts, first.id.overflow_count()))
            assert first.id.overflow_count() == 0
        a = torch.rand((n, 7), device='cuda', generator=g) * 2 - 1
        o, r, d, info = vec.step(a)
        assert bool(torch.isfinite(o).all()) and bool(torch.isfinite(r).all())
    assert bool(d.all()) and 'terminal_observation' in info and bool(torch.isfinite(info['terminal_observation']).all())
    assert vec.env is not first
    resets.append(report(vec.env, 'auto-reset'))
    assert vec.env.id.overflow_count() == 0
    o, r, d, info = vec.step(torch.zeros((n, 7), device='cuda'))
    assert bool(torch.isfinite(o).all()) and bool(torch.isfinite(r).all()) and not bool(d.any())
    vec.close()
    for c, hit in resets:
        assert (c[~hit] == N_WATER).mean() >= 0.9 and hit.mean() <= 0.5, np.bincount(c[~hit], minlength=N_WATER + 1)
