"""BedBathingPR2-v1 and BedBathingPR2Human-v1: BedBathing with PR2's left arm, placed by TOC (bed_bathing_robots_batch.py), on the fused
device step of BedBathingSawyer.

On the CPU: the templates against the reference's own recorded `reset()` (tests/golden/bathing_robots_reset_recipes.json), the
registry, reset quality and replay, and the fused step against the per-call step on the kernel bodies compiled for the host.  On the
H100: the same comparison at 1024 envs, graph replay against direct launches, and 200-step double-buffered vector-env episodes at 4096
envs with torch tensors."""
import json
import os

import numpy as np
import pytest

from assistive_gym_b200 import capi, envs
from assistive_gym_b200.bed_bathing_batch import R_ELBOW, R_WRIST, RIGHT_ARM_JOINTS
from assistive_gym_b200.bed_bathing_robots_batch import PR2, TARGET_EE_POS, BedBathingPR2Batch
from assistive_gym_b200.kinematics import ik_dls, q_from_rpy
from assistive_gym_b200.scene import JOINT_FIXED
from assistive_gym_b200.sim import BatchSim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RECIPES = json.load(open(os.path.join(ROOT, 'tests', 'golden', 'bathing_robots_reset_recipes.json')))
SINGLE, COOP = 'BedBathingPR2-v1', 'BedBathingPR2Human-v1'
_TEMPLATES = {}


def _template(coop):
    if coop not in _TEMPLATES:
        _TEMPLATES[coop] = BedBathingPR2Batch(controllable_person=coop)
    return _TEMPLATES[coop]


def _calls(rec, fn):
    return [c for c in rec['calls'] if c['fn'] == fn]


def _quat_close(a, b, tol=1e-9):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return min(np.abs(a - b).max(), np.abs(a + b).max()) < tol


def press_pad(bb, sim, s, gap=0.005, depth=0.05):
    """The pressed-pad start of BedBathing's semantics tests for PR2 (tests/test_bed_bathing._pressed_pair with the left arm): from
    the TOC start pose, IK (host, at the task's end-effector orientation) puts the wiper `gap` above the middle of the person's right
    forearm, and the arm's motors aim `depth` lower, with gain 0.1 and force 5.  Returns the start and the pressing arm angles and
    the IK errors."""
    n = sim.n
    male = s['male'].astype(bool)
    mid = np.zeros((n, 3))
    for g, hb in bb.humans.items():
        ls = sim.get_link_states([bb.gl(hb, R_ELBOW), bb.gl(hb, R_WRIST)])['pos']
        on = male if g == 'male' else ~male
        mid[on] = 0.5 * (ls[on, 0] + ls[on, 1])
    arm = np.array(PR2['arm']) + 1
    tq = np.tile(q_from_rpy(PR2['ee_orient_rpy']), (n, 1))

    def ik(target, q7):
        qf = np.zeros((n, bb.kin.nl)); qf[:, arm] = q7
        q, pe, oe = ik_dls(bb.kin, bb.base_pos, bb.base_quat, qf, arm, PR2['ee'] + 1, target, tq, bb.arm_lower, bb.arm_upper, iters=300)
        return q[:, arm], np.maximum(pe, oe)
    q_hi, _ = ik(mid + [0, 0, 0.25], np.asarray(s['q7'], dtype=np.float64))
    bb.place_robot(sim, bb.base_pos, bb.base_quat, q_hi)
    d = np.full(n, np.inf)
    for hb in bb.humans.values():
        c, k = sim.closest_points(bb.tool, hb, 1.0, max_pts=32)
        d = np.minimum(d, np.where(np.arange(32)[None, :] < k[:, None], c['distance'], np.inf).min(axis=1))
    h0 = 0.25 - (d - gap)
    q_hi, e_hi = ik(mid + np.stack([0 * h0, 0 * h0, h0], axis=1), q_hi)
    q_lo, e_lo = ik(mid + np.stack([0 * h0, 0 * h0, h0 - depth], axis=1), q_hi)
    bb.place_robot(sim, bb.base_pos, bb.base_quat, q_hi)
    sim.set_motor(bb.arm_links, 1, target=q_lo, kp=[0.1] * 7, kd=[1.0] * 7, max_force=[5.0] * 7)
    return q_hi, q_lo, np.maximum(e_hi, e_lo)


# ------------------------------------------------------------------ registry
def test_registry_resolves_both_ids():
    import assistive_gym
    import assistive_gym.envs as shim_envs
    from assistive_gym_b200.envs import bed_bathing_envs
    for env_id in (SINGLE, COOP):
        cls = getattr(bed_bathing_envs, env_id.split('-')[0] + 'Env')
        assert envs.ENV_REGISTRY[env_id] is cls and assistive_gym.ENV_REGISTRY[env_id] is cls
        assert getattr(shim_envs, env_id.split('-')[0] + 'Env') is cls
    env = envs.make('assistive_gym:' + SINGLE, n_envs=2)
    assert env.action_space.shape == (7,) and env.observation_space.shape == (24,)        # bed_bathing.py:10: 17 + 7
    assert env.robot.controllable_joint_indices == PR2['arm'] and env.robot.left_end_effector == 76
    assert isinstance(env._bb, BedBathingPR2Batch) and not env._bb.controllable_person
    env = envs.make(COOP, n_envs=2)
    assert env.action_space.shape == (17,) and env.action_robot_len == 7 and env.action_human_len == 10
    assert env.obs_robot_len == 24 and env.obs_human_len == 28 and env._bb.controllable_person
    # PR2's 'bed_bathing' constants (reference agents/pr2.py:19-46)
    r = env.robot
    assert r.gripper_pos['bed_bathing'] == [0.2] * 4 and r.tool_pos_offset['bed_bathing'] == [0, 0, 0]
    assert r.tool_orient_offset['bed_bathing'] == [0, 0, 0] and r.toc_base_pos_offset['bed_bathing'] == [-0.1, 0, 0]
    assert r.toc_ee_orient_rpy['bed_bathing'] == [0, 0, 0]
    for k in ('gripper_pos', 'tool_pos_offset', 'tool_orient_offset', 'toc_base_pos_offset'):
        assert PR2[k] == getattr(r, k)['bed_bathing'], k
    assert PR2['ee_orient_rpy'] == r.toc_ee_orient_rpy['bed_bathing']
    for unbuilt in ('BedBathingJaco-v1', 'BedBathingJacoHuman-v1', 'BedBathingBaxter-v1', 'BedBathingStretch-v1', 'BedBathingPanda-v1'):
        with pytest.raises(KeyError):
            envs.make(unbuilt)
        assert unbuilt not in assistive_gym.ENV_REGISTRY
    from assistive_gym_b200.envs.agents.human import Human
    from assistive_gym_b200.envs.agents.robot import Jaco
    from assistive_gym_b200.envs.bed_bathing import BedBathingEnv
    with pytest.raises(KeyError):                      # a robot without a BedBathing scene raises instead of falling back
        BedBathingEnv(robot=Jaco('left'), human=Human(RIGHT_ARM_JOINTS))


# ------------------------------------------------------------------ templates against the reference's recorded reset()
@pytest.mark.parametrize('key', ['bathing_pr2', 'bathing_pr2_coop'])
def test_template_matches_reference_reset_recipe(key):
    rec = RECIPES[key]
    coop = key.endswith('coop')
    bb = _template(coop)
    sc = bb.scene
    loads = {c['args'][0]: c['kw'] for c in _calls(rec, 'loadURDF')}
    # PR2 fixed at its load pose, with the inertias of its file
    assert loads['pr2_no_torso_lift_tall.urdf']['useFixedBase'] == 1 and np.allclose(loads['pr2_no_torso_lift_tall.urdf']['basePosition'], PR2['base_pos'])
    assert np.allclose(sc['base_pos0'][bb.robot], PR2['base_pos']) and PR2['load'] == dict(inertia_from_file=True)
    # the bed where the reference puts it, with lateral friction 5 (bed_bathing.py:117)
    assert np.allclose(loads['bed.urdf']['basePosition'], sc['base_pos0'][bb.bed])
    (bed,) = [int(k) for k, v in rec['bodies'].items() if v == 'bed.urdf']
    assert [c['kw']['lateralFriction'] for c in _calls(rec, 'changeDynamics') if c['args'] == [bed, -1] and 'lateralFriction' in c['kw']] == [5]
    assert sc['link_friction'][int(sc['body_link0'][bb.bed])] == 5
    ref_bb = envs.make('BedBathingSawyer-v1')._bb                    # the bed and the persons are BedBathingSawyer's
    for body in ('plane', 'bed'):
        k0, k1 = getattr(ref_bb, body), getattr(bb, body)
        l0, l1 = int(ref_bb.scene['body_link0'][k0]), int(sc['body_link0'][k1])
        assert np.array_equal(ref_bb.scene['link_friction'][l0], sc['link_friction'][l1])
        assert np.array_equal(ref_bb.scene['base_pos0'][k0], sc['base_pos0'][k1])
    # the wiper on a fixed constraint at the LEFT tool joint (76), with the task's offsets, max force 500
    assert 'wiper.urdf' in loads
    (con,) = _calls(rec, 'createConstraint')
    assert con['args'][1] == PR2['tool_joint'] == 76 and con['args'][2] == rec['tool_body'] and con['args'][4] == 4
    assert np.allclose(con['kw']['parentFramePosition'], bb.tool_pos_offset)
    assert _quat_close(con['kw']['parentFrameOrientation'], bb.tool_quat_offset)
    assert np.array_equal(sc['con_link'][0], [bb.gl(bb.robot, PR2['tool_joint']), int(sc['body_link0'][bb.tool])])
    assert _calls(rec, 'changeConstraint')[0]['kw']['maxForce'] == sc['con_maxforce'][0] == 500
    # gripper: joints, open position, gain and force; set_instantly clips the opening to the joint limits
    (grip,) = [c for c in _calls(rec, 'setJointMotorControlArray') if c['args'][0] == rec['robot_body']]
    assert grip['kw']['jointIndices'] == PR2['gripper'] and np.allclose(grip['kw']['targetPositions'], PR2['gripper_pos'])
    assert np.allclose(grip['kw']['positionGains'], 0.05) and np.allclose(grip['kw']['forces'], 500)
    lo, hi = sc['link_lower'][bb.gripper_links], sc['link_upper'][bb.gripper_links]
    for i, (j, v) in enumerate(zip(PR2['gripper'], PR2['gripper_pos'])):
        assert rec['robot_joint_resets'][str(j)] == pytest.approx(v) and lo[i] <= v <= hi[i]
    # collision filters: the left gripper's links 71-85 against wiper links -1, 0, 1 (tool.py:41-44)
    assert PR2['gripper_collision'] == list(range(71, 86))
    l0 = int(sc['body_link0'][bb.tool])
    tool_links = set(range(l0, l0 + int(sc['body_nlinks'][bb.tool])))
    off = {k for k, on in bb.builder.filter_overrides.items() if not on and tool_links & set(k)}
    assert off == {tuple(sorted((bb.gl(bb.robot, j), bb.gl(bb.tool, tj)))) for j in PR2['gripper_collision'] for tj in (-1, 0, 1)}
    # gravity: off on PR2 (not mobile) and the wiper, -1 on the person (bed_bathing.py:162-166)
    assert rec['motor_gains'] == {'robot': 0.05, 'human': 0.05}
    grav = {c['kw'].get('body'): tuple(c['args']) for c in _calls(rec, 'setGravity') if 'body' in c['kw']}
    assert grav == {rec['robot_body']: (0, 0, 0), rec['tool_body']: (0, 0, 0), rec['human_body']: (0, 0, -1)}
    for body in (bb.robot, bb.tool):
        assert np.all(sc['body_gravity'][body] == 0)
    for hb in bb.humans.values():
        assert np.allclose(sc['body_gravity'][hb], [0, 0, -1])
    # IK goals (bed_bathing.py:145-148): the randomised start pose with the task orientation, then shoulder, elbow, wrist by position
    ik = _calls(rec, 'calculateInverseKinematics')
    assert all(c['args'][1] == PR2['ee'] for c in ik) and len(ik) == 4
    assert np.abs(np.asarray(ik[0]['kw']['targetPosition']) - TARGET_EE_POS).max() <= 0.05 + 1e-12
    assert _quat_close(ik[0]['kw']['targetOrientation'], q_from_rpy(PR2['ee_orient_rpy'])) and all(c['kw']['targetOrientation'] is None for c in ik[1:])
    # the base-pose sampling box and yaw range (robot.py:140-144 with right_side=True, base yaw 0 +- 30 degrees)
    poses = [c['kw'] for c in _calls(rec, 'resetBasePositionAndOrientation') if c['args'][0] == rec['robot_body']]
    assert len(poses) >= 50
    d = np.array([p['pos'] for p in poses]) - (np.array([-0.85, -0.4, 0]) + PR2['toc_base_pos_offset'])
    assert np.all(d[:, 0] <= 0) and np.all(d[:, 0] >= -0.5) and np.all(np.abs(d[:, 1]) <= 0.5) and np.all(d[:, 2] == 0)
    # simulated joints: the left arm and the left gripper; every other joint welded at the angle reset_joints gives it
    l0, nl = int(sc['body_link0'][bb.robot]), int(sc['body_nlinks'][bb.robot])
    live = [j for j in range(nl - 1) if sc['link_jtype'][l0 + 1 + j] != JOINT_FIXED]
    assert sorted(live) == sorted(PR2['arm'] + PR2['gripper'])
    welded = {int(j): v for j, v in rec['robot_joint_resets'].items() if int(j) not in PR2['arm'] + PR2['gripper'] and abs(v) > 0}
    assert welded == pytest.approx({j: v for j, v in PR2['weld_preset'].items() if v != 0})
    assert [PR2['weld_preset'][j] for j in [42, 43, 44, 46, 47, 49, 50]] == [-1.75, 1.25, -1.5, -0.5, -1, 0, -1]
    # DoFs per env: 11 of PR2; 31 with both genders' right arms when the person is controllable
    assert len(live) == 11
    arm_joints = [bb.gl(hb, j) for hb in bb.humans.values() for j in RIGHT_ARM_JOINTS]
    assert np.all(sc['link_jtype'][arm_joints] != JOINT_FIXED) and len(arm_joints) == 20
    for hb in bb.humans.values():                     # the co-optimisation person's right arm keeps its mass; the static one has none
        mass = sum(sc['link_mass'][bb.gl(hb, j)] for j in RIGHT_ARM_JOINTS)
        assert (mass > 1) if coop else (mass == 0)
    assert len(live) + (len(arm_joints) if coop else 0) == (31 if coop else 11)


def test_sawyer_template_and_draws_unchanged_by_the_shared_helpers():
    """BedBathingBatch's template is built by the bed-and-person helper it now shares with PR2; a PR2 scene's persons, bed and plane
    carry the same data as Sawyer's, and both draw the same sample from the same seed."""
    from assistive_gym_b200.bed_bathing_batch import BedBathingBatch
    for coop in (False, True):
        a, b = BedBathingBatch(controllable_person=coop), _template(coop)
        for hb_a, hb_b in zip(a.humans.values(), b.humans.values()):
            la, lb = int(a.scene['body_link0'][hb_a]), int(b.scene['body_link0'][hb_b])
            nl = int(a.scene['body_nlinks'][hb_a])
            for k in ('link_mass', 'link_lower', 'link_upper', 'link_jtype'):
                assert np.array_equal(a.scene[k][la:la + nl], b.scene[k][lb:lb + nl]), k
            assert np.array_equal(a.scene['body_gravity'][hb_a], b.scene['body_gravity'][hb_b])
        assert a.max_targets == b.max_targets and a.cloth_link - int(a.scene['body_link0'][a.tool]) == b.cloth_link - int(b.scene['body_link0'][b.tool])
        sa, sb = a.sample(8, np.random.default_rng(2)), b.sample(8, np.random.default_rng(2))
        assert sa.keys() == sb.keys() and all(np.array_equal(sa[k], sb[k]) for k in sa)


# ------------------------------------------------------------------ reset quality
@pytest.mark.parametrize('coop', [False, True])
def test_toc_reset_quality(emu_lib, coop):
    bb = _template(coop)
    n = 64
    sim = BatchSim(bb.scene, capi.default_config(), n, _lib=emu_lib)
    s = bb.reset(sim, np.random.default_rng(11))
    short = int((bb.goals_reached < 1).sum())
    hit = bb.colliding(sim)
    print('BedBathingPR2 (controllable person %s): start goal missed in %d of %d envs, all four goals reached in %.3f; %d envs left colliding'
          % (coop, short, n, float((bb.goals_reached == 4).mean()), int(hit.sum())))
    assert short == 0, '%d envs miss the start goal' % short
    # the reference, too, keeps a colliding pose after its three rounds (env.py:282-309); `unresolved` counts every one of them
    assert bb.unresolved == int(hit.sum())
    ee = sim.get_link_states([bb.ee_link])['pos'][:, 0]
    assert np.linalg.norm(ee - (TARGET_EE_POS + s['ee_offset']), axis=1).max() < 0.03
    # a replayed sample puts every env back where the search left it, bit for bit
    q7 = sim.get_joint_states(bb.arm_links)[0]
    st = sim.state_get()
    sim2 = BatchSim(bb.scene, sim.cfg, n, _lib=emu_lib)
    bb.reset(sim2, np.random.default_rng(0), sample=s)
    assert np.array_equal(sim2.get_joint_states(bb.arm_links)[0], q7) and np.array_equal(sim2.state_get(), st)
    assert bb.unresolved == int(hit.sum())
    sim2.close()
    sim.step(25)
    cnt, _ = sim.solver_stats()
    print('contacts per env after 25 steps: median %d, max %d of %d' % (int(np.median(cnt)), int(cnt.max()), sim.cfg.max_contacts))
    assert sim.overflow_count() == 0
    sim.close()


# ------------------------------------------------------------------ fused step against the per-call step
def _single_fused_vs_percall(lib, n, steps=10, seed=7):
    a, b = envs.make(SINGLE, n_envs=n, seed=seed), envs.make(SINGLE, n_envs=n, seed=seed)
    a._sim_lib = b._sim_lib = lib
    oa, ob = a.reset(), b.reset()
    assert np.array_equal(oa, ob) and len(set(a.male.tolist())) == 2
    rng = np.random.default_rng(seed)
    d_obs, d_rew = [], []
    for t in range(steps):
        act = rng.uniform(-1, 1, size=(n, 7)).astype(np.float32)
        o1, r1, d1, i1 = a.step(act)
        o2, r2, d2, i2 = b.step_reference_api(act)
        assert np.array_equal(d1, d2) and np.array_equal(i1['task_success'], i2['task_success'])
        d_obs.append(np.abs(o1 - o2).max(axis=1))
        d_rew.append(np.abs(r1 - r2))
    a.close(); b.close()
    d = {'obs': np.array(d_obs), 'reward': np.array(d_rew)}
    for k, v in d.items():
        print('%s %s fused - per-call |diff| per env-step: median %.2e  p90 %.2e  max %.2e' % (SINGLE, k, np.median(v), np.quantile(v, 0.9), v.max()))
    return d


def _coop_env(n, lib, seed):
    """The co-optimisation env with both genders and the `limits` impairment at scale 0.5 in half of the envs."""
    env = envs.make(COOP, n_envs=n, seed=seed)
    env._sim_lib = lib
    sample = env._bb.sample

    def sample_both_genders_half_limited(*a, **kw):
        s = sample(*a, **kw)
        s['male'][:] = np.arange(n) % 2
        lim = np.arange(n) % 4 < 2
        s['impairment'] = np.where(lim, 1, s['impairment']).astype(np.int32)
        s['limit_scale'] = np.where(lim, 0.5, s['limit_scale'])
        return s
    env._bb.sample = sample_both_genders_half_limited
    return env


def _coop_fused_vs_percall(lib, n, steps, seed=5):
    per, fus = _coop_env(n, lib, seed), _coop_env(n, lib, seed)
    o_p, o_f = per.reset(), fus.reset()
    assert all(np.array_equal(o_p[k], o_f[k]) for k in ('robot', 'human'))
    assert set(per.male.tolist()) == {False, True} and set(np.round(per._bb.last_sample['limit_scale'], 6).tolist()) >= {0.5}
    rng = np.random.default_rng(seed)
    d = {'robot': [], 'human': [], 'reward': []}
    nf = {'robot': 23, 'human': 26}                   # the entries from these on are forces (N), compared relative to their size
    for t in range(steps):
        act = {'robot': rng.uniform(-1, 1, size=(n, 7)).astype(np.float32), 'human': rng.uniform(-1, 1, size=(n, 10)).astype(np.float32)}
        r_p, r_f = per.step(act), fus.step_fused(act)
        assert r_p[2]['__all__'] == r_f[2]['__all__'] and np.array_equal(r_p[3]['robot']['task_success'], r_f[3]['robot']['task_success'])
        for k in ('robot', 'human'):
            x, y = r_p[0][k], r_f[0][k]
            d[k].append(np.maximum(np.abs(x[:, :nf[k]] - y[:, :nf[k]]).max(axis=1), (np.abs(x[:, nf[k]:] - y[:, nf[k]:]) / (1 + np.abs(x[:, nf[k]:]))).max(axis=1)))
        d['reward'].append(np.abs(r_p[1]['robot'] - r_f[1]['robot']))
        assert np.all(r_f[1]['robot'] == r_f[1]['human'])
    per.close(); fus.close()
    d = {k: np.array(v) for k, v in d.items()}
    for k, v in d.items():
        print('%s %s fused - per-call |diff| per env-step: median %.2e  p90 %.2e  max %.2e' % (COOP, k, np.median(v), np.quantile(v, 0.9), v.max()))
    return d


def test_single_agent_fused_matches_per_call_host_compiled(emu_lib):
    d = _single_fused_vs_percall(emu_lib, n=8)
    assert np.median(d['obs']) < 1e-6 and np.median(d['reward']) < 1e-6
    assert d['obs'].max() < 1e-3 and d['reward'].max() < 1e-3


def test_coop_fused_matches_per_call_host_compiled(emu_lib):
    d = _coop_fused_vs_percall(emu_lib, n=8, steps=10)
    assert d['human'].max() < 1e-3 and d['robot'].max() < 1e-3 and d['reward'].max() < 1e-3     # test_bathing_coop.py's bounds


def test_pressed_pad_wipes_on_fused_and_per_call_host_compiled(emu_lib):
    """With the pad pressed onto the forearm, the fused step wipes the same targets as the per-call step."""
    n = 8
    pair = [envs.make(SINGLE, n_envs=n, seed=3) for _ in range(2)]
    for env in pair:
        env._sim_lib = emu_lib
        env.reset()
        _q_hi, q_lo, _err = press_pad(env._bb, env.id, env._bb.last_sample)
        env.robot.motor_gains, env.robot.motor_forces = 0.1, 5.0         # the pressing arm of press_pad, for the per-call step's motors
        env.id.forward_kinematics()
    fused, percall = pair
    assert np.array_equal(fused.id.state_get(), percall.id.state_get())
    for t in range(12):
        q = percall.id.get_joint_states(percall._bb.arm_links)[0]
        act = np.clip((q_lo - q) / 0.25, -1, 1).astype(np.float32)      # keep pressing (tests/test_bed_bathing._check_fused_wiping)
        o1, r1, d1, i1 = fused.step(act)
        o2, r2, d2, i2 = percall.step_reference_api(act)
        wiped_f, wiped_p = fused.task_success.copy(), percall.task_success.copy()       # targets wiped so far
        assert np.array_equal(wiped_f, wiped_p) and np.array_equal(i1['task_success'], i2['task_success']), (t, wiped_f, wiped_p)
        assert np.abs(o1 - o2)[:, :23].max() < 1e-4
    print('pressed pad: targets wiped per env after 12 steps', wiped_f.tolist())
    assert wiped_f.sum() > 0
    for env in pair:
        env.close()


@pytest.mark.parametrize('env_id', [SINGLE])
def test_vector_envs_host_compiled(emu_lib, env_id):
    """`AssistiveVecEnv` (host path, episode end with the in-step reset) and `AssistiveRLlibVectorEnv`."""
    from assistive_gym_b200.vec_env import AssistiveRLlibVectorEnv
    from tests.test_vec_env import _check_host_path
    _check_host_path(emu_lib, 'assistive_gym:' + env_id, 24)
    v = AssistiveRLlibVectorEnv('assistive_gym:' + env_id, n_envs=2, seed=5, _lib=emu_lib)
    obs = v.vector_reset()
    assert len(obs) == 2 and obs[0].shape == (24,) and v.num_envs == 2
    o, r, d, infos = v.vector_step([v.action_space.sample() for _ in range(2)])
    assert len(o) == 2 and isinstance(r[0], float) and d == [False] * 2
    v.vec.close()


def test_coop_vector_env_host_compiled(emu_lib):
    """`AssistiveVecEnv` with the dict actions of the co-optimisation id."""
    from assistive_gym_b200.vec_env import AssistiveVecEnv
    v = AssistiveVecEnv('assistive_gym:' + COOP, n_envs=2, seed=5, _lib=emu_lib)
    obs = v.reset()
    assert obs['robot'].shape == (2, 24) and obs['human'].shape == (2, 28)
    rng = np.random.default_rng(0)
    for _ in range(2):
        o, r, d, info = v.step({'robot': rng.uniform(-1, 1, (2, 7)).astype(np.float32), 'human': rng.uniform(-1, 1, (2, 10)).astype(np.float32)})
        assert o['robot'].shape == (2, 24) and o['human'].shape == (2, 28)
        assert np.all(np.isfinite(o['robot'])) and np.all(np.isfinite(o['human']))
    v.close()


# ------------------------------------------------------------------ H100
@pytest.mark.gpu
def test_single_agent_fused_matches_per_call_cuda(gpu_lib):
    d = _single_fused_vs_percall(gpu_lib, n=1024)
    for k in ('obs', 'reward'):                      # free-running fp32 with contacts: a few envs may part ways; the population must not
        assert np.median(d[k]) < 1e-4 and np.quantile(d[k], 0.9) < 1e-2, k


@pytest.mark.gpu
def test_coop_fused_matches_per_call_cuda(gpu_lib):
    d = _coop_fused_vs_percall(gpu_lib, n=1024, steps=10)
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
    o, oh = torch.zeros(n, 24, device=dev), torch.zeros(n, 28, device=dev)
    r, d, info = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, 4, device=dev)
    out = []
    for t in range(steps):
        a = (torch.rand((n, k), device=dev, generator=g) * 2 - 1).contiguous()
        torch.cuda.synchronize()
        if coop:
            sim.coop_step_dev(a.data_ptr(), o.data_ptr(), oh.data_ptr(), r.data_ptr(), d.data_ptr(), info.data_ptr())
        else:
            sim.bathing_step_dev(a.data_ptr(), o.data_ptr(), r.data_ptr(), d.data_ptr(), info.data_ptr())
        torch.cuda.synchronize()
        out.append(torch.cat([o, oh, r[:, None], d[:, None], info], dim=1).cpu().numpy())
    env.close()
    return np.array(out)


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', [SINGLE, COOP])
def test_graph_replay_matches_direct_launches_cuda(gpu_lib, env_id, monkeypatch):
    graph = _rollout_dev(env_id)
    monkeypatch.setenv('AG_GRAPH', '0')             # read by ag_create
    direct = _rollout_dev(env_id)
    assert np.all(np.isfinite(graph)) and np.array_equal(graph, direct)


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', [SINGLE, COOP])
def test_vec_env_episode_4096_double_buffered_cuda(gpu_lib, env_id):
    """A 200-step random-action episode at 4096 envs: torch tensors in and out (dict actions for the co-optimisation id), no env
    overflows its contact buffer, and the last step swaps in the standby copy."""
    import time
    import torch
    from assistive_gym_b200.vec_env import AssistiveVecEnv
    n = 4096
    vec = AssistiveVecEnv('assistive_gym:' + env_id, n_envs=n, double_buffer=True)
    coop = env_id == COOP
    t0 = time.perf_counter()
    obs = vec.reset()
    bb = vec.env._bb
    print('%s: first reset %.2f s; start goal missed in %d envs, %d envs left colliding'
          % (env_id, time.perf_counter() - t0, int((np.asarray(bb.goals_reached) < 1).sum()), bb.unresolved))
    if coop:
        assert obs['robot'].shape == (n, 24) and obs['human'].shape == (n, 28)
    else:
        assert obs.shape == (n, 24) and np.all(np.isfinite(obs))
    assert vec.env.id.overflow_count() == 0
    first = vec.env
    dev = torch.device('cuda:0')
    g = torch.Generator(device='cuda').manual_seed(0)
    cmax = 0
    for t in range(200):
        if t == 199:                                  # the last step auto-resets onto the standby copy
            cnt, _ = first.id.solver_stats()
            cmax = max(cmax, int(cnt.max()))
            print('%s: contacts per env at step 199: median %d, max %d of %d; overflowed envs %d'
                  % (env_id, int(np.median(cnt)), int(cnt.max()), first.id.cfg.max_contacts, first.id.overflow_count()))
            assert first.id.overflow_count() == 0
        a = torch.rand((n, 7), device=dev, generator=g) * 2 - 1
        if coop:
            a = {'robot': a, 'human': torch.rand((n, 10), device=dev, generator=g) * 2 - 1}
        o, r, d, info = vec.step(a)
        if coop:
            assert isinstance(o['human'], torch.Tensor) and o['human'].is_cuda and r['robot'] is r['human']
            assert bool(torch.isfinite(o['robot']).all()) and bool(torch.isfinite(o['human']).all()) and bool(torch.isfinite(r['robot']).all())
        else:
            assert isinstance(o, torch.Tensor) and bool(torch.isfinite(o).all()) and bool(torch.isfinite(r).all())
    if coop:
        assert d['__all__'] and torch.isfinite(info['human']['terminal_observation']).all()
    else:
        assert bool(d.all()) and 'terminal_observation' in info and bool(torch.isfinite(info['terminal_observation']).all())
    assert vec.env is not first and vec.env.id.overflow_count() == 0
    vec.close()


def test_sawyer_only_helpers_refuse_a_pr2_scene(emu_lib):
    """BedBathingBatch's IK, tool placement, hover pose and reset read Sawyer's joint table; on the PR2 scene they raise instead of
    moving the wrong joints."""
    bb = _template(False)
    sim = BatchSim(bb.scene, capi.default_config(), 1, _lib=emu_lib)
    s = bb.reset(sim, np.random.default_rng(1))
    for call in (lambda: bb.solve_ik(bb.base_pos, bb.base_quat, np.zeros((1, 3)), np.random.default_rng(0)),
                 lambda: bb.place_tool(sim, bb.base_pos, bb.base_quat, np.zeros((1, bb.kin.nl))),
                 lambda: bb.hover_over_forearm(sim, s, np.random.default_rng(0)),
                 lambda: bb._reset_sawyer(sim, s, np.random.default_rng(0), 6, 50)):
        with pytest.raises(NotImplementedError):
            call()
    sim.close()
