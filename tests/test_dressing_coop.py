"""The fused co-optimisation step of DressingPR2Human-v1 (ag_coop_* with task 3): the person's left arm is a second agent inside the
gown; after every stepSimulation k_coop_limits keeps the arm inside its (scaled) limits and the realistic joint limits (classifier
sign +1, the left arm's input mapping), then the gown's anchor follows the end effector.

On the CPU (kernel bodies compiled for the host): the reference's own rollout (tests/golden/dressing_coop_semantics.npz), the fused
step against the per-call `step` of the same env, the left arm's classifier mapping, the single-agent DressingPR2-v1 path against a
pin taken before this id existed, input checks and the env surface.  On the H100: the same comparison at a few hundred envs, a
cloth gravity change after a captured step, and a vector-env episode with torch tensors."""
import os
import sys

import numpy as np
import pytest

from assistive_gym_b200 import capi, envs
from assistive_gym_b200.dressing_batch import L_ARM_LIMIT_JOINTS, LEFT_ARM_JOINTS, DressingBatch
from assistive_gym_b200.feeding_batch import coop_params
from assistive_gym_b200.sim import BatchSim
from tests.test_reference_dressing_coop_semantics import G, golden_sample, settled_start

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
POSE = {'robot': 23, 'human': 26}          # the entries before these are poses and angles, the rest are forces (N)


def test_coop_dressing_golden_host_compiled(emu_lib):
    """ag_coop_step_host from the golden's start against what the reference's own step returned on the fp64 oracle."""
    db = DressingBatch(controllable_person=True)
    prod = BatchSim(db.scene, DressingBatch.config(), 1, _lib=emu_lib)
    settled_start(db, prod)
    smp = golden_sample()
    db.start_fused(prod, smp)
    db.start_coop(prod, smp)
    links = [db.gl(db.humans['male' if smp['male'][0] else 'female'], j) for j in LEFT_ARM_JOINTS]
    err = dict(arm=0.0, obs_robot=0.0, obs_human=0.0, reward=0.0)
    restored = np.flatnonzero(np.diff(np.concatenate([[0], G['restores']])) > 0)
    assert len(restored) >= 1
    for t, a in enumerate(G['actions']):
        obs_r, obs_h, rew, done, info = prod.coop_step_host(a[None].astype(np.float32))
        arm = prod.get_joint_states(links)[0][0]
        err['arm'] = max(err['arm'], np.abs(arm - G['arm_q'][t]).max())
        err['obs_robot'] = max(err['obs_robot'], np.abs(obs_r[0, :POSE['robot']] - G['obs_robot'][t][:POSE['robot']]).max())
        err['obs_human'] = max(err['obs_human'], np.abs(obs_h[0, :POSE['human']] - G['obs_human'][t][:POSE['human']]).max())
        err['reward'] = max(err['reward'], abs(rew[0] - G['reward'][t]))
        # the cloth force sum within the bound of the single-agent Dressing replay (test_reference_dressing_semantics.py)
        for got, want in ((obs_r[0, 23], G['obs_robot'][t][23]), (obs_h[0, 26], G['obs_human'][t][26])):
            assert abs(got - want) < 0.35 * want + 0.5, (t, got, want)
        assert abs(obs_h[0, 27] - G['obs_human'][t][27]) < 0.35 * G['obs_human'][t][27] + 0.5           # robot force on the person
        assert int(info[0, 3]) == int(G['sleeve'][t]) and int(info[0, 1]) == int(G['task_success'][t] >= 0.4), t
        assert bool(done[0]) == bool(G['done'][t])
    prod.close()
    print('dressing coop golden, max |error| over %d steps (restorations at steps %s):' % (len(G['reward']), restored.tolist()),
          {k: '%.2e' % v for k, v in err.items()})
    # the arm at every step, the restoration steps included, as close as the single-agent Dressing replay's observation (1e-5)
    assert err['arm'] < 1e-5 and err['obs_robot'] < 1e-5 and err['obs_human'] < 1e-5, err
    assert err['reward'] < 0.02, err


def _make_env(n, lib, seed):
    env = envs.make('DressingPR2Human-v1', n_envs=n, seed=seed, toc_attempts=6)
    env._sim_lib = lib
    sample = env._db.sample

    def sample_both_genders_half_limited(*a, **kw):
        s = sample(*a, **kw)
        s['male'][:] = np.arange(n) % 2
        lim = np.arange(n) % 4 < 2                    # the `limits` impairment at scale 0.5 in half of the envs
        s['impairment'] = np.where(lim, 1, s['impairment']).astype(np.int32)
        s['limit_scale'] = np.where(lim, 0.5, s['limit_scale'])
        return s
    env._db.sample = sample_both_genders_half_limited
    return env


def _fused_vs_percall(lib, n, steps, seed=5):
    """Two envs from the same seed: one stepped by `step` (per-call), one by `step_fused`; the same float32 actions."""
    per, fus = _make_env(n, lib, seed), _make_env(n, lib, seed)
    o_p, o_f = per.reset(), fus.reset()
    assert all(np.array_equal(o_p[k], o_f[k]) for k in ('robot', 'human'))       # reset is deterministic
    rng = np.random.default_rng(seed)
    d = {'robot': [], 'human': [], 'force_rel': [], 'reward': []}
    for t in range(steps):
        act = {'robot': rng.uniform(-1, 1, size=(n, 7)).astype(np.float32), 'human': rng.uniform(-1, 1, size=(n, 10)).astype(np.float32)}
        r_p, r_f = per.step(act), fus.step_fused(act)
        for a, b in zip(r_p, r_f):                    # the same dict shapes and keys
            assert a.keys() == b.keys()
            for key in a:
                if isinstance(a[key], dict):
                    assert a[key].keys() == b[key].keys()
                else:
                    assert np.shape(a[key]) == np.shape(b[key]), key
        assert r_p[2]['__all__'] == r_f[2]['__all__'] and np.array_equal(r_p[2]['robot'], r_f[2]['robot'])
        assert r_p[0]['robot'].shape == (n, 24) and r_p[0]['human'].shape == (n, 28)
        for key, k in POSE.items():
            d[key].append(np.abs(r_p[0][key][:, :k] - r_f[0][key][:, :k]).max(axis=1))
        d['force_rel'].append(np.max([(np.abs(r_p[0][k_][:, k:] - r_f[0][k_][:, k:]) / (1 + np.abs(r_p[0][k_][:, k:]))).max(axis=1) for k_, k in POSE.items()], axis=0))
        d['reward'].append(np.abs(r_p[1]['robot'] - r_f[1]['robot']))
        assert np.all(r_f[1]['robot'] == r_f[1]['human'])
    per.close(); fus.close()
    d = {k_: np.array(v) for k_, v in d.items()}
    for k_, v in d.items():
        print('DressingPR2Human-v1 %s fused - per-call |diff| per env-step: median %.2e  p90 %.2e  max %.2e' % (k_, np.median(v), np.quantile(v, 0.9), v.max()))
    return d


def test_coop_dressing_fused_matches_per_call_host_compiled(emu_lib):
    d = _fused_vs_percall(emu_lib, n=4, steps=4)
    assert d['human'].max() < 1e-3 and d['robot'].max() < 1e-3
    # the cloth force sums: contacts at the 4 cm margin chatter between fp32 and the per-call path's reads (the single-agent
    # Dressing test allows 5 % + 1 N); the reward carries them at weight 0.01
    assert d['force_rel'].max() < 0.1 and d['reward'].max() < 0.02


def _bad_left_pose(lo, hi):
    """A shoulder x / y / z + elbow pose inside the template limits that the classifier rejects with the left arm's input mapping
    (human.py:141-145, sign +1) and accepts with the right arm's (sign -1): a sign error in the mapping would not restore it."""
    from assistive_gym_b200.limits_model import load_model
    model = load_model()
    g = np.stack(np.meshgrid(*[np.linspace(l_ + 0.05, h_ - 0.05, 7) for l_, h_ in zip(lo, hi)], indexing='ij'), axis=-1).reshape(-1, 4)
    two_pi = 2 * np.pi

    def x(sign):
        return np.stack([(sign * g[:, 0] + two_pi) % two_pi, (g[:, 1] + two_pi) % two_pi, sign * g[:, 2], (-g[:, 3] + two_pi) % two_pi], axis=1)
    ok = (model.predict_classes(x(1.0))[:, 0] == 0) & (model.predict_classes(x(-1.0))[:, 0] == 1)
    assert ok.any()
    return g[np.flatnonzero(ok)[0]]


def _restored_envs(env, step, chosen, bad):
    """One step with zero action after a step that records each env's reachable pose, the arm of the `chosen` envs put into `bad`
    first; the envs whose arm the step sends away from where it started."""
    n = env.n_envs
    zero = {'robot': np.zeros((n, 7), dtype=np.float32), 'human': np.zeros((n, 10), dtype=np.float32)}
    step(zero)
    db = env._db
    links = {g: [db.gl(hb, j) for j in L_ARM_LIMIT_JOINTS] for g, hb in db.humans.items()}
    q0 = {}
    for g, lk in links.items():
        q = env.id.get_joint_states(lk)[0].astype(np.float64)
        sel = chosen & (env.male if g == 'male' else ~env.male)
        q[sel] = bad
        env.id.set_joint_state(lk, q=q, qd=np.zeros_like(q), mask=sel.astype(np.int32))
        q0[g] = q
    env.id.forward_kinematics()
    step(zero)
    moved = np.zeros(n)
    for g, lk in links.items():
        sel = env.male if g == 'male' else ~env.male
        moved[sel] = np.abs(env.id.get_joint_states(lk)[0] - q0[g]).max(axis=1)[sel]
    return moved > 0.2


def test_coop_dressing_left_arm_mapping_host_compiled(emu_lib):
    n = 4
    per, fus = _make_env(n, emu_lib, 7), _make_env(n, emu_lib, 7)
    per.reset(); fus.reset()
    db = per._db
    lk = [db.gl(db.humans['male'], j) for j in L_ARM_LIMIT_JOINTS]
    lo, hi = db.person_limits(lk)
    bad = _bad_left_pose(np.maximum(lo * 0.5, -3), np.minimum(hi * 0.5, 3))        # inside every env's (scaled) limits
    chosen = np.array([False, True, False, True])
    r_f = _restored_envs(fus, fus.step_fused, chosen, bad)
    r_p = _restored_envs(per, per.step, chosen, bad)
    per.close(); fus.close()
    assert np.array_equal(r_f, chosen) and np.array_equal(r_p, chosen), (r_f, r_p)


def test_single_agent_dressing_unchanged_host_compiled(emu_lib):
    """DressingPR2-v1's reset and four fused steps, bit for bit as before the co-optimisation id existed."""
    sys.path.insert(0, GOLDEN)
    from make_golden_dressing_single_agent import rollout
    P = np.load(os.path.join(GOLDEN, 'dressing_single_agent_pin.npz'))
    out = rollout(emu_lib)
    for k in P.files:
        assert np.array_equal(out[k], P[k]), k


def test_single_agent_template_and_draws_unchanged():
    a, b = DressingBatch(), DressingBatch(controllable_person=True)
    for k, v in a.scene.d.items():                          # the left arm already keeps its mass: the same template
        assert np.asarray(v).tobytes() == np.asarray(b.scene.d[k]).tobytes(), k
    s_a, s_b = a.sample(16, np.random.default_rng(3)), b.sample(16, np.random.default_rng(3), impairment='random')
    for k in s_a:                                           # `limit_scale` is drawn after every existing field
        assert np.array_equal(s_a[k], s_b[k]), k
    assert set(s_b) - set(s_a) == {'limit_scale'}
    s_c = b.sample(64, np.random.default_rng(3))
    assert set(np.unique(s_c['impairment'])) <= {0, 1, 2} and not np.any(s_c['tremors'])        # 'no_tremor'
    assert np.all((s_c['limit_scale'] == 1) | (s_c['impairment'] == 1)) and s_c['limit_scale'].min() >= 0.5


def test_coop_dressing_rejects_bad_input(emu_lib):
    db = DressingBatch(controllable_person=True)
    sim = BatchSim(db.scene, DressingBatch.config(), 2, _lib=emu_lib)
    P = coop_params(db.scene, db.humans, 3, LEFT_ARM_JOINTS, 0.01)
    with pytest.raises(RuntimeError, match='ag_dressing_init first'):
        sim.coop_init(P)
    sim.cloth_init(db.cloth, db.cloth_links, db.cloth_static, [2086, 2087, 2088, 2041], db.anchor_local)
    sim.dressing_init(db.dressing_params(), np.array([1, 0]))
    P4 = coop_params(db.scene, db.humans, 3, LEFT_ARM_JOINTS[:4], 0.01)
    with pytest.raises(RuntimeError, match='10 controllable joints'):
        sim.coop_init(P4)
    P5 = coop_params(db.scene, db.humans, 4, LEFT_ARM_JOINTS, 0.01)
    with pytest.raises(RuntimeError, match='3 \\(dressing\\)'):
        sim.coop_init(P5)
    sim.coop_init(P, limit_scale=[0.5, 1.0])
    sim.close()


def test_coop_dressing_env_surface():
    env = envs.make('DressingPR2Human-v1', n_envs=2)
    assert env.action_space.shape == (17,) and env.action_robot_len == 7 and env.action_human_len == 10
    assert env.obs_robot_len == 24 and env.obs_human_len == 28 and env.observation_space.shape == (52,)
    assert env._db.controllable_person
    import assistive_gym.envs
    assert assistive_gym.envs.DressingPR2HumanEnv is envs.DressingPR2HumanEnv
    single = envs.make('DressingPR2-v1', n_envs=2)
    assert single.action_space.shape == (7,) and single.obs_human_len == 0 and not single._db.controllable_person
    with pytest.raises(RuntimeError, match='no controllable person'):
        single.step_fused({'robot': np.zeros((2, 7)), 'human': np.zeros((2, 10))})


def test_sleeve_on_arm_reward_matches_the_test_restatement():
    """The package's sleeve_on_arm_reward (util.py:134-202) against the restatement the fused Dressing kernels are checked with."""
    from assistive_gym_b200.dressing_batch import sleeve_on_arm_reward
    from tests.dressing_cases import sleeve_on_arm_reward as restated
    rng = np.random.default_rng(0)
    hit = 0
    for _ in range(200):
        sh, el = rng.normal(size=3) * 0.05 + [0, 0, 0.3], rng.normal(size=3) * 0.05
        wr = el + [0.25, 0, 0] + rng.normal(size=3) * 0.05
        c = el + (wr - el) * rng.uniform(-0.5, 1.2) + rng.normal(size=3) * 0.02
        t1, t2 = c + rng.normal(size=(3, 3)) * 0.08, c + rng.normal(size=(3, 3)) * 0.08
        a = sleeve_on_arm_reward(t1, t2, sh, el, wr, 0.043, 0.043, 0.043)
        b = restated(t1, t2, sh, el, wr, 0.043, 0.043, 0.043)
        assert (a[0], a[1]) == (b[0], b[1]) and np.allclose([a[2], a[3], a[4], a[7], a[8]], b[2:], rtol=0, atol=1e-12)
        hit += int(a[0]) + int(a[1])
    assert hit > 0


# ------------------------------------------------------------------ H100
@pytest.mark.gpu
def test_coop_dressing_fused_matches_per_call_cuda(gpu_lib):
    d = _fused_vs_percall(gpu_lib, n=256, steps=3)
    # free-running fp32 with cloth contacts: a few envs may part ways; the population must not
    for k in ('robot', 'human'):
        assert np.median(d[k]) < 1e-4 and np.quantile(d[k], 0.9) < 1e-2, k
    assert np.median(d['force_rel']) < 0.05 and np.median(d['reward']) < 1e-3


@pytest.mark.gpu
def test_coop_dressing_cloth_gravity_reaches_a_captured_step_cuda(gpu_lib):
    """After a captured co-optimisation step, ag_cloth_set_gravity changes what the next replay computes: bit for bit what a sim
    without graph capture computes with that gravity."""
    n = 64
    db = DressingBatch(controllable_person=True)
    smp = None
    sims = []
    for graph in (True, False):
        old = os.environ.get('AG_GRAPH')
        if not graph:
            os.environ['AG_GRAPH'] = '0'
        try:
            sim = BatchSim(db.scene, DressingBatch.config(), n, _lib=gpu_lib)
        finally:
            if old is None:
                os.environ.pop('AG_GRAPH', None)
            else:
                os.environ['AG_GRAPH'] = old
        smp = db.reset(sim, np.random.default_rng(2), sample=smp, attempts=6, settle_steps=2)
        db.start_fused(sim, smp)
        db.start_coop(sim, smp)
        sims.append(sim)
    rng = np.random.default_rng(4)
    acts = [np.concatenate([rng.uniform(-1, 1, size=(n, 7)), rng.uniform(-1, 1, size=(n, 10))], axis=1).astype(np.float32) for _ in range(3)]
    out = []
    for sim in sims:
        first = sim.coop_step_host(acts[0])                # captured (graph) or launched directly
        sim.cloth_set_gravity([0, 0, -2.0])
        res = [sim.coop_step_host(a) for a in acts[1:]]
        out.append((first, res, sim.state_get(), sim.cloth_get_state()[0]))
    (f_g, r_g, s_g, x_g), (f_d, r_d, s_d, x_d) = out
    for a, b in zip(f_g, f_d):
        assert np.array_equal(a, b)                        # graph replay and direct launches agree bit for bit
    for step_g, step_d in zip(r_g, r_d):
        for a, b in zip(step_g, step_d):
            assert np.array_equal(a, b)
    assert np.array_equal(s_g, s_d) and np.array_equal(x_g, x_d)
    for sim in sims:
        sim.close()


@pytest.mark.gpu
def test_coop_dressing_vec_env_torch_episode(gpu_lib):
    import torch
    from assistive_gym_b200.vec_env import AssistiveVecEnv
    n = 64
    vec = AssistiveVecEnv('assistive_gym:DressingPR2Human-v1', n_envs=n, device=0, _lib=gpu_lib, double_buffer=True, toc_attempts=8)
    assert vec.coop
    obs = vec.reset()
    assert obs['robot'].shape == (n, 24) and obs['human'].shape == (n, 28)
    dev = torch.device('cuda:0')
    act = {'robot': torch.zeros(n, 7, device=dev), 'human': torch.zeros(n, 10, device=dev)}
    act['human'][:, 4] = 1.0                                                 # shoulder y: lifts the arm inside the gown
    q_slice = slice(7, 17)
    q0 = torch.as_tensor(obs['human'][:, q_slice], device=dev)
    for t in range(200):
        o, r, d, info = vec.step(act)
        assert isinstance(o['human'], torch.Tensor) and o['human'].is_cuda and o['robot'].shape == (n, 24)
        assert o['human'].shape == (n, 28) and r['robot'].shape == (n,) and r['robot'] is r['human']
        if t == 19:
            moved = (o['human'][:, q_slice] - q0).abs().max(dim=1).values
            print('DressingPR2Human-v1 person joint travel after 20 steps: median %.3f rad' % moved.median().item())
            assert (moved > 0.05).float().mean().item() > 0.9                 # the person's action moves the person
        if t < 199:
            assert not d['__all__'] and 'terminal_observation' not in info['robot']
            assert torch.isfinite(o['robot']).all() and torch.isfinite(o['human']).all() and torch.isfinite(r['robot']).all()
    assert d['__all__'] and bool(d['robot'].all())
    term = info['human']['terminal_observation']
    assert term.shape == (n, 28) and torch.isfinite(term).all() and torch.isfinite(info['robot']['terminal_observation']).all()
    o, r, d, info = vec.step(act)                                                    # the swapped-in copy steps
    assert not d['__all__'] and torch.isfinite(o['human']).all()
    vec.close()
