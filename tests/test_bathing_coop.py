"""The fused co-optimisation step of BedBathingSawyerHuman-v1 (ag_coop_* with task 2): the person's right arm is a second agent,
and k_bath_track re-places the wiping targets on the moving arm after the step's last substep.

On the CPU (kernel bodies compiled for the host): the reference's own rollout (tests/golden/bathing_coop_semantics.npz), the fused
step against the per-call `step` of the same env, the single-agent BedBathingSawyer-v1 path against a pin taken before this id
existed, input checks and the env surface.  On the H100: the same comparison at scale, the wiped targets with the pad pressed,
and a vector-env episode with torch tensors."""
import os
import sys

import numpy as np
import pytest

from assistive_gym_b200 import capi, envs
from assistive_gym_b200.bed_bathing_batch import R_ELBOW, RIGHT_ARM_JOINTS, SAWYER, BedBathingBatch
from assistive_gym_b200.feeding_batch import coop_params
from assistive_gym_b200.sim import BatchSim
from tests.test_bed_bathing import _pressed_pair

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def test_coop_bathing_golden_host_compiled(emu_lib):
    """ag_coop_step_host from the golden's start state against what the reference's own step returned on the fp64 oracle."""
    G = np.load(os.path.join(GOLDEN, 'bathing_coop_semantics.npz'))
    bb = BedBathingBatch(controllable_person=True)
    _cpu, prod, smp, _ik = _pressed_pair(bb, lambda sc, cfg, n: BatchSim(sc, cfg, n, _lib=emu_lib), 1, seed=8)
    smp = dict(smp, impairment=G['sample_impairment'], limit_scale=G['sample_limit_scale'], strength=G['sample_strength'])
    prod.state_set(G['start_state'].astype(np.float32)); prod.forward_kinematics()
    prod.set_motor(bb.arm_links, 1, target=prod.get_joint_states(bb.arm_links)[0], kp=[float(G['motor_gain'])] * 7, kd=[1.0] * 7, max_force=[float(G['motor_force'])] * 7)
    bb.start_fused(prod, smp)
    bb.start_coop(prod, smp)
    links = [bb.gl(bb.humans['male' if smp['male'][0] else 'female'], j) for j in RIGHT_ARM_JOINTS]
    err = dict(arm=0.0, obs_robot=0.0, obs_human=0.0, force=0.0, reward=0.0)
    wiped = 0
    for t, a in enumerate(G['actions']):
        obs_r, obs_h, rew, done, info = prod.coop_step_host(a[None].astype(np.float32))
        arm = prod.get_joint_states(links)[0][0]
        err['arm'] = max(err['arm'], np.abs(arm - G['arm_q'][t]).max())
        err['obs_robot'] = max(err['obs_robot'], np.abs(obs_r[0, :23] - G['obs_robot'][t][:23]).max())
        err['obs_human'] = max(err['obs_human'], np.abs(obs_h[0, :26] - G['obs_human'][t][:26]).max())
        err['force'] = max(err['force'], abs(obs_r[0, 23] - G['obs_robot'][t][23]), np.abs(obs_h[0, 26:] - G['obs_human'][t][26:]).max())
        err['reward'] = max(err['reward'], abs(rew[0] - G['reward'][t]))
        wiped += int(info[0, 3])
        assert int(info[0, 3]) == int(G['new_contact_points'][t]) and wiped == int(G['task_success'][t]), t
        assert int(info[0, 1]) == int(G['task_success'][t] >= G['total_target_count'] * 0.3) and bool(done[0]) == bool(G['done'][t])
    prod.close()
    print('bathing coop golden, max |error| over %d steps:' % len(G['reward']), {k: '%.2e' % v for k, v in err.items()})
    assert err['arm'] < 3e-6 and err['obs_robot'] < 3e-6 and err['obs_human'] < 3e-6, err
    assert err['force'] < 1e-3 and err['reward'] < 1e-5, err
    assert wiped == len(G['wiped_target']) >= 3


def _make_env(n, lib, seed):
    env = envs.make('BedBathingSawyerHuman-v1', n_envs=n, seed=seed)
    env._sim_lib = lib
    sample = env._bb.sample

    def sample_both_genders_half_limited(*a, **kw):
        s = sample(*a, **kw)
        s['male'][:] = np.arange(n) % 2
        lim = np.arange(n) % 4 < 2                    # the `limits` impairment at scale 0.5 in half of the envs
        s['impairment'] = np.where(lim, 1, s['impairment']).astype(np.int32)
        s['limit_scale'] = np.where(lim, 0.5, s['limit_scale'])
        return s
    env._bb.sample = sample_both_genders_half_limited
    return env


def _fused_vs_percall(lib, n, steps, seed=5):
    """Two envs from the same seed: one stepped by `step` (per-call), one by `step_fused`; the same float32 actions."""
    per, fus = _make_env(n, lib, seed), _make_env(n, lib, seed)
    o_p, o_f = per.reset(), fus.reset()
    assert all(np.array_equal(o_p[k], o_f[k]) for k in ('robot', 'human'))       # reset is deterministic
    rng = np.random.default_rng(seed)
    d_obs, d_rew, d_force = {'robot': [], 'human': []}, [], []
    nf = {'robot': 23, 'human': 26}                   # the entries before these are poses and angles, the rest are forces (N)
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
        assert np.array_equal(r_p[3]['robot']['task_success'], r_f[3]['robot']['task_success'])
        for key in ('robot', 'human'):
            d_obs[key].append(np.abs(r_p[0][key][:, :nf[key]] - r_f[0][key][:, :nf[key]]).max(axis=1))
        d_force.append(np.max([(np.abs(r_p[0][k_][:, nf[k_]:] - r_f[0][k_][:, nf[k_]:]) / (1 + np.abs(r_p[0][k_][:, nf[k_]:]))).max(axis=1) for k_ in nf], axis=0))
        d_rew.append(np.abs(r_p[1]['robot'] - r_f[1]['robot']))
        assert np.all(r_f[1]['robot'] == r_f[1]['human'])
    per.close(); fus.close()
    d = {k_: np.array(v) for k_, v in d_obs.items()}
    d['reward'], d['force_rel'] = np.array(d_rew), np.array(d_force)
    for k_, v in d.items():
        print('BedBathingSawyerHuman-v1 %s fused - per-call |diff| per env-step: median %.2e  p90 %.2e  max %.2e' % (k_, np.median(v), np.quantile(v, 0.9), v.max()))
    return d


def test_coop_bathing_fused_matches_per_call_host_compiled(emu_lib):
    d = _fused_vs_percall(emu_lib, n=8, steps=10)
    assert d['human'].max() < 1e-3 and d['robot'].max() < 1e-3 and d['reward'].max() < 1e-3
    # contact forces relative to their size: one env drives the wiper into the person at 55 N, where the fp32 rounding of the
    # robot's PD targets (the per-call path computes them in fp64) moves the force by about 0.3 % (BedBathingSawyer-v1's own
    # fused vs per-call test allows 5e-3 on every observation)
    assert d['force_rel'].max() < 5e-3


def test_single_agent_bathing_unchanged_host_compiled(emu_lib):
    """BedBathingSawyer-v1's reset and ten fused steps, bit for bit as before the co-optimisation id existed."""
    sys.path.insert(0, GOLDEN)
    from make_golden_bathing_single_agent import rollout
    G = np.load(os.path.join(GOLDEN, 'bathing_single_agent_pin.npz'))
    out = rollout(emu_lib)
    for k in G.files:
        assert np.array_equal(out[k], G[k]), k


def test_single_agent_template_unchanged():
    a, b = BedBathingBatch(), BedBathingBatch(controllable_person=True)
    s0 = BedBathingBatch().scene
    for k, v in a.scene.d.items():
        assert np.asarray(v).tobytes() == np.asarray(s0.d[k]).tobytes(), k
    arm = {a.gl(hb, j) for hb in a.humans.values() for j in RIGHT_ARM_JOINTS}
    for k in range(len(a.scene['link_mass'])):             # only the two right arms differ: they keep their mass
        same = a.scene['link_mass'][k] == b.scene['link_mass'][k]
        assert same or k in arm, k
    assert all(sum(b.scene['link_mass'][b.gl(hb, j)] for j in RIGHT_ARM_JOINTS) > 1 for hb in b.humans.values())     # the arms are live
    rng = np.random.default_rng(3)
    s_a, s_b = a.sample(16, np.random.default_rng(3)), b.sample(16, rng)
    for k in s_a:                                           # the extra draws come after every existing one
        assert np.array_equal(s_a[k], s_b[k]), k
    assert set(s_b) - set(s_a) == {'impairment', 'limit_scale', 'strength'} and set(np.unique(s_b['impairment'])) <= {0, 1, 2}


def test_coop_bathing_rejects_bad_input(emu_lib):
    bb = BedBathingBatch(controllable_person=True)
    sim = BatchSim(bb.scene, capi.default_config(), 2, _lib=emu_lib)
    P = coop_params(bb.scene, bb.humans, 2, RIGHT_ARM_JOINTS, 0.05)
    with pytest.raises(RuntimeError, match='ag_bathing_init first'):
        sim.coop_init(P)
    s = bb.sample(2, np.random.default_rng(0))
    link, local = bb.target_frames(s)
    with pytest.raises(RuntimeError, match='ag_bathing_init first'):
        sim.bathing_set_target_frames(link, local)
    tw, valid = bb.targets_world(sim, s)
    sim.bathing_init(bb.bathing_params(), s['male'], tw, valid)
    with pytest.raises(RuntimeError, match='set_target_frames first'):
        sim.coop_init(P)
    bad = link.copy(); bad[0, 0] = bb.arm_links[0]                           # a robot link
    with pytest.raises(RuntimeError, match='bad target link'):
        sim.bathing_set_target_frames(bad, local)
    bad[0, 0] = 10 ** 6
    with pytest.raises(RuntimeError, match='bad target link'):
        sim.bathing_set_target_frames(bad, local)
    sim.bathing_set_target_frames(link, local)
    P4 = coop_params(bb.scene, bb.humans, 2, RIGHT_ARM_JOINTS[:4], 0.05)
    with pytest.raises(RuntimeError, match='10 controllable joints'):
        sim.coop_init(P4)
    sim.coop_init(P, limit_scale=[0.5, 1.0])
    sim.bathing_init(bb.bathing_params(), s['male'], tw, valid)                  # a new episode: the frames have to follow
    with pytest.raises(RuntimeError, match='set_target_frames'):
        sim.coop_step_host(np.zeros((2, 17), dtype=np.float32))
    sim.close()


def test_coop_bathing_env_surface():
    env = envs.make('BedBathingSawyerHuman-v1', n_envs=2)
    assert env.action_space.shape == (17,) and env.action_robot_len == 7 and env.action_human_len == 10
    assert env.obs_robot_len == 24 and env.obs_human_len == 28 and env.observation_space.shape == (52,)
    import assistive_gym.envs
    assert assistive_gym.envs.BedBathingSawyerHumanEnv is envs.BedBathingSawyerHumanEnv
    single = envs.make('BedBathingSawyer-v1', n_envs=2)
    assert single.action_space.shape == (7,) and single.obs_human_len == 0 and not single._bb.controllable_person
    with pytest.raises(RuntimeError, match='no controllable person'):
        single.step_fused({'robot': np.zeros((2, 7)), 'human': np.zeros((2, 10))})


def test_coop_bathing_targets_follow_the_arm_host_compiled(emu_lib):
    """The per-call env re-places the targets from the current link poses; the same frames drive k_bath_track."""
    env = _make_env(2, emu_lib, 4)
    env.reset()
    t0 = env.targets_pos_world.copy()
    act = {'robot': np.zeros((2, 7)), 'human': np.zeros((2, 10))}
    act['human'][:, 7] = 1.0                                                 # roll the forearm
    for _ in range(3):
        env.step(act)
    link, local = env._bb.target_frames({'male': env.male})
    moved = np.linalg.norm(env.targets_pos_world - t0, axis=2)
    assert moved[link >= 0].max() > 0.01 and moved[link < 0].max() == 0      # the targets moved with the arm, the padding did not
    elbow = env._bb.gl(env._bb.humans['male' if env.male[0] else 'female'], R_ELBOW)
    ls = env.id.get_link_states([elbow])
    from assistive_gym_b200.kinematics import q_rot
    fore = link[0] == elbow
    w = ls['pos'][0, 0].astype(np.float64) + q_rot(np.broadcast_to(ls['quat'][0, 0].astype(np.float64), (int(fore.sum()), 4)), local[0, fore])
    assert fore.sum() > 0 and np.abs(w - env.targets_pos_world[0, fore]).max() < 1e-6
    env.close()


# ------------------------------------------------------------------ H100
@pytest.mark.gpu
def test_coop_bathing_fused_matches_per_call_cuda(gpu_lib):
    d = _fused_vs_percall(gpu_lib, n=1024, steps=10)
    # free-running fp32 with contacts: a few envs may part ways; the population must not
    for k in ('robot', 'human', 'force_rel'):
        assert np.median(d[k]) < 1e-4 and np.quantile(d[k], 0.9) < 1e-2, k
    assert np.median(d['reward']) < 1e-4 and np.quantile(d['reward'], 0.9) < 1e-2


@pytest.mark.gpu
def test_coop_bathing_pressed_pad_task_success_cuda(gpu_lib):
    """With the pad pressed onto the forearm and the person rolling it, the fused step wipes targets as the per-call step does."""
    n, steps = 512, 10
    bb = BedBathingBatch(controllable_person=True)
    cpu, _dev, smp, ik = _pressed_pair(bb, lambda sc, cfg, m: BatchSim(sc, cfg, m, _lib=gpu_lib), 1, seed=8)
    # the same pressed start in every env: per-call and fused sims from one state, each env with its own forearm roll
    per, fus = (BatchSim(bb.scene, capi.default_config(residual_threshold=0.0), n, _lib=gpu_lib) for _ in range(2))
    smp_n = {k: np.repeat(np.asarray(v)[:1], n, axis=0) for k, v in smp.items()}
    smp_n['limit_scale'] = np.ones(n)
    st = np.repeat(cpu.state_get().astype(np.float32), n, axis=0)
    arm = np.array(SAWYER['arm']) + 1
    q_lo = np.repeat(ik[2][:, arm], n, axis=0)
    rng = np.random.default_rng(0)
    roll = rng.uniform(-1, 1, size=n)
    succ = []
    for sim in (per, fus):
        bb.reset(sim, np.random.default_rng(8), sample=dict(smp_n))
        sim.state_set(st); sim.forward_kinematics()
        sim.set_motor(bb.arm_links, 1, target=sim.get_joint_states(bb.arm_links)[0], kp=[0.1] * 7, kd=[1.0] * 7, max_force=[5.0] * 7)
    env = envs.make('BedBathingSawyerHuman-v1', n_envs=n)
    env._bb, env.id = bb, per
    env.plane.init(bb.plane, per, env.np_random, indices=-1); env.robot.init(bb.robot, per, env.np_random)
    env.tool.init(bb.tool, per, env.np_random, indices=-1); env.furniture.init(bb.bed, per, env.np_random, indices=-1)
    env.robot.motor_gains, env.robot.motor_forces = 0.1, 5.0
    env.male = smp_n['male'].astype(bool)
    env.humans, env.agents = {}, [env.robot]
    for g, hb in bb.humans.items():
        h = type(env.human)(env.human.controllable_joint_indices, controllable=True)
        h.init(hb, per, env.np_random, env.human.controllable_joint_indices)
        h.env_mask = env.male if g == 'male' else ~env.male
        h.set_limit_scale(np.ones(n))
        env.humans[g] = h
        env.agents.append(h)
    env.targets_pos_world, env.targets_alive = bb.targets_world(per, smp_n)
    env.total_target_count = env.targets_alive.sum(axis=1)
    env.task_success, env.iteration = np.zeros(n, dtype=int), 0
    bb.start_fused(fus, smp_n)
    bb.start_coop(fus, smp_n)
    agree, fused_total = [], np.zeros(n, dtype=int)
    for t in range(steps):
        q = per.get_joint_states(bb.arm_links)[0]
        a_r = np.clip((q_lo - q) / 0.25, -1, 1).astype(np.float32)
        a_h = np.zeros((n, 10), dtype=np.float32); a_h[:, 7] = roll
        env.step({'robot': a_r, 'human': a_h})
        q_f = fus.get_joint_states(bb.arm_links)[0]
        a_rf = np.clip((q_lo - q_f) / 0.25, -1, 1).astype(np.float32)
        _o_r, _o_h, _rew, _done, info = fus.coop_step_host(np.concatenate([a_rf, a_h], axis=1))
        succ.append(env.task_success.copy())
        fused_total += info[:, 3].astype(int)
        agree.append(float(np.mean(env.task_success == fused_total)))
    per.close(); fus.close(); cpu.close()
    print('pressed pad: targets wiped per env after %d steps: per-call mean %.2f, fused mean %.2f; envs that agree, per step'
          % (steps, succ[-1].mean(), fused_total.mean()), np.round(agree, 4))
    assert succ[-1].mean() >= 1 and min(agree) >= 0.99


@pytest.mark.gpu
def test_coop_bathing_vec_env_torch_episode(gpu_lib):
    import torch
    from assistive_gym_b200.vec_env import AssistiveVecEnv
    n = 256
    vec = AssistiveVecEnv('assistive_gym:BedBathingSawyerHuman-v1', n_envs=n, device=0, _lib=gpu_lib, double_buffer=True)
    assert vec.coop
    obs = vec.reset()
    assert obs['robot'].shape == (n, 24) and obs['human'].shape == (n, 28)
    dev = torch.device('cuda:0')
    act = {'robot': torch.zeros(n, 7, device=dev), 'human': torch.zeros(n, 10, device=dev)}
    act['human'][:, 5] = 1.0                                                 # shoulder z: turns the upper arm on the mattress
    q_slice = slice(7, 17)
    q0 = torch.as_tensor(obs['human'][:, q_slice], device=dev)
    for t in range(200):
        o, r, d, info = vec.step(act)
        assert isinstance(o['human'], torch.Tensor) and o['human'].is_cuda and o['robot'].shape == (n, 24)
        assert o['human'].shape == (n, 28) and r['robot'].shape == (n,) and r['robot'] is r['human']
        if t == 19:
            moved = (o['human'][:, q_slice] - q0).abs().max(dim=1).values
            print('BedBathingSawyerHuman-v1 person joint travel after 20 steps: median %.3f rad' % moved.median().item())
            assert (moved > 0.05).float().mean().item() > 0.9                 # the person's action moves the person
        if t < 199:
            assert not d['__all__'] and 'terminal_observation' not in info['robot']
            assert torch.isfinite(o['robot']).all() and torch.isfinite(o['human']).all() and torch.isfinite(r['robot']).all()
    assert d['__all__'] and bool(d['robot'].all())
    term = info['human']['terminal_observation']
    assert term.shape == (n, 28) and torch.isfinite(term).all() and torch.isfinite(info['robot']['terminal_observation']).all()
    assert o['human'].shape == (n, 28) and not torch.equal(o['human'], term)          # the fresh episode's observation
    o, r, d, info = vec.step(act)                                                    # the swapped-in copy steps
    assert not d['__all__'] and torch.isfinite(o['human']).all()
    vec.close()
