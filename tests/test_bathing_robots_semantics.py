"""BedBathingPR2-v1 and BedBathingPR2Human-v1 against the reference's OWN `BedBathingEnv.step` with PR2
(tests/golden/bathing_pr2_semantics.npz and bathing_pr2_coop_semantics.npz, recorded on the CPU oracle by
make_golden_bathing_robots_semantics.py).  These pin what is robot-specific in the step: the left end effector of the velocity term,
PR2's base frame of the observation and the wiper held at the left tool joint.  The single-agent rollout starts with the wiper pad
pressed onto the forearm (up to 9 N on the person), so targets are wiped; in the co-optimisation rollout the person bends the elbow and
raises and turns the upper arm until the joint-limit classifier sends it back.

- the env's own per-call step on the oracle reproduces each rollout to rounding;
- the fused kernel bodies compiled for the host (`ag_bathing_step_host`, `ag_coop_step_host`) replay them from the golden start;
- on the H100, `bathing_step_dev` / `coop_step_dev` with torch tensors replay them."""
import os

import numpy as np
import pytest

from assistive_gym_b200 import capi, envs
from assistive_gym_b200.bed_bathing_batch import RIGHT_ARM_JOINTS
from assistive_gym_b200.bed_bathing_robots_batch import BedBathingPR2Batch
from assistive_gym_b200.sim import BatchSim

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
G = np.load(os.path.join(GOLDEN, 'bathing_pr2_semantics.npz'))
SMP = {k[len('sample_'):]: G[k] for k in G.files if k.startswith('sample_')}
GC = np.load(os.path.join(GOLDEN, 'bathing_pr2_coop_semantics.npz'))
SMP_C = {k[len('sample_'):]: GC[k] for k in GC.files if k.startswith('sample_')}


def test_per_call_step_reproduces_the_reference_s_rollout(monkeypatch):
    """`BedBathingEnv.step_reference_api` (take_step, _get_obs, get_total_force, human_preferences through the Agent getters)."""
    import assistive_gym_b200.envs.bed_bathing as bathing_mod
    from oracle.oracle_py import OracleSim
    env = envs.make('BedBathingPR2-v1', n_envs=1)
    bb = env._bb
    assert np.array_equal(G['robot_lower'], bb.arm_lower) and np.array_equal(G['robot_upper'], bb.arm_upper)     # the reference's own limits
    sim = OracleSim(bb.scene, capi.default_config(residual_threshold=0.0), 1)
    monkeypatch.setattr(bathing_mod, 'BatchSim', lambda *a, **k: sim)
    monkeypatch.setattr(bb, 'sample', lambda *a, **k: dict(SMP))     # the oracle has no batched IK: the placement is replayed
    monkeypatch.setattr(bb, 'start_fused', lambda s, smp: bb.targets_world(s, smp))     # the oracle has no fused step
    env.reset()
    sim.state_set(G['start_state']); sim.forward_kinematics()
    env.robot.motor_gains, env.robot.motor_forces = float(G['motor_gain']), float(G['motor_force'])
    env.targets_pos_world, env.targets_alive = bb.targets_world(sim, SMP)
    assert int(env.total_target_count[0]) == int(G['total_target_count'])
    env.task_success[:] = 0
    for t, a in enumerate(G['actions']):
        obs, rew, done, info = env.step_reference_api(a[None])
        assert np.allclose(obs[:23], G['obs'][t][:23], rtol=0, atol=1e-9), (t, np.abs(obs[:23] - G['obs'][t][:23]).max())
        assert abs(obs[23] - G['obs'][t][23]) < 1e-6 and abs(info['total_force_on_human'] - G['total_force'][t]) < 1e-6      # forces
        assert abs(env.tool_force_on_human[0] - G['tool_force_on_human'][t]) < 1e-6
        # the reward to 1e-9 beyond what the force terms of human_preferences (weights 0.01 and 0.05, config.ini) carry of the
        # forces' rounding: the reference sums fp32 contact records, the restatement asks the oracle for fp64 sums
        ferr = max(abs(info['total_force_on_human'] - G['total_force'][t]), abs(env.tool_force_on_human[0] - G['tool_force_on_human'][t]))
        assert abs(rew - G['reward'][t]) < 1e-9 + 0.06 * ferr, (t, rew, G['reward'][t], ferr)
        assert bool(done) == bool(G['done'][t])
        assert int(env.new_contact_points[0]) == int(G['new_contact_points'][t]) and int(env.task_success[0]) == int(G['task_success'][t])
    assert G['new_contact_points'].sum() >= 1 and G['tool_force_on_human'].max() > 3     # the pad presses and wipes targets


def _replay_fused(lib, step):
    bb = BedBathingPR2Batch()
    prod = BatchSim(bb.scene, capi.default_config(residual_threshold=0.0), 1, _lib=lib)
    bb.reset(prod, np.random.default_rng(0), sample=dict(SMP))
    prod.state_set(G['start_state'].astype(np.float32)); prod.forward_kinematics()
    prod.set_motor(bb.arm_links, 1, target=prod.get_joint_states(bb.arm_links)[0], kp=[float(G['motor_gain'])] * 7, kd=[1.0] * 7, max_force=[float(G['motor_force'])] * 7)
    bb.start_fused(prod, SMP)
    err, rerr, ferr, wiped = [], [], [], []
    for t, a in enumerate(G['actions']):
        obs, rew, info = step(prod, a[None].astype(np.float32))
        err.append(np.abs(obs[0, :23] - G['obs'][t][:23]).max()); rerr.append(abs(rew[0] - G['reward'][t])); wiped.append(int(info[0, 3]))
        # the tool force (obs[23]), the total force on the person (info[0]) and the cloth force on the person (info[2]), each relative
        # to a 5 % + 0.05 N bound (BedBathingSawyer-v1's, tests/test_reference_bathing_semantics.py)
        ferr.append(max(abs(f - g) / (0.05 * abs(g) + 0.05) for f, g in ((obs[0, 23], G['obs'][t][23]), (info[0, 0], G['total_force'][t]),
                                                                       (info[0, 2], G['tool_force_on_human'][t]))))
    prod.close()
    err, rerr, ferr = np.array(err), np.array(rerr), np.array(ferr)
    print('BedBathingPR2 fused replay: max |obs error| %.2e, max |reward error| %.2e, force error / bound %.2f (peak cloth force %.2f N), wiped per step %s'
          % (err.max(), rerr.max(), ferr.max(), G['tool_force_on_human'].max(), wiped))
    assert np.array_equal(wiped, G['new_contact_points'].astype(int)), (wiped, G['new_contact_points'])
    assert err.max() < 1e-5 and rerr.max() < 1e-3 and ferr.max() < 1, (err, rerr, ferr)


def test_fused_kernel_bodies_replay_the_reference_s_rollout(emu_lib):
    def step(sim, a):
        obs, rew, done, info = sim.bathing_step_host(a)
        return obs, rew, info
    _replay_fused(emu_lib, step)


def test_coop_per_call_step_reproduces_the_reference_s_rollout(monkeypatch):
    """The co-optimisation env's `step` (dict actions and observations, the person's arm inside the realistic joint limits, the
    targets following the arm) against the reference's own, with the classifier's restorations counted on both sides."""
    import assistive_gym_b200.envs.bed_bathing as bathing_mod
    from oracle.oracle_py import OracleSim
    env = envs.make('BedBathingPR2Human-v1', n_envs=1)
    bb = env._bb
    assert np.array_equal(GC['robot_lower'], bb.arm_lower) and np.array_equal(GC['robot_upper'], bb.arm_upper)
    sim = OracleSim(bb.scene, capi.default_config(residual_threshold=0.0), 1)
    monkeypatch.setattr(bathing_mod, 'BatchSim', lambda *a, **k: sim)
    monkeypatch.setattr(bb, 'sample', lambda *a, **k: dict(SMP_C))   # the oracle has no batched IK: the placement is replayed
    monkeypatch.setattr(bb, 'start_fused', lambda s, smp: bb.targets_world(s, smp))     # the oracle has no fused step
    monkeypatch.setattr(bb, 'start_coop', lambda *a, **k: None)
    env.reset()
    sim.state_set(GC['start_state']); sim.forward_kinematics()
    g = 'male' if env.male[0] else 'female'
    h = env.humans[g]
    from assistive_gym_b200.limits_model import load_model
    model, restores = load_model(), [0]

    def predict_classes(x):                     # the classifier's objections that send the arm back, as the golden counts them
        c = model.predict_classes(x)
        prev = h.arm_previous_valid_pose[True]
        if int(c[0, 0]) == 0 and prev is not None and not np.isnan(prev[0, 0]):
            restores[0] += 1
        return c
    h.limits_model = type('Classifier', (), {'predict_classes': staticmethod(predict_classes)})()
    links = [bb.gl(bb.humans[g], j) for j in RIGHT_ARM_JOINTS]
    for t, a_h in enumerate(GC['human_actions']):
        o, r, d, info = env.step({'robot': np.zeros(7), 'human': a_h})
        arm = sim.get_joint_states(links)[0][0]
        assert np.allclose(arm, GC['arm_q'][t], rtol=0, atol=1e-7), (t, np.abs(arm - GC['arm_q'][t]).max())
        assert np.allclose(o['robot'][:23], GC['obs_robot'][t][:23], rtol=0, atol=1e-6) and abs(o['robot'][23] - GC['obs_robot'][t][23]) < 1e-4 * (1 + abs(GC['obs_robot'][t][23]))
        assert np.allclose(o['human'][:26], GC['obs_human'][t][:26], rtol=0, atol=1e-6) and np.allclose(o['human'][26:], GC['obs_human'][t][26:], rtol=1e-4, atol=1e-4)
        assert abs(r['robot'] - GC['reward'][t]) < 1e-5 and r['robot'] == r['human'] and bool(d['__all__']) == bool(GC['done'][t])
        assert restores[0] == int(GC['restores'][t]), (t, restores[0], GC['restores'][t])
    assert GC['restores'][-1] >= 1                                             # the classifier sent the arm back


def _replay_coop(lib, step):
    bb = BedBathingPR2Batch(controllable_person=True)
    sim = BatchSim(bb.scene, capi.default_config(residual_threshold=0.0), 1, _lib=lib)
    bb.reset(sim, np.random.default_rng(0), sample=dict(SMP_C))
    sim.state_set(GC['start_state'].astype(np.float32)); sim.forward_kinematics()
    bb.start_fused(sim, SMP_C)
    bb.start_coop(sim, SMP_C)
    links = [bb.gl(bb.humans['male' if SMP_C['male'][0] else 'female'], j) for j in RIGHT_ARM_JOINTS]
    e = {k: [] for k in ('arm', 'obs_robot', 'obs_human', 'force', 'reward')}
    for t, a_h in enumerate(GC['human_actions']):
        obs_r, obs_h, rew = step(sim, np.concatenate([np.zeros(7), a_h])[None].astype(np.float32))
        arm = sim.get_joint_states(links)[0][0]
        e['arm'].append(np.abs(arm - GC['arm_q'][t]).max()); e['obs_robot'].append(np.abs(obs_r[0, :23] - GC['obs_robot'][t][:23]).max())
        e['obs_human'].append(np.abs(obs_h[0, :26] - GC['obs_human'][t][:26]).max()); e['reward'].append(abs(rew[0] - GC['reward'][t]))
        e['force'].append(max(abs(obs_r[0, 23] - GC['obs_robot'][t][23]), np.abs(obs_h[0, 26:] - GC['obs_human'][t][26:]).max()))
    sim.close()
    e = {k: np.array(v) for k, v in e.items()}
    print('BedBathingPR2Human coop replay, max |error| over %d steps:' % len(GC['reward']), {k: '%.2e' % v.max() for k, v in e.items()})
    # BedBathingSawyerHuman-v1's bounds for its golden (tests/test_bathing_coop.py)
    assert e['arm'].max() < 3e-6 and e['obs_robot'].max() < 3e-6 and e['obs_human'].max() < 3e-6, e
    assert e['force'].max() < 1e-3 and e['reward'].max() < 1e-5, e


def test_coop_kernel_bodies_replay_the_reference_s_rollout(emu_lib):
    def step(sim, a):
        obs_r, obs_h, rew, done, info = sim.coop_step_host(a)
        return obs_r, obs_h, rew
    _replay_coop(emu_lib, step)


@pytest.mark.gpu
def test_step_dev_replays_the_reference_s_rollout_cuda(gpu_lib):
    import torch
    dev = torch.device('cuda:0')
    o, r, d, i = torch.zeros(1, 24, device=dev), torch.zeros(1, device=dev), torch.zeros(1, device=dev), torch.zeros(1, 4, device=dev)

    def step(sim, a):
        at = torch.as_tensor(a, device=dev).contiguous()
        torch.cuda.synchronize()
        sim.bathing_step_dev(at.data_ptr(), o.data_ptr(), r.data_ptr(), d.data_ptr(), i.data_ptr())
        torch.cuda.synchronize()
        return o.cpu().numpy().astype(np.float64), r.cpu().numpy().astype(np.float64), i.cpu().numpy()
    _replay_fused(gpu_lib, step)
    oh = torch.zeros(1, 28, device=dev)

    def coop_step(sim, a):
        at = torch.as_tensor(a, device=dev).contiguous()
        torch.cuda.synchronize()
        sim.coop_step_dev(at.data_ptr(), o.data_ptr(), oh.data_ptr(), r.data_ptr(), d.data_ptr(), i.data_ptr())
        torch.cuda.synchronize()
        return o.cpu().numpy().astype(np.float64), oh.cpu().numpy().astype(np.float64), r.cpu().numpy().astype(np.float64)
    _replay_coop(gpu_lib, coop_step)
