"""Every fused env-step entry point against a pin recorded before their host halves were merged into one
(tests/golden/fused_step_pin.npz, make_golden_fused_step_pin.py): the four single-agent ids through `*_step_host` and the four
co-optimisation ids through `coop_step_host`, 4 envs of both genders.

On the CPU (kernel bodies compiled for the host): each path reproduces the pin bit for bit, kernel-launch counts included; the
device-pointer entry point computes what the host-buffer one does; every host-buffer entry point accepts a NULL `info`.
On the H100: the CUDA-graph replayed step gives bit for bit what direct launches give, with the pinned launch count."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.golden.make_golden_fused_step_pin import N_ENVS, PATHS, make_env, rollout

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _pin(env_id):
    P = np.load(os.path.join(GOLDEN, 'fused_step_pin.npz'))
    return {k.split('/', 1)[1]: P[k] for k in P.files if k.startswith(env_id + '/')}


@pytest.mark.parametrize('env_id', list(PATHS))
def test_fused_step_reproduces_pin_host_compiled(emu_lib, env_id):
    pin, out = _pin(env_id), rollout(emu_lib, env_id)
    assert out.keys() == pin.keys()
    for k in pin:
        assert np.array_equal(out[k], pin[k]), k


@pytest.mark.parametrize('env_id', list(PATHS))
def test_dev_step_and_null_info_match_host_step_host_compiled(emu_lib, env_id):
    """`*_step_dev` on host buffers (which the host-compiled library reads directly) equals the pinned `*_step_host`; a first
    step through the C ABI with a NULL `info` succeeds and returns the pinned outputs."""
    pin = _pin(env_id)
    out = rollout(emu_lib, env_id, dev=True)
    for k in pin:
        assert np.array_equal(out[k], pin[k]), k
    task, coop = PATHS[env_id]
    env = make_env(env_id, emu_lib)
    env.reset()
    sim = env.id
    a = np.ascontiguousarray(np.random.default_rng(17).uniform(-1, 1, size=(N_ENVS, 7 + (int(sim._coop_params.n_ctrl) if coop else 0))).astype(np.float32))
    outs = sim._step_outputs(task, coop)[:-1]
    fn = emu_lib.ag_coop_step_host if coop else getattr(emu_lib, 'ag_%s_step_host' % task)
    assert fn(sim.h, a.ctypes.data_as(C.c_void_p), *[o.ctypes.data_as(C.c_void_p) for o in outs], None) == 0, emu_lib.ag_last_error()
    for k, o in zip(('obs', 'obs_h', 'reward', 'done') if coop else ('obs', 'reward', 'done'), outs):
        assert np.array_equal(o, pin[k][0]), k
    env.close()


@pytest.mark.gpu
@pytest.mark.parametrize('env_id', list(PATHS))
def test_graph_replay_matches_direct_launches_cuda(gpu_lib, env_id, monkeypatch):
    graph = rollout(gpu_lib, env_id)
    monkeypatch.setenv('AG_GRAPH', '0')             # read by ag_create
    direct = rollout(gpu_lib, env_id)
    for k in graph:
        assert np.array_equal(graph[k], direct[k]), k
    assert np.array_equal(graph['launches'], _pin(env_id)['launches'])
