"""Edge cases and size-independent properties of the batched step (host-compiled kernel bodies on CPU,
the CUDA build on the H100): empty row streams, ragged batch sizes, batch-position invariance, state
round trips, contact-budget overflow, ABI error behaviour."""
import numpy as np
import pytest

from assistive_gym_b200 import capi
from assistive_gym_b200.scene import SceneBuilder
from assistive_gym_b200.sim import BatchSim


def _falling_sphere_scene(with_plane):
    b = SceneBuilder()
    b.set_gravity([0, 0, -9.81])
    if with_plane:
        b.load_urdf('plane')
    sh = b.create_collision_shape('sphere', radius=0.05)
    ball = b.create_multibody(base_mass=0.3, base_shape=sh, base_pos=[0, 0, 2.0], name='ball')
    return b.finalize(), ball


def _check_empty_stream(mk):
    """A single body, nothing to collide with: zero constraint rows (the solver's stream is empty) and the
    integrator alone reproduces symplectic-Euler free fall, z_n = z0 - g dt^2 n (n + 1) / 2."""
    scene, ball = _falling_sphere_scene(False)
    cfg = capi.default_config(linear_damping=0, angular_damping=0)
    sim = mk(scene, cfg, 3)
    sim.step(20)
    cnt, it = sim.solver_stats()
    assert np.all(cnt == 0) and np.all(it == 0)
    z = 2.0 - 9.81 * 0.02 ** 2 * 20 * 21 / 2
    st = sim.state_get()
    assert np.abs(st[:, ball * 13 + 2] - z).max() < 2e-5, (st[:, ball * 13 + 2], z)
    assert sim.overflow_count() == 0


def _check_rest_on_plane(mk):
    """Sphere dropped on the plane comes to rest at its radius; normal force = m g (within solver slop)."""
    scene, ball = _falling_sphere_scene(True)
    cfg = capi.default_config()
    sim = mk(scene, cfg, 2)
    sim.set_base_pose(ball, np.tile([0, 0, 0.0505], (2, 1)), np.tile([0, 0, 0, 1.0], (2, 1)))
    sim.forward_kinematics()
    sim.step(150)
    st = sim.state_get()
    assert np.abs(st[:, ball * 13 + 2] - 0.05).max() < 2e-3
    f = sim.contact_force_sum(ball)
    assert np.abs(f - 0.3 * 9.81).max() < 0.05 * 0.3 * 9.81, f


def _check_batch_invariance(fb, mk):
    """An env's trajectory does not depend on the batch size or on its position in the batch (ragged sizes
    included): env 0 of N = 1 == env 2 of N = 3 == env 32 of N = 33, bit for bit."""
    cfg = capi.default_config()
    rng = np.random.default_rng(3)
    s1 = fb.sample(1, rng)
    outs = []
    for n, pos in ((1, 0), (3, 2), (33, 32)):
        s = {k: np.repeat(v, n, axis=0).copy() for k, v in s1.items()}
        filler = fb.sample(n, np.random.default_rng(100 + n))
        for k in s:                                    # every other env gets different randomisation
            for e in range(n):
                if e != pos:
                    s[k][e] = filler[k][e]
        sim = mk(fb.scene, cfg, n)
        fb.reset(sim, np.random.default_rng(7), settle_steps=0, sample=s)
        if n == 1:
            st0 = sim.state_get()[0].copy()
        st = sim.state_get(); st[pos] = st0; sim.state_set(st)      # identical start state (IK is not batch-invariant)
        q = sim.get_joint_states(fb.arm_links)[0]
        sim.set_motor_targets(fb.arm_links, np.tile(q[pos], (n, 1)) + 0.1)
        sim.step(15)
        outs.append(sim.state_get()[pos].copy())
        assert np.all(np.isfinite(sim.state_get()))
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2])


def _check_state_roundtrip(fb, mk):
    """state_get/state_set are inverse, and stepping twice from the same state gives the same bits."""
    cfg = capi.default_config()
    sim = mk(fb.scene, cfg, 4)
    fb.reset(sim, np.random.default_rng(11), settle_steps=5)
    st = sim.state_get()
    sim.state_set(st)
    assert np.array_equal(sim.state_get(), st)
    sim.step(5)
    a = sim.state_get()
    sim.state_set(st)
    sim.step(5)
    assert np.array_equal(sim.state_get(), a)


def _check_overflow_determinism(fb, mk):
    """Contact budget too small (64 for ~80 contacts while the food settles; the raw contact buffer and the
    candidate list hold 4x the budget): the surviving contacts are chosen by key, not by the order in which
    threads happened to append them, so runs from the same state agree bit for bit; the flag is sticky until read."""
    cfg = capi.default_config(max_contacts=64)
    sim = mk(fb.scene, cfg, 64)
    fb.reset(sim, np.random.default_rng(2), settle_steps=0)
    st = sim.state_get()
    sim.step(10)
    a = sim.state_get()
    assert sim.overflow_count() >= 32          # most envs exceed 64 contacts while the food settles
    for _ in range(3):
        sim.state_set(st)
        sim.step(10)
        assert np.array_equal(sim.state_get(), a)
    assert np.all(np.isfinite(a))


def _check_abi_errors(lib):
    scene, ball = _falling_sphere_scene(True)
    cfg = capi.default_config()
    import ctypes as C
    desc = scene.as_ctypes()
    assert not lib.ag_create(C.byref(desc), C.byref(cfg), 0, 0)          # zero envs
    assert lib.ag_last_error()
    sim = BatchSim(scene, cfg, 2, _lib=lib) if lib is not None else BatchSim(scene, cfg, 2)
    with pytest.raises(RuntimeError):
        sim.get_joint_states([10 ** 6])                                   # link id out of range
    with pytest.raises(RuntimeError):
        sim.set_motor([10 ** 6], 1, target=np.zeros((2, 1)), kp=[0.1], kd=[1.0], max_force=[1.0])


# ------------------------------------------------------------------ CPU: host-compiled kernel bodies
@pytest.fixture(scope='module')
def mk_cpu(emu_lib):
    return lambda scene, cfg, n: BatchSim(scene, cfg, n, _lib=emu_lib)


def test_empty_stream_cpu(mk_cpu):
    _check_empty_stream(mk_cpu)


def test_rest_on_plane_cpu(mk_cpu):
    _check_rest_on_plane(mk_cpu)


def test_batch_invariance_cpu(feeding, mk_cpu):
    _check_batch_invariance(feeding, mk_cpu)


def test_state_roundtrip_cpu(feeding, mk_cpu):
    _check_state_roundtrip(feeding, mk_cpu)


def test_overflow_determinism_cpu(feeding, mk_cpu):
    _check_overflow_determinism(feeding, mk_cpu)


def test_abi_errors_cpu(emu_lib):
    _check_abi_errors(emu_lib)


# ------------------------------------------------------------------ GPU: the CUDA build
@pytest.fixture(scope='module')
def mk_gpu(gpu_lib):
    return lambda scene, cfg, n: BatchSim(scene, cfg, n, device=0)


@pytest.mark.gpu
def test_empty_stream_gpu(mk_gpu):
    _check_empty_stream(mk_gpu)


@pytest.mark.gpu
def test_rest_on_plane_gpu(mk_gpu):
    _check_rest_on_plane(mk_gpu)


@pytest.mark.gpu
def test_batch_invariance_gpu(feeding, mk_gpu):
    _check_batch_invariance(feeding, mk_gpu)


@pytest.mark.gpu
def test_state_roundtrip_gpu(feeding, mk_gpu):
    _check_state_roundtrip(feeding, mk_gpu)


@pytest.mark.gpu
def test_overflow_determinism_gpu(feeding, mk_gpu):
    _check_overflow_determinism(feeding, mk_gpu)


@pytest.mark.gpu
def test_abi_errors_gpu(gpu_lib):
    _check_abi_errors(gpu_lib)


@pytest.mark.gpu
def test_entry_points_keep_the_callers_device(feeding, mk_gpu):
    """ADVICE r1: every entry point runs on the sim's GPU and restores the caller's current device."""
    import torch
    if torch.cuda.device_count() < 2:
        # one GPU: the guard must at least be a no-op that leaves device 0 current
        sim = mk_gpu(feeding.scene, capi.default_config(), 4)
        feeding.reset(sim, np.random.default_rng(0), settle_steps=1)
        assert torch.cuda.current_device() == 0
        return
    torch.cuda.set_device(0)
    from assistive_gym_b200.sim import BatchSim
    sim = BatchSim(feeding.scene, capi.default_config(), 4, device=1)
    feeding.reset(sim, np.random.default_rng(0), settle_steps=1)
    sim.step(2)
    assert np.all(np.isfinite(sim.state_get()))
    assert torch.cuda.current_device() == 0
