#!/usr/bin/env python3
"""Diagnostic: one SHA-256 per env id over everything the fused step kernels and the read-back kernels produce, for showing that a
change to the kernels' source leaves their results bit for bit the same: run it from a checkout of each commit and compare.

The eight pinned ids run the seeded rollout of tests/golden/make_golden_fused_step_pin.py (observations, rewards, dones, info,
launch counts, final state); DrinkingJaco-v1 replays its golden rollout (one particle swallowed, one spilled) and then reads
back link states, contacts and closest points.  Then every registered id's env API at 1 and 2 envs: what `reset`, `step`,
`step_fused` and `step_reference_api` return, Python types and dict / list structure included.

usage: python tools/fused_step_digest.py [library]     (default: the CUDA library; or tests/kernel_harness/libagphys_emu.so)"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, 'tests', 'golden')]


def digest(arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def drinking(lib):
    from tests.test_drinking_fused import G, N_GOLDEN_STEPS, _golden_sim, _inject
    db, sim = _golden_sim(lib)
    out = []
    for t, a in enumerate(G['actions'][:N_GOLDEN_STEPS]):
        _inject(db, sim, t)
        out += list(sim.drinking_step_host(np.asarray(a, dtype=np.float32)[None])) + list(sim.drinking_get_state())
    out += list(sim.get_link_states(np.arange(db.scene.n_links)).values()) + [sim.contact_force_sum(db.tool)]
    for hb in db.humans.values():             # the env's person and the switched-off one
        out += list(sim.get_contacts(hb)) + list(sim.closest_points(db.tool, hb, 0.5))
    out.append(sim.state_get())
    sim.close()
    return digest(out)


def surface(x, h):
    """Feeds `x` into `h`: the Python type and the dict / list / tuple structure as well as every array's dtype, shape and bytes."""
    h.update(type(x).__name__.encode())
    if isinstance(x, dict):
        for k, v in x.items():
            h.update(repr(k).encode())
            surface(v, h)
    elif isinstance(x, (list, tuple)):
        h.update(str(len(x)).encode())
        for v in x:
            surface(v, h)
    elif isinstance(x, (np.ndarray, np.generic)):
        h.update(str(x.dtype).encode() + str(x.shape).encode() + np.ascontiguousarray(x).tobytes())
    else:
        h.update(repr(x).encode())


def env_api(lib, env_id, n=2, n_steps=3):
    """`reset`, then `step`, `step_fused` and `step_reference_api` three times each (the last two where the id has them), with
    seeded actions, on `env_id`'s env at `n` envs of both genders.  A RuntimeError (step_fused of a single-agent id) is hashed
    as such."""
    from assistive_gym_b200 import envs
    env = envs.make(env_id, n_envs=n, **({'toc_attempts': 6} if env_id.startswith('Dressing') else {}))
    env._sim_lib = lib
    batch = next(getattr(env, a) for a in ('_fb', '_sb', '_bb', '_db') if hasattr(env, a))
    sample = batch.sample

    def both_genders(*a, **kw):
        s = sample(*a, **kw)
        s['male'][:] = np.arange(n) % 2
        return s
    batch.sample = both_genders
    h = hashlib.sha256()
    surface(env.reset(), h)
    rng = np.random.default_rng(5)
    coop = bool(env.human.controllable)
    for name in ('step', 'step_fused', 'step_reference_api'):
        if not hasattr(env, name):
            continue
        for _ in range(n_steps):
            a = rng.uniform(-1, 1, size=(n, env.action_space.shape[0])).astype(np.float32)
            if coop and name != 'step_reference_api':
                a = {'robot': a[:, :env.action_robot_len], 'human': a[:, env.action_robot_len:]}
            try:
                surface(getattr(env, name)(a), h)
            except RuntimeError as e:
                surface(str(e), h)
    env.close()
    return h.hexdigest()


def main():
    from assistive_gym_b200 import capi, envs
    from make_golden_fused_step_pin import PATHS, rollout
    lib = capi.load_library(*sys.argv[1:2])
    for env_id in PATHS:
        out = rollout(lib, env_id)
        print(env_id, digest(out[k] for k in sorted(out)), flush=True)
    print('DrinkingJaco-v1', drinking(lib), flush=True)
    for env_id in envs.ENV_REGISTRY:
        for n in (1, 2):
            print(env_id, 'env API, n_envs=%d' % n, env_api(lib, env_id, n), flush=True)


if __name__ == '__main__':
    main()
