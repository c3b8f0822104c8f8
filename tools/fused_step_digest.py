#!/usr/bin/env python3
"""Diagnostic: one SHA-256 per env id over everything the fused step kernels and the read-back kernels produce, for showing that a
change to the kernels' source leaves their results bit for bit the same: run it from a checkout of each commit and compare.

The eight pinned ids run the seeded rollout of tests/golden/make_golden_fused_step_pin.py (observations, rewards, dones, info,
launch counts, final state); DrinkingJaco-v1 replays its golden rollout (one particle swallowed, one spilled) and then reads
back link states, contacts and closest points.

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


def main():
    from assistive_gym_b200 import capi
    from make_golden_fused_step_pin import PATHS, rollout
    lib = capi.load_library(*sys.argv[1:2])
    for env_id in PATHS:
        out = rollout(lib, env_id)
        print(env_id, digest(out[k] for k in sorted(out)), flush=True)
    print('DrinkingJaco-v1', drinking(lib), flush=True)


if __name__ == '__main__':
    main()
