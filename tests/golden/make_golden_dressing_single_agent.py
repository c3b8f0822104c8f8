"""Pin of the single-agent DressingPR2-v1 path: the batched reset (random draws, robot base pose, cloth placement, a short settle)
and four fused steps of `ag_dressing_step_host` on the kernel bodies compiled for the host, from a fixed seed.  Generated before
DressingPR2Human-v1 (the co-optimisation id) was added, so that tests/test_dressing_coop.py can show that the new id leaves the
single-agent id bit for bit as it was: the same draws, the same template, the same kernels.
Output: tests/golden/dressing_single_agent_pin.npz.

usage: python tests/golden/make_golden_dressing_single_agent.py   (after tests/kernel_harness/build.sh)"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

N_ENVS, N_STEPS, SEED = 2, 4, 13


def rollout(lib):
    """(sample, reset state, cloth after the settle, per-step obs / reward / done / info, final state and cloth) of DressingPR2-v1 on `lib`."""
    from assistive_gym_b200.dressing_batch import DressingBatch
    from assistive_gym_b200.sim import BatchSim
    db = DressingBatch()
    sim = BatchSim(db.scene, DressingBatch.config(), N_ENVS, _lib=lib)
    rng = np.random.default_rng(SEED)
    smp = db.reset(sim, rng, attempts=6, settle_steps=2)
    out = {('sample_' + k): np.asarray(v) for k, v in smp.items()}
    out.update(reset_state=sim.state_get(), reset_cloth=sim.cloth_get_state()[0], obs=[], reward=[], done=[], info=[])
    db.start_fused(sim, smp)
    for _ in range(N_STEPS):
        a = rng.uniform(-1, 1, size=(N_ENVS, 7)).astype(np.float32)
        o, r, d, info = sim.dressing_step_host(a)
        out['obs'].append(o); out['reward'].append(r); out['done'].append(d); out['info'].append(info)
    out['final_state'] = sim.state_get()
    out['final_cloth'] = sim.cloth_get_state()[0]
    sim.close()
    return {k: np.asarray(v) for k, v in out.items()}


def main():
    from assistive_gym_b200 import capi
    lib = capi.load_library(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'tests', 'kernel_harness', 'libagphys_emu.so'))
    out = rollout(lib)
    np.savez_compressed(os.path.join(HERE, 'dressing_single_agent_pin.npz'), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main()
