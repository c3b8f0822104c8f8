"""Pin of the single-agent BedBathingSawyer-v1 path: the reset state and ten fused steps of `BedBathingSawyerEnv` on the kernel
bodies compiled for the host, from a fixed seed.  Generated before BedBathingSawyerHuman-v1 (the co-optimisation id) was added,
so that tests/test_bathing_coop.py can show that the new id leaves the single-agent id bit for bit as it was: the same random
draws at reset, the same template, the same kernels.  Output: tests/golden/bathing_single_agent_pin.npz.

usage: python tests/golden/make_golden_bathing_single_agent.py   (after tests/kernel_harness/build.sh)"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

N_ENVS, N_STEPS, SEED = 4, 10, 11


def rollout(lib):
    """(reset state, reset obs, per-step obs / reward / done / info, final state) of BedBathingSawyer-v1 on `lib`."""
    from assistive_gym_b200 import envs
    env = envs.make('BedBathingSawyer-v1', n_envs=N_ENVS, seed=SEED)
    env._sim_lib = lib
    obs0 = env.reset()
    state0 = env.id.state_get()
    rng = np.random.default_rng(SEED)
    out = dict(reset_state=state0, reset_obs=np.asarray(obs0, dtype=np.float32), male=env.male.astype(np.int32), obs=[], reward=[], done=[], total_force=[], task_success=[])
    for _ in range(N_STEPS):
        a = rng.uniform(-1, 1, size=(N_ENVS, 7)).astype(np.float32)
        o, r, d, info = env.step(a)
        out['obs'].append(o); out['reward'].append(r); out['done'].append(d)
        out['total_force'].append(info['total_force_on_human']); out['task_success'].append(info['task_success'])
    out['final_state'] = env.id.state_get()
    env.close()
    return {k: np.asarray(v) for k, v in out.items()}


def main():
    from assistive_gym_b200 import capi
    lib = capi.load_library(os.path.join(ROOT, 'tests', 'kernel_harness', 'libagphys_emu.so'))
    out = rollout(lib)
    np.savez_compressed(os.path.join(HERE, 'bathing_single_agent_pin.npz'), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == '__main__':
    main()
