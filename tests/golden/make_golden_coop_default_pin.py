"""Pin of the co-optimisation ids with default arguments, one id per task: reset plus 10 fused steps (`step_fused`) at 4 envs, on
the kernel bodies compiled for the host.  Taken from the commit before `human_impairment` existed, so that
tests/test_coop_tremor.py can show the default draw and step are bit for bit what they were.

usage (from a checkout of that commit): python tests/golden/make_golden_coop_default_pin.py tests/kernel_harness/libagphys_emu.so out.npz"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
IDS = ['FeedingJacoHuman-v1', 'ScratchItchJacoHuman-v1', 'BedBathingSawyerHuman-v1', 'DressingPR2Human-v1']
N, STEPS = 4, 10


def rollout(lib, env_id):
    from assistive_gym_b200 import envs
    env = envs.make(env_id, n_envs=N, seed=11, **(dict(toc_attempts=6) if env_id.startswith('Dressing') else {}))
    env._sim_lib = lib
    o = env.reset()
    out = [o['robot'], o['human']]
    rng = np.random.default_rng(3)
    k = env.action_human_len
    for _ in range(STEPS):
        r = env.step_fused({'robot': rng.uniform(-1, 1, size=(N, 7)).astype(np.float32), 'human': rng.uniform(-1, 1, size=(N, k)).astype(np.float32)})
        out += [r[0]['robot'], r[0]['human'], r[1]['robot'], r[2]['robot']]
    env.close()
    return out


def main():
    from assistive_gym_b200 import capi
    lib = capi.load_library(sys.argv[1])
    res = {}
    for env_id in IDS:
        for i, a in enumerate(rollout(lib, env_id)):
            res['%s_%03d' % (env_id, i)] = np.asarray(a)
    np.savez_compressed(sys.argv[2], **res)


if __name__ == '__main__':
    main()
