"""Pin of every fused env-step entry point: the four single-agent ids through `*_step_host` and the four co-optimisation ids
through `coop_step_host`, on the kernel bodies compiled for the host, from a fixed seed.  4 envs of both genders; for the
co-optimisation ids half of them at limit scale 0.5.  Per step: both observations, reward, done, info and the kernel-launch
count; at the end a SHA-256 of `state_get()`.  Generated before the host halves of the five step paths were merged into one,
so that tests/test_fused_step_paths.py can show that every path computes and launches exactly what it did.
Output: tests/golden/fused_step_pin.npz.

usage: python tests/golden/make_golden_fused_step_pin.py   (after tests/kernel_harness/build.sh)"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

N_ENVS, N_STEPS, SEED = 4, 6, 17
# env id -> (task name of the BatchSim entry points, co-optimisation)
PATHS = {'FeedingJaco-v1': ('feeding', False), 'ScratchItchJaco-v1': ('scratch', False),
         'BedBathingSawyer-v1': ('bathing', False), 'DressingPR2-v1': ('dressing', False),
         'FeedingJacoHuman-v1': ('feeding', True), 'ScratchItchJacoHuman-v1': ('scratch', True),
         'BedBathingSawyerHuman-v1': ('bathing', True), 'DressingPR2Human-v1': ('dressing', True)}


def make_env(env_id, lib, n=N_ENVS, seed=SEED):
    """`env_id` on `lib`, reset draws patched to both genders (and, with a controllable person, limit scale 0.5 in half the envs)."""
    from assistive_gym_b200 import envs
    coop = PATHS[env_id][1]
    env = envs.make(env_id, n_envs=n, seed=seed, **({'toc_attempts': 6} if env_id.startswith('Dressing') else {}))
    env._sim_lib = lib
    batch = next(getattr(env, a) for a in ('_fb', '_sb', '_bb', '_db') if hasattr(env, a))
    sample = batch.sample

    def both_genders(*a, **kw):
        s = sample(*a, **kw)
        s['male'][:] = np.arange(n) % 2
        if coop:
            lim = np.arange(n) % 4 < 2
            s['impairment'] = np.where(lim, 1, s['impairment']).astype(np.int32)
            s['limit_scale'] = np.where(lim, 0.5, s['limit_scale'])
        return s
    batch.sample = both_genders
    return env


def step_dev(sim, task, coop, a):
    """One step through `*_step_dev` / `coop_step_dev` with host buffers (the host-compiled library reads them directly)."""
    n = sim.n
    ro, ho = {'feeding': (25, 23), 'scratch': (30, 34), 'bathing': (24, 28), 'dressing': (24, 28)}[task]
    obs, obs_h = np.zeros((n, ro), np.float32), np.zeros((n, ho), np.float32)
    rew, done, info = np.zeros(n, np.float32), np.zeros(n, np.float32), np.zeros((n, 4), np.float32)
    p = lambda x: x.ctypes.data
    if coop:
        sim.coop_step_dev(p(a), p(obs), p(obs_h), p(rew), p(done), p(info))
        return obs, obs_h, rew, done, info
    getattr(sim, task + '_step_dev')(p(a), p(obs), p(rew), p(done), p(info))
    return obs, rew, done, info


def rollout(lib, env_id, dev=False):
    """Per-step outputs and launch counts of `env_id`'s fused step, and the final state's SHA-256; `dev` steps through the
    device-pointer entry point instead of the host-buffer one."""
    task, coop = PATHS[env_id]
    env = make_env(env_id, lib)
    env.reset()
    sim = env.id
    width = 7 + (int(sim._coop_params.n_ctrl) if coop else 0)
    rng = np.random.default_rng(SEED)
    keys = ('obs', 'obs_h', 'reward', 'done', 'info') if coop else ('obs', 'reward', 'done', 'info')
    out = {k: [] for k in keys + ('launches',)}
    for _ in range(N_STEPS):
        a = np.ascontiguousarray(rng.uniform(-1, 1, size=(N_ENVS, width)).astype(np.float32))
        l0 = sim.kernel_launches()
        if dev:
            r = step_dev(sim, task, coop, a)
        else:
            r = sim.coop_step_host(a) if coop else getattr(sim, task + '_step_host')(a)
        out['launches'].append(sim.kernel_launches() - l0)
        for k, v in zip(keys, r):
            out[k].append(v)
    out = {k: np.asarray(v) for k, v in out.items()}
    out['state_sha256'] = np.array(hashlib.sha256(np.ascontiguousarray(sim.state_get()).tobytes()).hexdigest())
    env.close()
    return out


def main():
    from assistive_gym_b200 import capi
    lib = capi.load_library(os.path.join(ROOT, 'tests', 'kernel_harness', 'libagphys_emu.so'))
    pin = {}
    for env_id in PATHS:
        for k, v in rollout(lib, env_id).items():
            pin[env_id + '/' + k] = v
        print(env_id, 'launches per step', pin[env_id + '/launches'])
    np.savez_compressed(os.path.join(HERE, 'fused_step_pin.npz'), **pin)


if __name__ == '__main__':
    main()
