"""Throughput of the co-optimisation envs (FeedingJacoHuman-v1, ScratchItchJacoHuman-v1, BedBathingSawyerHuman-v1, DressingPR2Human-v1) on one GPU: the fused device step
(`step_fused` / ag_coop_step_dev, graph-replayed) against the per-call `step` (take_step + _get_obs through the C ABI, with the
host round trips of enforce_joint_limits / the realistic-arm-limit classifier after every substep), at the same batch size.

Prints one JSON line per id: fused env-steps/s (CUDA events around the timed steps after warm-up), per-call env-steps/s (a host
clock around fewer steps, each of which ends in device-to-host reads), k_coop_limits ms per launch (ag_profile_get, in a
separate profiled run of the fused step; for BedBathing also k_bath_track, which re-places the wiping targets on the moving arm)
and the card's name and power limit, read in the same run.  Without --n, each id runs at its bench size: 4096 envs, and 2048 for
DressingPR2Human-v1 (the Dressing bench size); its per-call leg runs at 256 envs (`percall_note`), because the per-call Dressing step
evaluates the sleeve-on-arm reward env by env on the host.

    python tools/gpu_coop_bench.py --n 4096 --steps 50 --warmup 5 --percall-steps 3 [--ids BedBathingSawyerHuman-v1] [--out profiles/h100_coop_bench.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


DEFAULT_N = {'DressingPR2Human-v1': 2048}
PERCALL_N = {'DressingPR2Human-v1': (256, 'the per-call Dressing step evaluates the sleeve-on-arm reward env by env on the host; measured at 256 envs')}


def card():
    import torch
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                         capture_output=True, text=True).stdout.strip()
    return dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=out)


def bench(env_id, n, steps, warmup, percall_steps, seed=1001):
    import torch
    from assistive_gym_b200 import envs
    env = envs.make(env_id, n_envs=n, seed=seed)
    t0 = time.perf_counter()
    env.reset()
    reset_s = time.perf_counter() - t0
    sim = env.id
    k = env.action_human_len
    dev = torch.device('cuda:0')
    ro, ho = env.obs_robot_len, env.obs_human_len
    obs_r, obs_h = torch.zeros(n, ro, device=dev), torch.zeros(n, ho, device=dev)
    rew, done, info = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, 4, device=dev)
    gen = torch.Generator(device=dev).manual_seed(seed)
    acts = [torch.rand(n, 7 + k, device=dev, generator=gen) * 2 - 1 for _ in range(8)]
    stream = torch.cuda.ExternalStream(sim.stream_ptr(), device=dev)
    torch.cuda.synchronize()

    def step(i):
        sim.coop_step_dev(acts[i % len(acts)].data_ptr(), obs_r.data_ptr(), obs_h.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for i in range(steps):
        step(i)
    e1.record(stream)
    e1.synchronize()
    fused_ms = e0.elapsed_time(e1) / steps
    finite = bool(torch.isfinite(obs_r).all() and torch.isfinite(obs_h).all() and torch.isfinite(rew).all())
    # per-kernel device time of the fused step (events around every launch: a separate, slower run)
    sim.profile_enable(True)
    sim.profile_get()
    for i in range(3):
        step(i)
    prof = sim.profile_get()
    sim.profile_enable(False)
    lim_ms, lim_n = prof.get('k_coop_limits', (0.0, 0))
    pgs_ms, pgs_n = prof.get('k_pgs', (0.0, 0))
    track = {}
    if 'k_bath_track' in prof:
        tr_ms, tr_n = prof['k_bath_track']
        track = dict(k_bath_track_ms_per_launch=round(tr_ms / max(tr_n, 1), 4), k_bath_track_launches_per_step=tr_n // 3)
    env.close()
    # the per-call path from the same kind of start state (a fresh reset), fewer steps; should it fail at this batch size, it is
    # measured at 1024 envs and the line says so (`percall_n_envs`, `percall_note`)
    percall_n, note = PERCALL_N.get(env_id, (n, None))
    try:
        percall_s = percall(env_id, percall_n, k, percall_steps, seed)
    except RuntimeError as ex:
        percall_n, note = 1024, 'per-call step fails at %d envs (%s); measured at 1024' % (n, ex)
        percall_s = percall(env_id, percall_n, k, percall_steps, seed)
    return dict(id=env_id, n_envs=n, fused_env_steps_per_s=round(n / (fused_ms * 1e-3), 1), fused_ms_per_step=round(fused_ms, 3),
                fused_steps_timed=steps, warmup=warmup, outputs_finite=finite, percall_n_envs=percall_n, percall_note=note,
                percall_env_steps_per_s=round(percall_n / percall_s, 1), percall_ms_per_step=round(percall_s * 1e3, 1), percall_steps_timed=percall_steps,
                fused_over_percall_env_steps=round((n / (fused_ms * 1e-3)) / (percall_n / percall_s), 1),
                k_coop_limits_ms_per_launch=round(lim_ms / max(lim_n, 1), 4), k_coop_limits_launches_per_step=lim_n // 3,
                k_pgs_ms_per_launch=round(pgs_ms / max(pgs_n, 1), 4), reset_s=round(reset_s, 2), **track)


def percall(env_id, n, k, steps, seed):
    import torch
    from assistive_gym_b200 import envs
    env = envs.make(env_id, n_envs=n, seed=seed)
    try:
        env.reset()
        rng = np.random.default_rng(seed)
        a = {'robot': rng.uniform(-1, 1, size=(n, 7)).astype(np.float32), 'human': rng.uniform(-1, 1, size=(n, k)).astype(np.float32)}
        env.step(a)                                       # warm-up: first calls grow the staging buffers
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            env.step(a)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / steps
    finally:
        env.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=None, help='envs per id (default: 4096; 2048 for DressingPR2Human-v1)')
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--percall-steps', type=int, default=3)
    ap.add_argument('--ids', default='FeedingJacoHuman-v1,ScratchItchJacoHuman-v1')
    ap.add_argument('--out', help='also append the lines to this file')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this measurement runs on the GPU only')
    c = card()
    for env_id in args.ids.split(','):
        n = args.n or DEFAULT_N.get(env_id, 4096)
        r = dict(bench(env_id, n, args.steps, args.warmup, args.percall_steps), **c)
        line = json.dumps(r)
        print(line, flush=True)
        if args.out:
            with open(args.out, 'a') as f:
                f.write(line + '\n')


if __name__ == '__main__':
    main()
