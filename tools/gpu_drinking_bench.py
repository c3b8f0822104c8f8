#!/usr/bin/env python3
"""GPU box: fused Drinking step throughput (ag_drinking_step_*), device-timed; not the headline metric.

One JSON line: the card and its power limit (read in the same run), reset time, the graph-replayed device step
(`drinking_step_dev`, CUDA events) and the host-buffer step (`drinking_step_host`, host clock; the call ends in a stream
synchronise) over the same number of steps after a warm-up, a per-kernel split from a separate profiled pass, contacts and PGS
iterations per env, overflowed envs and the sim's device memory.  With `--ids` one line per id (DrinkingJaco-v1, DrinkingSawyer-v1,
DrinkingPR2-v1; the TOC ids also report the envs their placement left colliding).

usage: python tools/gpu_drinking_bench.py [--ids DrinkingJaco-v1,...] [--n 4096] [--steps 100] [--warmup 10] [--profile-steps 5] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from assistive_gym_b200.envs import ENV_REGISTRY  # noqa: E402
from assistive_gym_b200.envs.drinking import drinking_batch_for  # noqa: E402
from assistive_gym_b200.sim import BatchSim  # noqa: E402


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits', '-i', '0'],
                       capture_output=True, text=True)
    name, power, sm = [x.strip() for x in q.stdout.strip().splitlines()[0].split(',')]
    return {'name': name, 'power_limit_w': float(power), 'sm_max_mhz': float(sm)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ids', default='DrinkingJaco-v1', help='comma-separated Drinking ids, one JSON line each')
    ap.add_argument('--n', type=int, default=4096)
    ap.add_argument('--steps', type=int, default=100)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--profile-steps', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this measurement needs the GPU')
    lines = [bench(env_id, args) for env_id in args.ids.split(',')]
    if args.out:
        with open(args.out, 'w') as f:
            f.write(''.join(line + '\n' for line in lines))


def bench(env_id, args):
    n, K, W = args.n, args.steps, args.warmup
    gpu = gpu_info()
    db = drinking_batch_for(ENV_REGISTRY[env_id]().robot)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    sim = BatchSim(db.scene, db.config(), n)
    t0 = time.time()
    s = db.reset(sim, np.random.default_rng(0), settle_steps=50, impairment='no_tremor')
    db.start_fused(sim, s)
    reset_s = time.time() - t0
    torch.cuda.synchronize()
    sim_bytes = free0 - torch.cuda.mem_get_info()[0]
    overflow_reset = sim.overflow_count()

    dev = torch.device('cuda')
    stream = torch.cuda.ExternalStream(sim.stream_ptr())
    g = torch.Generator(device=dev).manual_seed(0)
    act = torch.rand((W + K, n, 7), device=dev, generator=g) * 2 - 1
    obs, rew, done, info = torch.zeros((n, 25), device=dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros((n, 4), device=dev)
    torch.cuda.synchronize()
    for i in range(W):
        sim.drinking_step_dev(act[i].data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for i in range(K):
        sim.drinking_step_dev(act[W + i].data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    b.record(stream)
    torch.cuda.synchronize()
    dev_ms = a.elapsed_time(b) / K
    finite = bool(torch.isfinite(obs).all()) and bool(torch.isfinite(rew).all())
    cnt, it = sim.solver_stats()
    ts, w, wa = sim.drinking_get_state()
    in_play = np.array([bin(int(x)).count('1') for x in w])

    act_h = np.random.default_rng(1).uniform(-1, 1, size=(K, n, 7)).astype(np.float32)
    sim.drinking_step_host(act_h[0])
    t0 = time.perf_counter()
    for i in range(K):
        sim.drinking_step_host(act_h[i])
    host_ms = (time.perf_counter() - t0) * 1e3 / K

    sim.profile_get()
    sim.profile_enable(True)
    for i in range(args.profile_steps):
        sim.drinking_step_dev(act[i].data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    prof = sim.profile_get()
    sim.profile_enable(False)
    total = sum(ms for ms, _ in prof.values())
    kernels = {k: {'ms_per_step': ms / args.profile_steps, 'launches_per_step': c / args.profile_steps, 'share': ms / total}
               for k, (ms, c) in sorted(prof.items(), key=lambda kv: -kv[1][0])}
    overflow = sim.overflow_count()
    out = {'workload': '%s fused step' % env_id, 'gpu': gpu, 'n_envs': n, 'steps': K, 'warmup': W,
           'num_substeps': 4, 'frame_skip': 5, 'num_solver_iters': 10, 'max_contacts': 512,
           'reset_s': reset_s, 'device_step_ms': dev_ms, 'device_env_steps_per_s': n / dev_ms * 1e3,
           'host_step_ms': host_ms, 'host_env_steps_per_s': n / host_ms * 1e3,
           'contacts_per_env_mean': float(cnt.mean()), 'contacts_per_env_max': int(cnt.max()), 'pgs_iters_mean': float(it.mean()),
           'overflow_envs_reset': overflow_reset, 'overflow_envs_steps': overflow, 'sim_device_bytes': int(sim_bytes),
           'particles_in_play_mean': float(in_play.mean()), 'task_success_mean': float(ts.mean()), 'finite': finite,
           'profiled_steps': args.profile_steps, 'profiled_ms_per_step': total / args.profile_steps, 'kernels': kernels}
    if hasattr(db, 'unresolved'):
        out['toc_envs_left_colliding'] = int(db.unresolved)
    line = json.dumps(out)
    print(line, flush=True)
    sim.close()
    return line


if __name__ == '__main__':
    main()
