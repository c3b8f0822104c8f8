#!/usr/bin/env python3
"""GPU box: ScratchItch on each robot -- ScratchItchJaco-v1 and ScratchItchJacoHuman-v1 for comparison, ScratchItchSawyer-v1,
ScratchItchPR2-v1 and the co-optimisation ids ScratchItchSawyerHuman-v1, ScratchItchPR2Human-v1 -- through the public env (`envs.make`), device-timed; not the headline metric.

One JSON line: the card and its power limit (read in the same run) and per id: the env's full `reset()` (person, TOC base-pose search
or the mounted arm's IK, arming the fused step), the graph-replayed device step (`scratch_step_dev` or
`coop_step_dev`, CUDA events) and the host-buffer step (`scratch_step_host` / `coop_step_host`, host clock; the call ends in a stream
synchronise) over the same number of steps after a warm-up, the three costliest kernels from a separate profiled pass, contacts and PGS
iterations per env, overflowed envs and the sim's device memory.

usage: python tools/gpu_scratch_robots_bench.py [--n 4096] [--steps 50] [--warmup 10] [--profile-steps 3] [--ids A,B] [--out FILE]"""
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

from assistive_gym_b200 import envs  # noqa: E402

IDS = ['ScratchItchJaco-v1', 'ScratchItchJacoHuman-v1', 'ScratchItchSawyer-v1', 'ScratchItchPR2-v1', 'ScratchItchSawyerHuman-v1', 'ScratchItchPR2Human-v1']


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader,nounits', '-i', '0'],
                       capture_output=True, text=True)
    name, power, sm = [x.strip() for x in q.stdout.strip().splitlines()[0].split(',')]
    return {'name': name, 'power_limit_w': float(power), 'sm_max_mhz': float(sm)}


def measure(env_id, n, K, W, profile_steps):
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    env = envs.make(env_id, n_envs=n, seed=1001)
    t0 = time.time()
    env.reset()
    torch.cuda.synchronize()
    reset_s = time.time() - t0
    sim = env.id
    sim_bytes = free0 - torch.cuda.mem_get_info()[0]
    overflow_reset = sim.overflow_count()
    coop = bool(env.human.controllable)
    k = 7 + (env.action_human_len if coop else 0)
    dev = torch.device('cuda')
    stream = torch.cuda.ExternalStream(sim.stream_ptr())
    g = torch.Generator(device=dev).manual_seed(0)
    act = torch.rand((W + K, n, k), device=dev, generator=g) * 2 - 1
    obs, obs_h = torch.zeros((n, env.obs_robot_len), device=dev), torch.zeros((n, max(env.obs_human_len, 1)), device=dev)
    rew, done, info = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros((n, 4), device=dev)

    def step_dev(a):
        if coop:
            sim.coop_step_dev(a.data_ptr(), obs.data_ptr(), obs_h.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
        else:
            sim.scratch_step_dev(a.data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    torch.cuda.synchronize()
    for i in range(W):
        step_dev(act[i])
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for i in range(K):
        step_dev(act[W + i])
    b.record(stream)
    torch.cuda.synchronize()
    dev_ms = a.elapsed_time(b) / K
    finite = bool(torch.isfinite(obs).all()) and bool(torch.isfinite(rew).all())
    cnt, it = sim.solver_stats()
    overflow = sim.overflow_count()
    act_h = np.random.default_rng(1).uniform(-1, 1, size=(K, n, k)).astype(np.float32)
    host = sim.coop_step_host if coop else sim.scratch_step_host
    host(act_h[0])
    t0 = time.perf_counter()
    for i in range(K):
        host(act_h[i])
    host_ms = (time.perf_counter() - t0) * 1e3 / K
    sim.profile_get()
    sim.profile_enable(True)
    for i in range(profile_steps):
        step_dev(act[i])
    prof = sim.profile_get()
    sim.profile_enable(False)
    total = sum(ms for ms, _ in prof.values())
    top = {kk: round(ms / total, 3) for kk, (ms, c) in sorted(prof.items(), key=lambda kv: -kv[1][0])[:3]}
    sb = env._sb
    out = {'reset_s': reset_s, 'device_step_ms': dev_ms, 'device_env_steps_per_s': n / dev_ms * 1e3,
           'host_step_ms': host_ms, 'host_env_steps_per_s': n / host_ms * 1e3,
           'episode_device_s': 200 * dev_ms / 1e3,
           'contacts_per_env_mean': float(cnt.mean()), 'contacts_per_env_max': int(cnt.max()), 'max_contacts': int(sim.cfg.max_contacts),
           'pgs_iters_mean': float(it.mean()), 'overflow_envs_reset': int(overflow_reset), 'overflow_envs_steps': int(overflow),
           'sim_device_bytes': int(sim_bytes), 'finite': finite, 'profiled_ms_per_step': total / profile_steps, 'top_kernels_share': top}
    if getattr(sb, 'goals_reached', None) is not None:
        out['toc_start_goal_reached'] = float((np.asarray(sb.goals_reached) >= 1).mean())
        out['reset_unresolved_envs'] = int(sb.unresolved)
    env.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=4096)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--profile-steps', type=int, default=3)
    ap.add_argument('--ids', default=','.join(IDS))
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this measurement needs the GPU')
    res = {'workload': 'ScratchItch on each robot, fused step', 'gpu': gpu_info(), 'n_envs': args.n, 'steps': args.steps, 'warmup': args.warmup, 'ids': {}}
    for env_id in args.ids.split(','):
        res['ids'][env_id] = measure(env_id, args.n, args.steps, args.warmup, args.profile_steps)
        print(env_id, json.dumps(res['ids'][env_id]), file=sys.stderr, flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
