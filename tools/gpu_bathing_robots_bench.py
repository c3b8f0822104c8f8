#!/usr/bin/env python3
"""GPU box: BedBathing on each robot -- BedBathingSawyer-v1 and BedBathingSawyerHuman-v1 for comparison, BedBathingPR2-v1 and
BedBathingPR2Human-v1 -- through the public env (`envs.make`), device-timed; not the headline metric.

The GPU is kept busy for `--gpu-warmup` seconds before the first id, so that no id is timed while the clocks ramp up, and the ids are
measured in `--rounds` rounds, every other round in reverse order, so that drift in the card's clock does not favour one id.

One JSON line: the card, its power limit and SM clock (read in the same run, before and after) and per id and round: the env's full
`reset()` (person, robot placement, arming the fused step), the graph-replayed device step (`bathing_step_dev` or `coop_step_dev`, CUDA
events) over `--steps` steps after `--warmup`, then the rest of a random-action episode of `--episode` steps in all, with the contacts
per env (mean of the per-step means, and the largest) read after each of those steps, the envs whose contact buffer overflowed, and
the sim's device memory; per id also the median rate over the rounds.

usage: python tools/gpu_bathing_robots_bench.py [--n 4096] [--steps 150] [--warmup 10] [--episode 200] [--rounds 2] [--gpu-warmup 10] [--ids A,B] [--out FILE]"""
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

IDS = ['BedBathingSawyer-v1', 'BedBathingSawyerHuman-v1', 'BedBathingPR2-v1', 'BedBathingPR2Human-v1']


def gpu_info():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader,nounits', '-i', '0'],
                       capture_output=True, text=True)
    name, power, sm_max, sm = [x.strip() for x in q.stdout.strip().splitlines()[0].split(',')]
    return {'name': name, 'power_limit_w': float(power), 'sm_max_mhz': float(sm_max), 'sm_mhz': float(sm)}


def warm_gpu(seconds):
    """Matrix products for `seconds`, so that the SM clock has reached its sustained value before anything is timed."""
    x = torch.randn(4096, 4096, device='cuda')
    t0 = time.time()
    while time.time() - t0 < seconds:
        for _ in range(20):
            x = torch.tanh(x @ x * 1e-3)
        torch.cuda.synchronize()


def measure(env_id, n, K, W, episode):
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
    act = torch.rand((episode, n, k), device=dev, generator=g) * 2 - 1
    obs, obs_h = torch.zeros((n, env.obs_robot_len), device=dev), torch.zeros((n, max(env.obs_human_len, 1)), device=dev)
    rew, done, info = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros((n, 4), device=dev)

    def step_dev(a):
        if coop:
            sim.coop_step_dev(a.data_ptr(), obs.data_ptr(), obs_h.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
        else:
            sim.bathing_step_dev(a.data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    cnt_mean, cnt_max = [], 0
    torch.cuda.synchronize()
    for i in range(W):
        step_dev(act[i])
    torch.cuda.synchronize()
    sm_mhz = gpu_info()['sm_mhz']
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for i in range(K):
        step_dev(act[W + i])
    b.record(stream)
    torch.cuda.synchronize()
    dev_ms = a.elapsed_time(b) / K
    for i in range(W + K, episode):             # the rest of the episode, with the contact count read after every step
        step_dev(act[i])
        cnt, _ = sim.solver_stats()
        cnt_mean.append(float(cnt.mean())); cnt_max = max(cnt_max, int(cnt.max()))
    finite = bool(torch.isfinite(obs).all()) and bool(torch.isfinite(rew).all())
    out = {'sm_mhz_before_timing': sm_mhz, 'reset_s': reset_s, 'device_step_ms': dev_ms, 'device_env_steps_per_s': n / dev_ms * 1e3, 'episode_steps': episode,
           'contacts_per_env_mean': float(np.mean(cnt_mean)), 'contacts_per_env_max': cnt_max, 'max_contacts': int(sim.cfg.max_contacts),
           'overflow_envs_reset': int(overflow_reset), 'overflow_envs_episode': int(sim.overflow_count()),
           'sim_device_bytes': int(sim_bytes), 'finite': finite}
    bb = env._bb
    if getattr(bb, 'goals_reached', None) is not None:
        out['toc_start_goal_reached'] = float((np.asarray(bb.goals_reached) >= 1).mean())
    out['reset_unresolved_envs'] = int(bb.unresolved)
    env.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=4096)
    ap.add_argument('--steps', type=int, default=150)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--episode', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=2)
    ap.add_argument('--gpu-warmup', type=float, default=10.0)
    ap.add_argument('--ids', default=','.join(IDS))
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: this measurement needs the GPU')
    if args.warmup + args.steps >= args.episode:
        raise SystemExit('--warmup + --steps must leave steps of the episode for the contact count')
    ids = args.ids.split(',')
    res = {'workload': 'BedBathing on each robot, fused step', 'gpu': gpu_info(), 'n_envs': args.n, 'steps': args.steps, 'warmup': args.warmup,
           'rounds': args.rounds, 'ids': {i: {'rounds': []} for i in ids}}
    warm_gpu(args.gpu_warmup)
    res['gpu_after_warmup'] = gpu_info()
    for r in range(args.rounds):
        for env_id in (ids if r % 2 == 0 else ids[::-1]):
            m = measure(env_id, args.n, args.steps, args.warmup, args.episode)
            res['ids'][env_id]['rounds'].append(m)
            print(r, env_id, json.dumps(m), file=sys.stderr, flush=True)
    for env_id in ids:
        rates = [m['device_env_steps_per_s'] for m in res['ids'][env_id]['rounds']]
        res['ids'][env_id]['device_env_steps_per_s_median'] = float(np.median(rates))
    res['gpu_after'] = gpu_info()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
