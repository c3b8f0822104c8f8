#!/usr/bin/env python3
"""GPU box: fused Dressing step throughput (ag_dressing_step_*) per robot, device-timed; not the headline metric.

One JSON line per id: the card and its power limit (read in the same run), reset time and the envs the placement left colliding
with the person or the wheelchair, the graph-replayed device step (`dressing_step_dev`, CUDA events) and the host-buffer step
(`dressing_step_host`, host clock; the call ends in a stream synchronise) over the same number of steps after a warm-up, a
per-kernel split from a separate profiled pass (with `k_cloth` ms per launch), rigid and cloth contacts per env against their
budgets, overflowed envs (one sticky flag per env for both budgets, read after the settle and again after all the steps that
follow: warm-up, timed device steps, host steps and profiled steps, `overflow_steps` in all) and the sim's device memory.  The
co-optimisation ids are measured by tools/gpu_coop_bench.py.

usage: python tools/gpu_dressing_robots_bench.py [--ids DressingPR2-v1,DressingSawyer-v1,DressingJaco-v1] [--n 2048] [--steps 50]
                                                 [--warmup 5] [--profile-steps 3] [--out profiles/h100_dressing_robots_bench.jsonl]"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from assistive_gym_b200.envs.agents.robot import PR2, Jaco, Sawyer  # noqa: E402
from assistive_gym_b200.envs.dressing import dressing_batch_for  # noqa: E402
from assistive_gym_b200.sim import BatchSim  # noqa: E402
from tools.gpu_drinking_bench import gpu_info  # noqa: E402

ROBOTS = {'DressingPR2-v1': PR2, 'DressingSawyer-v1': Sawyer, 'DressingJaco-v1': Jaco}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--ids', default='DressingPR2-v1,DressingSawyer-v1,DressingJaco-v1', help='comma-separated Dressing ids, one JSON line each')
    ap.add_argument('--n', type=int, default=2048)
    ap.add_argument('--steps', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--profile-steps', type=int, default=3)
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
    db = dressing_batch_for(ROBOTS[env_id]('left'))
    cfg = db.config()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    sim = BatchSim(db.scene, cfg, n)
    t0 = time.time()
    s = db.reset(sim, np.random.default_rng(0))
    db.start_fused(sim, s)
    torch.cuda.synchronize()
    reset_s = time.time() - t0
    sim_bytes = free0 - torch.cuda.mem_get_info()[0]
    overflow_reset = sim.overflow_count()
    colliding = int(db.colliding(sim).sum())

    dev = torch.device('cuda')
    stream = torch.cuda.ExternalStream(sim.stream_ptr())
    g = torch.Generator(device=dev).manual_seed(0)
    act = torch.rand((W + K, n, 7), device=dev, generator=g) * 2 - 1
    obs, rew, done, info = torch.zeros((n, 24), device=dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros((n, 4), device=dev)
    torch.cuda.synchronize()
    for i in range(W):
        sim.dressing_step_dev(act[i].data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(stream)
    for i in range(K):
        sim.dressing_step_dev(act[W + i].data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    b.record(stream)
    torch.cuda.synchronize()
    dev_ms = a.elapsed_time(b) / K
    finite = bool(torch.isfinite(obs).all()) and bool(torch.isfinite(rew).all())
    cnt, it = sim.solver_stats()
    ccnt = sim.cloth_get_contacts(1)[0]

    act_h = np.random.default_rng(1).uniform(-1, 1, size=(K, n, 7)).astype(np.float32)
    sim.dressing_step_host(act_h[0])
    t0 = time.perf_counter()
    for i in range(K):
        sim.dressing_step_host(act_h[i])
    host_ms = (time.perf_counter() - t0) * 1e3 / K

    sim.profile_get()
    sim.profile_enable(True)
    for i in range(args.profile_steps):
        sim.dressing_step_dev(act[i].data_ptr(), obs.data_ptr(), rew.data_ptr(), done.data_ptr(), info.data_ptr())
    prof = sim.profile_get()
    sim.profile_enable(False)
    total = sum(ms for ms, _ in prof.values())
    kernels = {k: {'ms_per_step': ms / args.profile_steps, 'launches_per_step': c / args.profile_steps, 'share': ms / total}
               for k, (ms, c) in sorted(prof.items(), key=lambda kv: -kv[1][0])}
    overflow = sim.overflow_count()
    out = {'workload': '%s fused step' % env_id, 'gpu': gpu, 'n_envs': n, 'steps': K, 'warmup': W,
           'num_substeps': cfg.num_substeps, 'frame_skip': 5, 'max_contacts': cfg.max_contacts, 'max_cloth_contacts': 1024,
           'cloth_links': len(db.cloth_links), 'reset_s': reset_s, 'envs_left_colliding': colliding,
           'device_step_ms': dev_ms, 'device_env_steps_per_s': n / dev_ms * 1e3,
           'host_step_ms': host_ms, 'host_env_steps_per_s': n / host_ms * 1e3,
           'k_cloth_ms_per_launch': prof['k_cloth'][0] / prof['k_cloth'][1] if 'k_cloth' in prof else None,
           'contacts_per_env_mean': float(cnt.mean()), 'contacts_per_env_max': int(cnt.max()), 'pgs_iters_mean': float(it.mean()),
           'cloth_contacts_per_env_mean': float(ccnt.mean()), 'cloth_contacts_per_env_max': int(ccnt.max()),
           'overflow_envs_after_settle': overflow_reset, 'overflow_envs_after_steps': overflow, 'overflow_steps': W + K + 1 + K + args.profile_steps, 'sim_device_bytes': int(sim_bytes),
           'finite': finite, 'profiled_steps': args.profile_steps, 'profiled_ms_per_step': total / args.profile_steps, 'kernels': kernels}
    line = json.dumps(out)
    print(line, flush=True)
    sim.close()
    return line


if __name__ == '__main__':
    main()
