#!/usr/bin/env python3
"""Where k_narrow's work goes, from the host-compiled kernel bodies (a CPU run; no GPU needed).

Builds the kernel bodies for the host with AG_NARROW_STAT defined to record one entry per candidate pair (ag_device.cuh: GJK
iterations, face-axis fallback, manifold pool fill, contacts), starts FeedingJaco-v1 from bench.py's seeded start state (the same
per-env samples as the bench's first `--n` envs), takes one fused env step and prints one JSON line per k_narrow launch (substep):

  candidates per env; pairs within max_dist; pairs that take the pen_faces fallback; GJK iterations per pair; pool fill per
  surviving pair; and `gjk_lane_use`, the share of lane-iterations that do work when each warp of the kernel's (slot, env) mapping
  runs as long as its longest lane (1.0: no divergence in the GJK loop).

usage: python tools/narrow_work.py [--n 256]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PRELUDE = r'''
#include <vector>
struct NarrowRec { int tid, gjk_iters, pen_faces, pool, contacts; };
static std::vector<NarrowRec> g_rec;
static bool g_in = false;        // between a candidate's `cand` and `done`: other callers of narrow_pair are not counted
static void ns_cand(int tid) { g_rec.push_back(NarrowRec{tid, 0, 0, -1, 0}); g_in = true; }
static void ns_gjk_iter(int) { if (g_in) g_rec.back().gjk_iters++; }
static void ns_pen_faces(int) { if (g_in) g_rec.back().pen_faces++; }
static void ns_pool(int n) { if (g_in) g_rec.back().pool = n; }
static void ns_done(int n) { if (g_in) { g_rec.back().contacts = n; g_in = false; } }
#define AG_NARROW_STAT(event, value) ns_##event(value)
#include "agphys.cu"
extern "C" int narrow_work_count() { return (int)g_rec.size(); }
extern "C" void narrow_work_take(int* out) {
  for (size_t i = 0; i < g_rec.size(); i++) {
    const NarrowRec& r = g_rec[i];
    int* o = out + 5 * i; o[0] = r.tid; o[1] = r.gjk_iters; o[2] = r.pen_faces; o[3] = r.pool; o[4] = r.contacts;
  }
  g_rec.clear();
}
'''


def build(tmp):
    src, so = os.path.join(tmp, 'narrow_work.cpp'), os.path.join(tmp, 'libnarrow_work.so')
    with open(src, 'w') as f:
        f.write(PRELUDE)
    subprocess.check_call(['g++', '-x', 'c++', '-std=c++17', '-O2', '-fPIC', '-shared', '-DAG_CPU_EMU', '-w',
                           '-I', os.path.join(ROOT, 'assistive_gym_b200', 'csrc'), '-o', so, src])
    return so


def take(lib):
    import ctypes as C
    n = lib.narrow_work_count()
    buf = np.zeros((n, 5), dtype=np.int32)
    lib.narrow_work_take(buf.ctypes.data_as(C.POINTER(C.c_int)))
    return buf


def summary(rec, n_envs):
    tid, iters, pen, pool, ncon = rec.T
    env = tid % n_envs
    cands = np.bincount(env, minlength=n_envs)
    gjk = iters > 0
    surv = pool >= 0
    # the kernel's warps: 32 consecutive tids, i.e. 32 envs at one candidate slot
    warp = tid // 32
    wmax = np.zeros(warp.max() + 1, dtype=np.int64)
    np.maximum.at(wmax, warp, iters)
    lanes_busy = iters.sum()
    lanes_held = 32 * wmax.sum()
    return {
        'envs': n_envs,
        'candidates_per_env': {'mean': float(cands.mean()), 'p50': float(np.median(cands)), 'max': int(cands.max())},
        'pairs': int(len(rec)),
        'within_max_dist': int(surv.sum()),
        'gjk_pairs': int(gjk.sum()),
        'pen_faces_fallback': int(pen.sum()),
        'gjk_iters_per_pair': {'mean': float(iters[gjk].mean()) if gjk.any() else 0.0,
                               'p50': float(np.median(iters[gjk])) if gjk.any() else 0.0,
                               'p99': float(np.percentile(iters[gjk], 99)) if gjk.any() else 0.0,
                               'max': int(iters.max())},
        'gjk_lane_use': float(lanes_busy / lanes_held) if lanes_held else None,
        'pool_fill_per_surviving_pair': {'mean': float(pool[surv].mean()) if surv.any() else 0.0,
                                         'hist': np.bincount(pool[surv], minlength=13).tolist()},
        'contacts_per_surviving_pair': float(ncon[surv].mean()) if surv.any() else 0.0,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--n', type=int, default=256, help="envs: bench.py's first N envs")
    args = ap.parse_args()
    from assistive_gym_b200 import capi
    from assistive_gym_b200.feeding_batch import FeedingBatch
    from assistive_gym_b200.sharding import sample_block
    from assistive_gym_b200.sim import BatchSim
    with tempfile.TemporaryDirectory() as tmp:
        lib = capi.load_library(build(tmp))
        fb = FeedingBatch()
        sim = BatchSim(fb.scene, capi.default_config(), args.n, _lib=lib)
        sg = fb.reset(sim, np.random.default_rng(1001), settle_steps=25, sample=sample_block(fb, 0, args.n))     # as bench.py
        fb.start_fused(sim, sg, seed=1001)
        take(lib)                                                                     # drop the reset's substeps
        sim.feeding_step_host(np.random.default_rng(0).uniform(-1, 1, size=(args.n, 7)).astype(np.float32))
        rec = take(lib)
        sim.close()
    # one launch per substep; within a launch the host build visits the tids in ascending order
    starts = [0] + [i for i in range(1, len(rec)) if rec[i, 0] <= rec[i - 1, 0]] + [len(rec)]
    for k in range(len(starts) - 1):
        print(json.dumps(dict(substep=k, **summary(rec[starts[k]:starts[k + 1]], args.n))), flush=True)


if __name__ == '__main__':
    main()
