#!/usr/bin/env python3
"""Diagnostic (GPU box): per-env PGS cycles, warp trip counts and row-stream sizes after a few bench-like steps."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
import numpy as np
from assistive_gym_b200 import capi
from assistive_gym_b200.feeding_batch import FeedingBatch
from assistive_gym_b200.sim import BatchSim
n = int(os.environ.get("AG_N", "4096")); steps = int(os.environ.get("AG_STEPS", "8"))
fb = FeedingBatch(); sim = BatchSim(fb.scene, capi.default_config(), n)
rng = np.random.default_rng(0)
s = fb.reset(sim, rng, settle_steps=25)
fb.start_fused(sim, s)
acts = np.random.default_rng(1).uniform(-1, 1, size=(steps, n, 7)).astype(np.float32)
for i in range(steps):
    sim.feeding_step_host(acts[i])
cyc = sim.pgs_cycles().astype(np.float64); cnt, it = sim.solver_stats(); trips, fl = sim.pgs_trips()
q = [50, 90, 99, 99.9]
print('k_pgs: %d CTAs per SM, %d B of shared memory per CTA' % sim.pgs_occupancy())
print('cycles: mean %.0f p50 %.0f p90 %.0f p99 %.0f p99.9 %.0f max %.0f' % (cyc.mean(), *np.percentile(cyc, q), cyc.max()))
print('trips : mean %.0f p50 %.0f p90 %.0f p99 %.0f p99.9 %.0f max %d' % (trips.mean(), *np.percentile(trips, q), trips.max()))
print('stream bytes: mean %.0f p50 %.0f p99 %.0f max %d' % (4 * fl.mean(), *np.percentile(4 * fl, [50, 99]), 4 * fl.max()))
print('iters : mean %.1f p50 %.0f p99 %.0f max %d; contacts mean %.1f max %d' % (it.mean(), *np.percentile(it, [50, 99]), it.max(), cnt.mean(), cnt.max()))
print('cycles per trip: mean %.0f p50 %.0f p99 %.0f' % ((cyc / np.maximum(trips, 1)).mean(), *np.percentile(cyc / np.maximum(trips, 1), [50, 99])))
w = np.argsort(-cyc)[:5]
for e in w:
    print('env %d cycles %.2fM trips %d iters %d contacts %d stream %d B' % (e, cyc[e] / 1e6, trips[e], it[e], cnt[e], 4 * fl[e]))
