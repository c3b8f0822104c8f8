"""Batched reset (SURVEY.md §8(f)1 / reference env.py:276-310): every env starts from a pose the reference would accept --
IK converged and neither the arm nor the tool it holds intersects the person, the table or the wheelchair.  An env that
starts in collision keeps 60-128 contacts for its whole episode and single-handedly sets the duration of the
narrowphase and PGS kernels of the whole batch."""
import numpy as np

from assistive_gym_b200 import capi
from assistive_gym_b200.sim import BatchSim


def test_feeding_reset_is_collision_free(feeding, emu_lib):
    fb = feeding
    n = 48
    sim = BatchSim(fb.scene, capi.default_config(), n, _lib=emu_lib)
    fb.reset(sim, np.random.default_rng(123), settle_steps=0)
    assert fb.ik_colliding == 0 and float(fb.ik_err.max()) < 0.01
    for ob in (fb.humans['male'], fb.humans['female'], fb.table, fb.wheelchair):
        assert int((sim.closest_points(fb.robot, ob, 0.0, max_pts=1)[1] > 0).sum()) == 0
        assert int((sim.closest_points(fb.tool, ob, 0.0, max_pts=1)[1] > 0).sum()) == 0
    # the food starts inside the spoon: 8 spheres within 3 cm of the tool, none touching anything else yet
    for f in fb.foods:
        assert np.all(sim.closest_points(f, fb.tool, 0.03, max_pts=1)[1] > 0)
    sim.step(25)
    cnt, it = sim.solver_stats()
    assert cnt.max() <= 100, cnt         # ~70 while the food settles into the spoon; nowhere near the 128-contact budget
    assert sim.overflow_count() == 0


def test_bed_bathing_reset_is_collision_free(emu_lib):
    from assistive_gym_b200.bed_bathing_batch import BedBathingBatch
    bb = BedBathingBatch()
    n = 16
    sim = BatchSim(bb.scene, capi.default_config(), n, _lib=emu_lib)
    bb.reset(sim, np.random.default_rng(5))
    assert bb.unresolved == 0 and float(bb.ik_err.max()) < 0.03
    for ob in (bb.humans['male'], bb.humans['female'], bb.bed):
        assert int((sim.closest_points(bb.robot, ob, 0.0, max_pts=1)[1] > 0).sum()) == 0
        assert int((sim.closest_points(bb.tool, ob, 0.0, max_pts=1)[1] > 0).sum()) == 0
