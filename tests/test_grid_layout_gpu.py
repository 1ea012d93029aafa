"""Pins the bytes of the grid and delta-field that s4g_set_cloud_p builds and k_verify reads (the layout helpers of
s4g_internal.cuh, DESIGN.md sections 2 and 3.1).

A writer and a reader that disagree about a layout -- a boundary slot off by one, a shift that reads MAYBE where CERTAIN
was written -- do not change any count: the pair only goes on to the exact test.  What they change is the work Verify
does, so every workload here pins the six grid statistics and the five probe statistics of a fixed candidate set to the
values measured on an H100, exactly, besides comparing the counts with the port.  The statistics do not depend on the
query-patch schedule (test_verify_patches_gpu.py); they change when a table or the probe changes.  If a change to a
layout is intended, the constants below change with it.
"""
import numpy as np
import pytest

from oracle import port as oport
from tests import common
from tests.test_verify_patches_gpu import mixed_candidates

pytestmark = pytest.mark.gpu

# workload -> (grid_stats(), verify_probe_stats()), measured on an H100 80GB HBM3 at commit 35a764f, before the layout
# helpers of s4g_internal.cuh existed; the helpers change none of them
PINNED = {
    "mixed": (
        dict(cell_edge=0.02019999921321869, bricks=1906, brick_edge=4, cells=121984,
             points_per_occupied_cell=1.4659532360917686, resident_bytes=6290122.0),
        dict(points_tested=161913, ranges_read=109314, brick_entries_read=112099, bitmap_words_read=646639,
             tile_pairs_culled=13937)),
    "brick8": (
        dict(cell_edge=0.0016159999649971724, bricks=16966, brick_edge=8, cells=8686592,
             points_per_occupied_cell=1.0027575833542242, resident_bytes=343787998.0),
        dict(points_tested=221, ranges_read=225, brick_entries_read=241, bitmap_words_read=357945,
             tile_pairs_culled=14451)),
    "maybe": (
        dict(cell_edge=0.02019999921321869, bricks=1906, brick_edge=4, cells=121984,
             points_per_occupied_cell=1.4659532360917686, resident_bytes=6290122.0),
        dict(points_tested=1345848, ranges_read=875608, brick_entries_read=892809, bitmap_words_read=2228076,
             tile_pairs_culled=0)),
    "mixed_cshift3": (
        dict(cell_edge=0.02019999921321869, bricks=1906, brick_edge=4, cells=121984,
             points_per_occupied_cell=1.4659532360917686, resident_bytes=6290122.0),
        dict(points_tested=161913, ranges_read=109314, brick_entries_read=112099, bitmap_words_read=675638,
             tile_pairs_culled=11900)),
}


def _eye_shifts(K, length, seed):
    """K column-major translations of `length` in random directions"""
    rng = np.random.RandomState(seed)
    T = np.tile(np.eye(4, dtype=np.float32), (K, 1, 1))
    for k in range(K):
        v = rng.standard_normal(3)
        T[k, :3, 3] = (v / np.linalg.norm(v) * length).astype(np.float32)
    return np.ascontiguousarray(T.transpose(0, 2, 1)).reshape(K, 16)


def workload(name):
    """(P, Q, delta, column-major candidates)"""
    if name in ("mixed", "mixed_cshift3"):
        sc = common.scenario(20000, 0.4, 0.01, seed=5)
        return sc["P"], sc["Q"], 0.01, mixed_candidates(sc, 48)
    if name == "brick8":
        # 1372 x 1426 x 853 cells: 4-cell bricks would need more than 2^24 brick-table entries
        sc = common.scenario(20000, 0.4, 0.0008, seed=5)
        return sc["P"], sc["Q"], 0.0008, mixed_candidates(sc, 48)
    if name == "maybe":
        # every query lies 0.9 delta from its own source point: mostly boundary voxels, decided below the first level
        sc = common.scenario(20000, 0.4, 0.01, seed=5)
        return sc["P"], sc["P"], 0.01, _eye_shifts(32, 0.009, seed=1)
    raise KeyError(name)


def measure(ctx, name):
    P, Q, delta, T = workload(name)
    ctx.set_cloud_p(P, delta)
    ctx.set_cloud_q(Q)
    return ctx.grid_stats(), ctx.verify_probe_stats(T), ctx.verify(T)


@pytest.fixture
def context(s4g_lib, monkeypatch):
    from super4pcs_b200 import Context

    def make(cshift_min=None):
        if cshift_min is None:
            monkeypatch.delenv("S4G_CSHIFT_MIN", raising=False)
        else:
            monkeypatch.setenv("S4G_CSHIFT_MIN", str(cshift_min))
        return Context(0)
    return make


@pytest.mark.parametrize("name", ["mixed", "brick8", "maybe", "mixed_cshift3"])
def test_grid_and_probe_statistics_are_pinned(context, name):
    with context(3 if name == "mixed_cshift3" else None) as ctx:
        gs, st, counts = measure(ctx, name)
    P, Q, delta, T = workload(name)
    pt = oport.Port(P, Q, delta)
    _, good, _ = pt.verify_batch(T, 0.0, nthreads=oport.num_threads())
    assert np.array_equal(counts, good)
    # the layout each workload is meant to reach
    if name == "brick8":
        assert gs["brick_edge"] == 8                      # k_verify<false, 0>
    else:
        assert gs["brick_edge"] == 4                      # k_verify<false, 2>
    if name == "maybe":
        assert (counts == len(Q)).all()
        assert st["ranges_read"] > len(Q) * len(T) // 2   # most pairs are MAYBE at the first level
    if name == "mixed_cshift3":
        with context(None) as ref:
            assert st["tile_pairs_culled"] < measure(ref, "mixed")[1]["tile_pairs_culled"]   # coarser cull blocks
    assert (gs, st) == PINNED[name]
