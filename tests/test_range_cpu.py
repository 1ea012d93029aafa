"""The range query (s4g_range) without a GPU: the port's brute force against the compiled reference's own kd-tree
(KdTree::doQueryDistIndices, every list sorted by index), and the C++ layer's getNeighbors on the oracle stand-in of
libs4g.

Contract (include/s4g.h): the list of query i is every P index j with d^2 < sq_radius (strict, as the kd-tree's point
test), in ascending j, with d^2 bit for bit.  The kd-tree prunes with strict tests too, so the two sides agree exactly,
list for list, at every radius."""
import os

import numpy as np
import pytest

from oracle import range as orange
from tests import common, range as trange

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not orange.ref_available(), reason="oracle/_ref (compiled reference) not present")


def same(a, b):
    """two CSR results are equal: offsets, indices, and d^2 bit for bit"""
    assert np.array_equal(a[0], b[0])
    assert np.array_equal(a[1], b[1])
    assert np.array_equal(common.bits(a[2]), common.bits(b[2]))


def queries(P, delta, rng, n_in=300, n_edge=60, n_far=60):
    """inside the cloud (P points jittered), on the edge of its box, far outside (up to 1e3 cell widths), and NaN rows"""
    lo, hi = P.min(0), P.max(0)
    pick = P[rng.randint(0, len(P), n_in)] + rng.normal(0, delta, (n_in, 3))
    edge = rng.uniform(lo, hi, (n_edge, 3))
    ax = rng.randint(0, 3, n_edge)
    edge[np.arange(n_edge), ax] = np.where(rng.rand(n_edge) < 0.5, lo[ax], hi[ax])
    far = rng.normal(0, 1, (n_far, 3))
    far = far / np.linalg.norm(far, axis=1, keepdims=True) * (np.abs(hi - lo).max() + rng.uniform(1, 1000, (n_far, 1))
                                                              * 2.02 * delta)
    nan = np.array([[np.nan, 0, 0], [0, np.nan, 0], [np.nan] * 3], np.float32)
    return np.concatenate([pick, edge, far, nan]).astype(np.float32)


def radii(delta, extent):
    """0, delta^2, MeanDistance's squared radius (0.2 x the extent, a length passed as a squared radius, as the reference
    does), a large radius, +inf"""
    return [0.0, delta * delta, float(np.float32(extent) * np.float32(0.2)), float(np.float32(0.5 * extent) ** 2), np.inf]


def compare_all(m, P, X, delta, T16s):
    extent = float(np.abs(P.max(0) - P.min(0)).max())
    total = 0
    for T16 in T16s:
        for r in radii(delta, extent):
            got = orange.bruteforce(P, X, r, T16)
            same(got, m.query(X, r, T16))
            off = got[0]
            assert (np.diff(off)[-3:] == 0).all()                              # NaN queries: empty lists
            for i in range(len(X)):                                            # ascending, no repeats
                assert (np.diff(got[1][off[i]:off[i + 1]]) > 0).all()
            assert (got[2] < np.float32(r)).all()
            if r == 0.0:
                assert off[-1] == 0
            total += int(off[-1])
    return total


@needs_ref
@pytest.mark.parametrize("n,delta,seed", [(2000, 0.02, 1), (3000, 0.01, 4)])
def test_bruteforce_matches_reference_kdtree_on_seeded_clouds(n, delta, seed):
    sc = common.scenario(n, 0.4, delta, seed=seed)
    m = orange.RefRange(sc["raw"]["P"], sc["raw"]["Q"], delta)
    P, _ = m.sampled()
    rng = np.random.RandomState(seed)
    X = queries(P, delta, rng)
    T16s = [None, common.candidates_colmajor(sc, 2, seed=seed, n_near=1)[0], common.candidates_colmajor(sc, 2, seed=seed)[1]]
    assert compare_all(m, P, X, delta, T16s) > 10000


@needs_ref
def test_bruteforce_matches_reference_kdtree_on_hippo_samples():
    g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
    m = orange.RefRange(g["stage_P"], g["stage_Q"], 0.01)
    P, Q = m.sampled()
    rng = np.random.RandomState(3)
    X = np.concatenate([queries(P, 0.01, rng, 200, 40, 40)[:-3], Q[:200], queries(P, 0.01, rng, 0, 0, 0)])
    assert compare_all(m, P, X, 0.01, [None, g["stage_b0_tcs_T"]]) > 10000


@needs_ref
def test_boundary_excluded_and_one_ulp_below_included():
    """a radius equal to a computed d^2 excludes that point on both sides; the next float above it includes it"""
    sc = common.scenario(1500, 0.4, 0.02, seed=9)
    m = orange.RefRange(sc["raw"]["P"], sc["raw"]["Q"], 0.02)
    P, _ = m.sampled()
    rng = np.random.RandomState(2)
    X = queries(P, 0.02, rng, 60, 0, 0)[:60]
    T16 = common.candidates_colmajor(sc, 1, seed=3, n_near=1)[0]
    for T in (None, T16):
        for i in range(0, 60, 6):
            # the d^2 of query i to its 5th nearest point, as both sides compute it
            off, idx, sq = orange.bruteforce(P, X[i:i + 1], np.inf, T)
            k = np.argsort(sq, kind="stable")[4]
            r, j = sq[k], idx[k]
            below = orange.bruteforce(P, X, r, T)
            same(below, m.query(X, r, T))
            assert j not in below[1][below[0][i]:below[0][i + 1]]
            above = orange.bruteforce(P, X, np.nextafter(r, np.float32(np.inf)), T)
            same(above, m.query(X, np.nextafter(r, np.float32(np.inf)), T))
            assert j in above[1][above[0][i]:above[0][i + 1]]


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    from tests import build_shim
    d = tmp_path_factory.mktemp("range")
    exe = trange.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


def check_program(r):
    """getNeighbors of the C++ layer against the brute force under the transform that was found"""
    sP, sQ = r["sP"], r["sQ"]
    for dist, got in zip(r["max_distance"], r["lists"]):
        same(got, orange.bruteforce(sP, sQ, np.float32(dist) * np.float32(dist), r["C"]))
    assert r["lists"][0][0][-1] > 0 and r["lists"][1][0][-1] > r["lists"][0][0][-1]


def test_get_neighbors_on_oracle_shim_hippo(program, tmp_path):
    """the run-example options (-o 0.7 -d 0.01 -n 200) on the hippo golden: the registration is the golden one, and
    getNeighbors equals the brute force; it throws before a registration"""
    exe, shim = program
    h = np.load(os.path.join(ROOT, "tests", "golden", "hippo.npz"))
    g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
    r = trange.run(exe, tmp_path, h["P"], h["Q"], 0.01, 0.7, 200, preload=shim)
    assert r["threw_before"] == 1
    assert r["score"] == g["score"]
    check_program(r)


def test_get_neighbors_on_oracle_shim_synthetic(program, tmp_path):
    d = common.scenario(6000, 0.5, 0.01, seed=12)["raw"]
    exe, shim = program
    r = trange.run(exe, tmp_path, d["P"], d["Q"], 0.01, 0.5, 1000, preload=shim)
    assert r["threw_before"] == 1
    check_program(r)
