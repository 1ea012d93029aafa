"""The k-nearest query (s4g_knn) without a GPU: the port's brute force against the compiled reference's own kd-tree, and
the C++ layer's getKNearest on the oracle stand-in of libs4g.

Contract (include/s4g.h): row i is the k smallest (d^2, j) with d^2 <= sq_radius and j != exclude[i], ascending, padded
with -1 / +inf.  The reference's kd-tree has no k-nearest query; its range query (doQueryDistIndices, strict d^2 < r) at
r = nextafterf(sq_radius, +inf) holds exactly the points with d^2 <= sq_radius, so every row must be the first k of that
list with exclude[i] removed, ordered by (d^2, j).  At k = 1 the row is the reference's restricted closest-point answer
wherever the kd-tree finds one (up to the index of a tie)."""
import os

import numpy as np
import pytest

from oracle import knn as oknn
from oracle import nearest_any as ona
from oracle import range as orange
from tests import common, knn as tknn
from tests.test_nearest_any_cpu import check_against_reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not orange.ref_available(), reason="oracle/_ref (compiled reference) not present")
KS = [1, 2, 5, 16, 33, 64]


def same(a, b):
    """two (index, sq_dist) results are equal: indices, and d^2 bit for bit"""
    assert np.array_equal(a[0], b[0]), np.argwhere(a[0] != b[0])[:5]
    assert np.array_equal(common.bits(a[1]), common.bits(b[1]))


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
    """0, (0.1 delta)^2, delta^2, 9 delta^2, MeanDistance's squared radius (0.2 x the extent), +inf"""
    return [0.0, (0.1 * delta) ** 2, delta * delta, 9 * delta * delta, float(np.float32(extent) * np.float32(0.2)), np.inf]


def compare_all(m, P, X, delta, T16s, excl, ks=KS):
    """every radius x T x exclusion x k: the brute force equals the reference tree's range-list prefix; returns the
    number of non-padding entries seen"""
    extent = float(np.abs(P.max(0) - P.min(0)).max())
    held = 0
    for T16 in T16s:
        for r in radii(delta, extent):
            lists = m.query(X, oknn.range_radius(r), T16)
            for ex in (None, excl):
                for k in ks:
                    got = oknn.bruteforce(P, X, k, r, T16, ex)
                    same(got, oknn.from_range(lists, k, ex))
                    assert (got[0][-3:] == -1).all() and np.isinf(got[1][-3:]).all()     # NaN queries: padding
                    if ex is not None:
                        assert not ((got[0] >= 0) & (got[0] == ex[:, None])).any()
                    if r == 0.0:
                        assert (got[1][got[0] >= 0] == 0).all()
                    held += int((got[0] >= 0).sum())
    return held


@needs_ref
@pytest.mark.parametrize("n,delta,seed", [(2000, 0.02, 1), (3000, 0.01, 4)])
def test_bruteforce_equals_reference_range_prefix_on_seeded_clouds(n, delta, seed):
    sc = common.scenario(n, 0.4, delta, seed=seed)
    m = orange.RefRange(sc["raw"]["P"], sc["raw"]["Q"], delta)
    P, _ = m.sampled()
    rng = np.random.RandomState(seed)
    X = queries(P, delta, rng)
    excl = rng.randint(-1, len(P), len(X)).astype(np.int32)
    T16s = [None, common.candidates_colmajor(sc, 2, seed=seed, n_near=1)[0], common.candidates_colmajor(sc, 2, seed=seed)[1]]
    assert compare_all(m, P, X, delta, T16s, excl) > 100000
    # the sampled P points themselves, each excluding itself: the normal-estimation query
    self_ = np.arange(len(P), dtype=np.int32)
    lists = m.query(P, np.inf)
    for k in (8, 16):
        same(oknn.bruteforce(P, P, k, np.inf, None, self_), oknn.from_range(lists, k, self_))


@needs_ref
def test_bruteforce_equals_reference_range_prefix_on_hippo_samples():
    g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
    m = orange.RefRange(g["stage_P"], g["stage_Q"], 0.01)
    P, Q = m.sampled()
    rng = np.random.RandomState(3)
    X = np.concatenate([queries(P, 0.01, rng, 200, 40, 40)[:-3], Q[:200], queries(P, 0.01, rng, 0, 0, 0)])
    excl = rng.randint(-1, len(P), len(X)).astype(np.int32)
    assert compare_all(m, P, X, 0.01, [None, g["stage_b0_tcs_T"]], excl, ks=[1, 5, 16, 64]) > 10000


@needs_ref
def test_boundary_kept_and_one_ulp_above_dropped():
    """a point whose d^2 equals sq_radius is in the row; at the float below sq_radius (the point one ulp above it) it is
    not -- on both sides"""
    sc = common.scenario(1500, 0.4, 0.02, seed=9)
    m = orange.RefRange(sc["raw"]["P"], sc["raw"]["Q"], 0.02)
    P, _ = m.sampled()
    rng = np.random.RandomState(2)
    X = queries(P, 0.02, rng, 60, 0, 0)[:60]
    T16 = common.candidates_colmajor(sc, 1, seed=3, n_near=1)[0]
    for T in (None, T16):
        for i in range(0, 60, 6):
            idx, sq = oknn.bruteforce(P, X[i:i + 1], 64, np.inf, T)
            r, j = sq[0, 4], idx[0, 4]                           # the 5th nearest point's d^2, as both sides compute it
            below = np.nextafter(r, np.float32(-np.inf))
            for rad, kept in ((r, True), (below, False)):
                got = oknn.bruteforce(P, X, 64, rad, T)
                same(got, oknn.from_range(m.query(X, oknn.range_radius(rad), T), 64))
                assert (j in got[0][i]) == kept
                assert (got[1][i][got[0][i] >= 0] <= np.float32(rad)).all()


@needs_ref
@pytest.mark.parametrize("n,delta,seed", [(2000, 0.02, 1), (3000, 0.01, 4)])
def test_k1_equals_reference_closest_point(n, delta, seed):
    """k = 1: sq_dist equals the reference's closest-point query wherever the kd-tree finds a point, and index equals it
    wherever that minimum is unique (check_against_reference of the s4g_nearest tests)"""
    sc = common.scenario(n, 0.4, delta, seed=seed)
    m = ona.RefNearestAny(sc["raw"]["P"], sc["raw"]["Q"], delta)
    P, _ = m.sampled()
    rng = np.random.RandomState(seed)
    X = queries(P, delta, rng)
    excl = rng.randint(-1, len(P), len(X)).astype(np.int32)
    extent = float(np.abs(P.max(0) - P.min(0)).max())
    hits = 0
    for T16 in (None, common.candidates_colmajor(sc, 1, seed=seed, n_near=1)[0]):
        for r in radii(delta, extent):
            for ex in (None, excl):
                ri, rs = m.query(X, r, T16, ex)
                pi, ps = oknn.bruteforce(P, X, 1, r, T16, ex)
                check_against_reference(P, X, r, T16, pi[:, 0], ps[:, 0], ri, rs)
                same((pi[:, 0], ps[:, 0]), ona.bruteforce(P, X, r, T16, ex))
                hits += int((ri >= 0).sum())
    assert hits > 1000


def test_bruteforce_pads_and_orders_ties():
    """all P points identical: every d^2 ties and the row is the k smallest indices; fewer points than k pad"""
    P = np.tile(np.float32([[0.25, -0.5, 1.0]]), (40, 1))
    X = np.float32([[0.25, -0.5, 1.0], [1, 2, 3]])
    idx, sq = oknn.bruteforce(P, X, 64, np.inf, None, np.int32([3, -1]))
    assert list(idx[0, :39]) == [j for j in range(40) if j != 3] and (idx[:, 40:] == -1).all()
    assert (idx[1, :40] == np.arange(40)).all() and idx[0, 39] == -1
    assert (sq[0, :39] == 0).all() and np.isinf(sq[:, 40:]).all()


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    from tests import build_shim
    d = tmp_path_factory.mktemp("knn")
    exe = tknn.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


def check_program(r):
    """getKNearest of the C++ layer against the brute force under the transform that was found"""
    sP, sQ = r["sP"], r["sQ"]
    for (k, dist), got in zip(r["runs"], r["rows"]):
        same(got, oknn.bruteforce(sP, sQ, k, np.float32(dist) * np.float32(dist), r["C"]))
    assert (r["rows"][0][0] >= 0).any() and (r["rows"][-1][0][:, -1] >= 0).all()


def test_get_k_nearest_on_oracle_shim_hippo(program, tmp_path):
    """the run-example options (-o 0.7 -d 0.01 -n 200) on the hippo golden: the registration is the golden one, and
    getKNearest equals the brute force; it throws before a registration"""
    exe, shim = program
    h = np.load(os.path.join(ROOT, "tests", "golden", "hippo.npz"))
    g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
    r = tknn.run(exe, tmp_path, h["P"], h["Q"], 0.01, 0.7, 200, preload=shim)
    assert r["threw_before"] == 1
    assert r["score"] == g["score"]
    check_program(r)


def test_get_k_nearest_on_oracle_shim_synthetic(program, tmp_path):
    d = common.scenario(6000, 0.5, 0.01, seed=12)["raw"]
    exe, shim = program
    r = tknn.run(exe, tmp_path, d["P"], d["Q"], 0.01, 0.5, 1000, preload=shim)
    assert r["threw_before"] == 1
    check_program(r)
