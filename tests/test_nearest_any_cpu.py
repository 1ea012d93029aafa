"""The restricted closest-point query at any radius (s4g_nearest) and MeanDistance without a GPU: the port's brute force
against the compiled reference's own kd-tree (KdTree::doQueryRestrictedClosestIndex) and its P_mean_distance_, and the
C++ layer's MeanDistance / getCorrespondences(nearest, sq_dist, max_distance) on the oracle stand-in of libs4g.

Contract (include/s4g.h): index = the P point with the smallest d^2 <= sq_radius and index != exclude, equal d^2 -> the
smallest index, -1 when none; sq_dist = that d^2 bit for bit (+inf for -1).  The kd-tree keeps the last point of equal
distance its traversal visits, and its pruning test (node distance < best, strict) can stop it before a point whose d^2
equals sq_radius exactly (at sq_radius = 0 it finds nothing).  So: wherever the reference finds a neighbour ours has the
same d^2, and the same index unless that d^2 is a tie (then ours is the smaller index); where only ours finds one, its
d^2 is exactly sq_radius."""
import os

import numpy as np
import pytest

from oracle import nearest_any as ona
from tests import common, nearest_any

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not ona.ref_available(), reason="oracle/_ref (compiled reference) not present")


def transformed(X, T16):
    """y = T x in the reference's operation order (fp32), or x"""
    X = np.asarray(X, np.float32)
    if T16 is None:
        return X
    T = np.asarray(T16, np.float32).reshape(4, 4).T
    y = np.empty_like(X)
    for r in range(3):
        y[:, r] = (((T[r, 0] * X[:, 0]).astype(np.float32) + (T[r, 1] * X[:, 1]).astype(np.float32)).astype(np.float32)
                   + (T[r, 2] * X[:, 2]).astype(np.float32)).astype(np.float32) + T[r, 3]
    return y


def sq_to(P, Y, idx):
    d = (Y - P[idx]).astype(np.float32)
    return (d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])).astype(np.float32)


def check_against_reference(P, X, sq_radius, T16, index, sq, ref_index, ref_sq):
    """ours (index, sq) against the reference's kd-tree answer for the same queries; returns (#ties, #boundary-only)"""
    ref_hit, hit = ref_index >= 0, index >= 0
    assert (hit[ref_hit]).all()
    assert np.array_equal(common.bits(sq[ref_hit]), common.bits(ref_sq[ref_hit]))
    only = hit & ~ref_hit                                   # the kd-tree's strict pruning at d^2 == sq_radius
    assert (sq[only] == np.float32(sq_radius)).all()
    assert np.isinf(sq[~hit]).all() and (index[~hit] == -1).all()
    diff = np.nonzero(ref_hit & (index != ref_index))[0]
    if len(diff):
        Y = transformed(X[diff], T16)
        assert np.array_equal(common.bits(sq_to(P, Y, index[diff])), common.bits(sq_to(P, Y, ref_index[diff])))
        assert (index[diff] < ref_index[diff]).all()
    return len(diff), int(only.sum())


def queries(P, delta, rng, n_in=400, n_edge=100, n_far=100):
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


def radii(delta, diameter):
    return [0.0, (0.1 * delta) ** 2, delta * delta, (3 * delta) ** 2, float(np.float32(diameter) * np.float32(0.2)), np.inf]


def compare_all(m, P, X, delta, diameter, T16s, excl):
    """every radius x T x with / without exclusion: bit-equal brute force vs the reference's kd-tree"""
    ties = hits = 0
    for T16 in T16s:
        for r in radii(delta, diameter):
            for ex in (None, excl):
                ri, rs = m.query(X, r, T16, ex)
                pi, ps = ona.bruteforce(P, X, r, T16, ex)
                t, _ = check_against_reference(P, X, r, T16, pi, ps, ri, rs)
                ties += t
                hits += int((ri >= 0).sum())
                assert (pi[-3:] == -1).all()                # NaN queries find nothing
                if ex is not None:
                    assert not ((pi >= 0) & (pi == ex)).any()     # the excluded point is never returned
    return ties, hits


@needs_ref
@pytest.mark.parametrize("n,delta,seed", [(2000, 0.02, 1), (3000, 0.01, 4)])
def test_bruteforce_matches_reference_kdtree_on_seeded_clouds(n, delta, seed):
    sc = common.scenario(n, 0.4, delta, seed=seed)
    m = ona.RefNearestAny(sc["raw"]["P"], sc["raw"]["Q"], delta)
    P, Q = m.sampled()
    diameter, _ = m.diameter_and_mean_distance()
    rng = np.random.RandomState(seed)
    X = queries(P, delta, rng)
    excl = rng.randint(-1, len(P), len(X)).astype(np.int32)
    T16s = [None, common.candidates_colmajor(sc, 2, seed=seed, n_near=1)[0], common.candidates_colmajor(sc, 2, seed=seed)[1]]
    ties, hits = compare_all(m, P, X, delta, diameter, T16s, excl)
    assert hits > 1000
    # the sampled P points themselves, each excluding itself (MeanDistance's query) and not
    self_ = np.arange(len(P), dtype=np.int32)
    for r in radii(delta, diameter):
        ri, rs = m.query(P, r, None, self_)
        pi, ps = ona.bruteforce(P, P, r, None, self_)
        check_against_reference(P, P, r, None, pi, ps, ri, rs)
        assert (pi != self_).all()


@needs_ref
def test_bruteforce_matches_reference_kdtree_on_hippo_samples():
    g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
    m = ona.RefNearestAny(g["stage_P"], g["stage_Q"], 0.01)
    P, Q = m.sampled()
    diameter, _ = m.diameter_and_mean_distance()
    rng = np.random.RandomState(3)
    X = np.concatenate([queries(P, 0.01, rng, 300, 60, 60)[:-3], Q[:300], queries(P, 0.01, rng, 0, 0, 0)])
    excl = rng.randint(-1, len(P), len(X)).astype(np.int32)
    _, hits = compare_all(m, P, X, 0.01, diameter, [None, g["stage_b0_tcs_T"]], excl)
    assert hits > 1000


@needs_ref
def test_exact_ties_resolve_to_the_smallest_index():
    """duplicated P points: every neighbour that has a copy is a tie at any radius; ours is the first copy"""
    sc = common.scenario(1500, 0.4, 0.02, seed=9)
    P0 = sc["raw"]["P"]
    m = ona.RefNearestAny(np.concatenate([P0, P0[::2]]), sc["raw"]["Q"], 0.02)
    P, _ = m.sampled()
    n0 = len(P0)
    X = queries(P, 0.02, np.random.RandomState(2), 500, 50, 50)
    for r in (0.02 ** 2, np.inf):
        ri, rs = m.query(X, r)
        pi, ps = ona.bruteforce(P, X, r)
        ties, _ = check_against_reference(P, X, r, None, pi, ps, ri, rs)
        assert (pi[pi >= 0] < n0).all()                                    # never a later copy
        assert ties > 0
    # self-exclusion on the duplicated points: the copy is found at d^2 = 0
    self_ = np.arange(len(P), dtype=np.int32)
    pi, ps = ona.bruteforce(P, P, np.inf, None, self_)
    ri, rs = m.query(P, np.inf, None, self_)
    check_against_reference(P, P, np.inf, None, pi, ps, ri, rs)
    dup = np.arange(0, n0, 2)
    assert (pi[dup] == n0 + dup // 2).all() and (ps[dup] == 0).all()


@needs_ref
@pytest.mark.parametrize("which", ["seeded", "hippo_keep_all", "hippo_sampled"])
def test_mean_distance_reproduced_from_bruteforce(which):
    """the reference's P_mean_distance_ (its init, on the P_diameter_ its RNG drew) bit for bit from the brute force's
    neighbours of every sampled-P point with exclusion of itself at squared radius 0.2 x P_diameter_"""
    if which == "seeded":
        sc = common.scenario(2500, 0.4, 0.01, seed=7)
        m = ona.RefNearestAny(sc["raw"]["P"], sc["raw"]["Q"], 0.01)
    elif which == "hippo_keep_all":
        g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
        m = ona.RefNearestAny(g["stage_P"], g["stage_Q"], 0.01)
    else:
        h = np.load(os.path.join(ROOT, "tests", "golden", "hippo.npz"))
        m = ona.RefNearestAny(h["P"], h["Q"], 0.01, overlap=0.7, sample_size=200)
    P, _ = m.sampled()
    diameter, want = m.diameter_and_mean_distance()
    r = np.float32(diameter) * np.float32(0.2)
    pi, _ = ona.bruteforce(P, P, r, None, np.arange(len(P), dtype=np.int32))
    assert (pi >= 0).sum() > 0.9 * len(P)
    assert common.bits(np.float32(ona.mean_distance(P, pi))) == common.bits(np.float32(want))


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    from tests import build_shim
    d = tmp_path_factory.mktemp("nearest_any")
    exe = nearest_any.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


def check_program(r, delta, P=None):
    """MeanDistance and the getCorrespondences overload of the C++ layer against the brute force"""
    sP, sQ = r["sP"], r["sQ"]
    pi, _ = ona.bruteforce(sP, sP, np.float32(r["diameter"]) * np.float32(0.2), None, np.arange(len(sP), dtype=np.int32))
    assert common.bits(r["mean_distance"]) == common.bits(ona.mean_distance(sP, pi))
    for k, dist in enumerate(r["max_distance"]):
        qi, qs = ona.bruteforce(sP, sQ, np.float32(dist) * np.float32(dist), r["C"])
        assert np.array_equal(r["nearest"][k], qi)
        assert np.array_equal(common.bits(r["sq"][k]), common.bits(qs))
    assert np.array_equal(r["nearest"][0], r["nearest_delta"])       # max_distance = delta: the two-argument form
    assert np.array_equal(common.bits(r["sq"][0]), common.bits(r["sq_delta"]))
    assert (r["nearest"][-1] >= 0).all()                              # +inf: every sampled-Q point has a neighbour


def test_mean_distance_and_correspondences_on_oracle_shim_hippo(program, tmp_path):
    """the run-example options (-o 0.7 -d 0.01 -n 200) on the hippo golden: the registration is the golden one,
    MeanDistance equals the brute force's (and the reference's P_mean_distance_ when the reference is present)"""
    exe, shim = program
    h = np.load(os.path.join(ROOT, "tests", "golden", "hippo.npz"))
    g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
    r = nearest_any.run(exe, tmp_path, h["P"], h["Q"], 0.01, 0.7, 200, preload=shim)
    assert r["threw_before"] == 1
    assert r["score"] == g["score"] and np.array_equal(common.bits(r["T"]), common.bits(g["T_colmajor"]))
    check_program(r, 0.01)
    if ona.ref_available():
        m = ona.RefNearestAny(h["P"], h["Q"], 0.01, overlap=0.7, sample_size=200)
        diameter, want = m.diameter_and_mean_distance()
        assert common.bits(r["diameter"]) == common.bits(np.float32(diameter))
        assert common.bits(r["mean_distance"]) == common.bits(np.float32(want))


def test_mean_distance_and_correspondences_on_oracle_shim_synthetic(program, tmp_path):
    d = common.scenario(6000, 0.5, 0.01, seed=12)["raw"]
    exe, shim = program
    r = nearest_any.run(exe, tmp_path, d["P"], d["Q"], 0.01, 0.5, 1000, preload=shim)
    check_program(r, 0.01)
    if ona.ref_available():
        m = ona.RefNearestAny(d["P"], d["Q"], 0.01, overlap=0.5, sample_size=1000)
        assert common.bits(r["mean_distance"]) == common.bits(np.float32(m.diameter_and_mean_distance()[1]))
