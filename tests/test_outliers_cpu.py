"""Outlier removal (s4g_statistical_outliers, s4g_radius_outliers) without a GPU: the port's radius counts against the
compiled reference's own kd-tree, its statistical filter against scipy's cKDTree + numpy float64, the rules of both
contracts on degenerate clouds and extreme parameters, the C++ layer's Utils::RemoveStatisticalOutliers and
Utils::RemoveRadiusOutliers on the oracle stand-in, and a labelled cfg3-style pair: the share of outliers removed and of
surface points kept, and a registration of the filtered pair against the compiled reference.

Contracts (include/s4g.h): mean_dist[j] = the mean of sqrt(d^2) over the s4g_knn row of p_j with exclude = j, mu and
sigma in a fixed summation order, j kept iff mean_dist[j] <= mu + std_ratio * sigma; c_j = #{i != j : d^2 < sq_radius},
j kept iff c_j >= min_neighbors, counts capped at min_neighbors."""
import numpy as np
import pytest

from oracle import _build, normals as onormals, outliers as oo, range as orange
from tests import build_shim, common, edges as E, outliers as tout
from tests.test_normals_cpu import register_both, same_registration

needs_ref = pytest.mark.skipif(not orange.ref_available(), reason="oracle/_ref (compiled reference) not present")


def bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


def boundary_cloud(n=2000, delta=0.02, seed=9):
    """a seeded cloud plus, for 6 of its points, targets placed ulps around fl(delta^2) from them
    (tests/edges.py walk_targets): (raw P, raw Q, indices of the anchors, index of the first target)"""
    sc = common.scenario(n, 0.4, delta, seed=seed)
    P0, Q0 = sc["raw"]["P"], sc["raw"]["Q"]
    rng = np.random.RandomState(seed)
    anchors = rng.choice(len(P0), 6, replace=False)
    T = [t for a in anchors for u in E.directions(rng, 1)[:4] for t in E.walk_targets(P0[a], u, delta).values()]
    return np.concatenate([P0, np.asarray(T, np.float32)]).astype(np.float32), Q0, anchors, len(P0)


@needs_ref
def test_radius_counts_equal_reference_range_lists():
    """c_j = the reference kd-tree's range list of p_j minus p_j itself, for every point, at generic radii and at radii
    equal to (and one ulp either side of) fl(d^2) of point pairs placed ulps around delta"""
    delta = 0.02
    Praw, Qraw, anchors, first = boundary_cloud(delta=delta)
    m = orange.RefRange(Praw, Qraw, delta)
    P, _ = m.sampled()
    assert len(P) == len(Praw)
    d2 = np.unique(E.fp32_d2(P[first:], P[anchors]).ravel())
    d2 = d2[np.abs(d2 - np.float32(delta) ** 2) <= 1e-3 * delta ** 2][:8]
    assert len(d2) >= 4
    rs = [-1.0, 0.0, (0.1 * delta) ** 2, 9 * delta * delta, np.inf]
    for x in d2:
        rs += [float(x), float(np.nextafter(x, np.float32(np.inf))), float(np.nextafter(x, np.float32(-np.inf)))]
    flips = 0
    prev = None
    for r in rs:
        off, _, _ = m.query(P, r)
        want = np.diff(off) - (1 if r > 0 else 0)
        keep, counts, raw = oo.radius(P, r, 3, raw=True)
        assert np.array_equal(raw, want), (r, np.argwhere(raw != want)[:5])
        assert np.array_equal(counts, np.minimum(want, 3))
        assert np.array_equal(keep, np.nonzero(want >= 3)[0])
        if prev is not None and r != prev[0]:
            flips += int((raw != prev[1]).sum())
        prev = (r, raw)
    assert flips > 0                                   # the boundary radii do move some counts


@pytest.mark.parametrize("kind", ["synthetic", "labelled", "offcentre1e3"])
def test_statistical_port_agrees_with_scipy(kind):
    """mean distances within a relative 1e-6 of scipy cKDTree + numpy float64 (d^2 is fp32 here), mu and sigma likewise,
    and the masks identical except for points within that tolerance of the threshold"""
    from super4pcs_b200 import synth
    if kind == "synthetic":
        P = synth.make_pair(3000, 0.6, seed=3)["P"]
    elif kind == "labelled":
        P = tout.labelled_pair(6000, seed=5)["P"]
    else:
        P = (synth.make_pair(3000, 0.6, seed=5)["P"].astype(np.float64) * 0.3 + 1e3).astype(np.float32)
    for k in (1, 8, 16, 33, 64):
        mean = oo.mean_rows(P, k)
        mu, sigma = oo.moments(mean)
        for r in (-1.0, 0.0, 1.0, 2.0):
            keep, pmean, pmu, psigma = oo.statistical(P, k, r)
            assert np.array_equal(bits(pmean), bits(mean)) and (pmu, psigma) == (mu, sigma)
            mask, smean, smu, ssigma = oo.scipy_statistical(P, k, r)
            assert np.allclose(mean, smean, rtol=1e-6, atol=0)
            assert abs(mu - smu) <= 1e-6 * smu and abs(sigma - ssigma) <= 1e-6 * ssigma + 1e-6 * smu
            ours = np.zeros(len(P), bool)
            ours[keep] = True
            thr = smu + r * ssigma
            near = np.abs(smean - thr) <= 1e-6 * (abs(thr) + smu)
            assert np.array_equal(ours[~near], mask[~near]), (k, r)
            assert 0 < len(keep) <= len(P)


def test_statistical_rules():
    """nP = 1; identical points and n = 2 (sigma = 0: everything kept at any std_ratio); duplicates; extreme std_ratio"""
    one = np.float32([[0.5, -0.25, 2.0]])
    keep, mean, mu, sigma = oo.statistical(one, 8, -3.0)
    assert list(keep) == [0] and mean[0] == 0 and mu == 0 and sigma == 0
    same = np.tile(np.float32([[0.1, 0.2, 0.3]]), (300, 1))
    two = np.float32([[0, 0, 0], [0.3, 0.4, 0]])
    for P in (same, two):
        for r in (-1e6, -1.0, 0.0, 1.0):
            keep, mean, mu, sigma = oo.statistical(P, 16, r)
            assert sigma == 0 and len(keep) == len(P)
    assert (oo.statistical(two, 1, 0.0)[1] == np.float32(0.5)).all()      # |(0.3, 0.4, 0)| in fp32 then double sqrt
    rng = np.random.RandomState(2)
    P0 = rng.uniform(-1, 1, (500, 3)).astype(np.float32)
    P = np.concatenate([P0, P0[:50]])                                      # 50 points twice: their nearest is at 0
    keep, mean, mu, sigma = oo.statistical(P, 1, 0.0)
    assert (mean[:50] == 0).all() and (mean[500:] == 0).all() and (mean[50:500] > 0).all()
    assert sigma > 0
    assert len(oo.statistical(P, 8, 1e6)[0]) == len(P)
    assert len(oo.statistical(P, 8, -1e6)[0]) == 0
    keep0 = oo.statistical(P, 8, 0.0)
    assert np.array_equal(keep0[0], np.nonzero(keep0[1] <= keep0[2])[0])


def test_radius_rules():
    rng = np.random.RandomState(3)
    P = np.concatenate([rng.uniform(-1, 1, (400, 3)), np.tile([[5, 5, 5]], (4, 1)), [[9, 9, 9]]]).astype(np.float32)
    for mn in (1, 2, 10 ** 4):
        keep, counts, raw = oo.radius(P, 0.0, mn, raw=True)                  # radius 0: every point alone
        assert len(keep) == 0 and (raw == 0).all() and (counts == 0).all()
    keep, counts, raw = oo.radius(P, 1e-12, 1, raw=True)                       # only coincident points count
    assert list(np.nonzero(raw)[0]) == [400, 401, 402, 403] and (raw[400:404] == 3).all()
    assert list(keep) == [400, 401, 402, 403]
    keep, counts, raw = oo.radius(P, np.inf, 10 ** 4, raw=True)               # min_neighbors above every count
    assert (raw == len(P) - 1).all() and np.array_equal(counts, raw) and len(keep) == 0
    keep, counts = oo.radius(P, np.inf, len(P) - 1)
    assert len(keep) == len(P) and (counts == len(P) - 1).all()
    keep, counts, raw = oo.radius(P, 0.25, 2, raw=True)
    assert (counts == np.minimum(raw, 2)).all() and raw[-1] == 0 and -1 + len(P) not in keep


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    d = tmp_path_factory.mktemp("outliers")
    exe = tout.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


def attributes(n, seed):
    rng = np.random.RandomState(seed)
    return rng.normal(0, 1, (n, 3)).astype(np.float32), rng.uniform(0, 1, (n, 3)).astype(np.float32)


@pytest.mark.parametrize("mode,a,b", [("statistical", 16, 1.0), ("statistical", 1, -0.5), ("statistical", 64, 3.0),
                                      ("radius", 0.03, 4), ("radius", 0.0, 1), ("radius", float("inf"), 5000)])
def test_cpp_functions_on_oracle_shim(program, tmp_path, mode, a, b):
    """the port's kept points, in order, with their normals and colours as Point3D held them, and the removed count"""
    exe, shim = program
    P = tout.labelled_pair(4000, seed=8)["P"]
    normals, rgb = attributes(len(P), 2)
    got = tout.run(exe, tmp_path, P, normals, rgb, mode, a, b, preload=shim)
    assert got is not None
    if mode == "statistical":
        keep = oo.statistical(P, a, b)[0]
    else:
        keep = oo.radius(P, np.float32(a) * np.float32(a), b)[0]
    assert got[0] == len(P) - len(keep)
    assert np.array_equal(common.bits(got[1]), common.bits(tout.held(P, normals, rgb)[keep]))
    assert 0 < len(keep) < len(P) or (mode == "radius" and a == 0.0 and len(keep) == 0) or \
        (mode == "radius" and b > len(P) and len(keep) == 0)


def test_cpp_functions_throw_on_bad_arguments(program, tmp_path):
    exe, shim = program
    P = np.random.RandomState(1).rand(100, 3).astype(np.float32)
    normals, rgb = attributes(len(P), 3)
    for mode, a, b in (("statistical", 0, 1.0), ("statistical", 65, 1.0), ("statistical", 8, float("nan")),
                       ("statistical", 8, float("inf")), ("radius", -1.0, 4), ("radius", float("nan"), 4),
                       ("radius", 0.1, 0)):
        assert tout.run(exe, tmp_path, P, normals, rgb, mode, a, b, preload=shim) is None, (mode, a, b)


def test_labelled_pair_removes_outliers_and_keeps_the_surface():
    """cfg3's recipe at 20 000 points, labels known, k = 16, std_ratio = 1: the port removes 74.52 % (P) and 77.65 % (Q)
    of the uniform outliers and keeps every surface point but none or one; at std_ratio = 0.5 it removes 81.47 % /
    84.38 % and keeps 99.99 % of the surface"""
    d = tout.labelled_pair()
    for key, floor1, floor05 in (("P", 0.745, 0.814), ("Q", 0.776, 0.843)):
        X, out = d[key], d["out_" + key]
        assert out.mean() == 0.2
        for r, floor, surface in ((1.0, floor1, 0.9999), (0.5, floor05, 0.999)):
            keep = np.zeros(len(X), bool)
            keep[oo.statistical(X, 16, r)[0]] = True
            assert (~keep[out]).mean() >= floor, (key, r)
            assert keep[~out].mean() >= surface, (key, r)


@pytest.mark.skipif(_build.build_ref() is None, reason="oracle/_ref (compiled reference) not present")
def test_registration_of_filtered_pair_on_oracle_shim(s4g_lib, tmp_path):
    """remove outliers -> estimate normals -> register: the labelled pair filtered by the port (k = 16, std_ratio = 1),
    normals from the port, registered by the C++ layer on the stand-in and by the compiled reference, bit for bit"""
    from super4pcs_b200 import build_cpp
    if build_cpp.build_all()["lib"] is None or _build.build_dropin_harness() is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    d = tout.labelled_pair()
    P, Q = (np.ascontiguousarray(d[key][oo.statistical(d[key], 16, 1.0)[0]]) for key in ("P", "Q"))
    ref, ours = register_both(P, Q, onormals.port(P, 16)[0], onormals.port(Q, 16)[0], tmp_path,
                              preload=build_shim.build())
    same_registration(ref, ours)
