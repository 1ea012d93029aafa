"""The outlier filters on the GPU: s4g_statistical_outliers and s4g_radius_outliers over the resident P.

keep, n_kept, mean_dist, mu, sigma and counts are bit-equal to the port's restatement (oracle/outliers_port.cc on the
brute-force rows of oracle/knn_port.cc) over the grid regimes of the k-nearest tests, at k on both sides of every k_knn
capacity, several std_ratio, degenerate clouds, radii at and one ulp either side of pair distances, and min_neighbors from
1 to 10^4.  On a 1M-point cloud, sampled rows are checked against the port and mu, sigma and the kept set against the
port's reductions of the GPU's mean distances.  The _dev and host forms agree, the error codes hold, the C++ functions
equal Context, and a labelled cfg3-style pair filtered on the GPU registers as the compiled reference does on the
port-filtered clouds, bit for bit."""
import ctypes as C

import numpy as np
import pytest

from oracle import _build, outliers as oo
from tests import common, edges as E, outliers as tout
from tests.test_decision_edges_gpu import cloud
from tests.test_knn_gpu import make_ctx  # noqa: F401  (fixture)
from tests.test_normals_cpu import register_both, same_registration

pytestmark = pytest.mark.gpu

S4G_OK, S4G_ERR_ARG, S4G_ERR_STATE = 0, 2, 3   # include/s4g.h
KS = [1, 8, 9, 16, 17, 32, 33, 64]              # both sides of every k_knn capacity (8, 16, 32, 64 slots)
RATIOS = [-1.0, 0.0, 1.0, 2.0, 1e6]
MIN_NEIGHBORS = [1, 2, 64, 10 ** 4]


def bits(x):
    return np.asarray(x, np.float64).view(np.uint64)


def check_statistical(ctx, P, ks=KS, ratios=RATIOS):
    """every k x std_ratio against the port; returns the number of points removed over all cases"""
    removed = 0
    for k in ks:
        mean = oo.mean_rows(P, k)
        mu, sigma = oo.moments(mean)
        for r in ratios:
            keep, gmean, gmu, gsigma = ctx.statistical_outliers(k, r)
            assert np.array_equal(bits(gmean), bits(mean)), (k, r, np.argwhere(gmean != mean)[:5])
            assert bits(gmu) == bits(mu) and bits(gsigma) == bits(sigma), (k, r)
            want = np.nonzero(oo.flags(mean, mu, sigma, r))[0]
            assert np.array_equal(keep, want), (k, r)
            removed += len(P) - len(keep)
    return removed


def check_radius(ctx, P, radii, mns=MIN_NEIGHBORS):
    kept = 0
    for r in radii:
        for mn in mns:
            keep, counts = ctx.radius_outliers(r, mn)
            wk, wc = oo.radius(P, r, mn)
            assert np.array_equal(counts, wc), (r, mn, np.argwhere(counts != wc)[:5])
            assert np.array_equal(keep, wk), (r, mn)
            kept += len(keep)
    return kept


def radii(delta):
    return [-1.0, 0.0, (0.1 * delta) ** 2, delta * delta, 9 * delta * delta, np.inf]


@pytest.mark.parametrize("name,cshift_min", [("centred", None), ("centred", 3), ("brick8", None), ("widened", None),
                                             ("offcentre1e3", None), ("offcentre1e4", None)])
def test_bit_equal_to_port_over_grid_regimes(make_ctx, name, cshift_min):  # noqa: F811
    delta = E.REGIMES[name][0]
    P, _, _ = cloud(name, cshift_min=cshift_min or 1)
    ctx = make_ctx(cshift_min)
    ctx.set_cloud_p(P, delta)
    assert check_statistical(ctx, P) > 0
    assert check_radius(ctx, P, radii(delta)) > 0


@pytest.mark.parametrize("kind", ["identical", "planar", "line", "duplicates", "single", "pair", "fewer_than_k"])
def test_bit_equal_to_port_on_degenerate_clouds(make_ctx, kind):  # noqa: F811
    rng = np.random.RandomState(11)
    delta = 0.01
    if kind == "identical":
        P = np.tile([[0.1, -0.2, 0.3]], (300, 1))
    elif kind == "planar":
        P = np.concatenate([rng.uniform(-0.3, 0.3, (4000, 2)), np.zeros((4000, 1))], 1)
    elif kind == "line":
        P = np.concatenate([rng.uniform(-0.5, 0.5, (3000, 1)), np.zeros((3000, 2))], 1)
    elif kind == "duplicates":
        P0 = rng.uniform(-0.2, 0.2, (2000, 3))
        P = np.concatenate([P0, P0[::3], P0[::2], np.tile(P0[:1], (70, 1))])
    elif kind == "single":
        P = np.array([[0.1, -0.2, 0.3]])
    elif kind == "pair":
        P = np.array([[0.1, -0.2, 0.3], [0.15, -0.2, 0.3]])
    else:
        P = rng.uniform(-0.05, 0.05, (20, 3))
    P = P.astype(np.float32)
    ctx = make_ctx()
    ctx.set_cloud_p(P, delta)
    check_statistical(ctx, P)
    check_radius(ctx, P, radii(delta))
    if kind in ("identical", "single", "pair"):
        for r in RATIOS:                                # sigma = 0: everything kept
            assert len(ctx.statistical_outliers(8, r)[0]) == len(P)


def test_bit_equal_to_port_at_boundary_radii(make_ctx):  # noqa: F811
    """radii equal to fl(d^2) of P pairs placed ulps around delta (tests/edges.py walk_targets), and one ulp either
    side: the strict test drops the pair at the radius and keeps it one ulp above"""
    rng = np.random.RandomState(4)
    delta = 0.02
    P0 = common.scenario(3000, 0.4, delta, seed=9)["P"]
    anchors = rng.choice(len(P0), 6, replace=False)
    T = [t for a in anchors for u in E.directions(rng, 1)[:4] for t in E.walk_targets(P0[a], u, delta).values()]
    P = np.concatenate([P0, np.asarray(T, np.float32)]).astype(np.float32)
    pair_d2 = np.unique(E.fp32_d2(P[len(P0):], P[anchors]).ravel())
    pair_d2 = pair_d2[np.abs(pair_d2 - np.float32(delta) ** 2) <= 1e-3 * delta ** 2][:6]
    assert len(pair_d2) >= 3
    rs = []
    for d2 in pair_d2:
        rs += [float(d2), float(np.nextafter(d2, np.float32(np.inf))), float(np.nextafter(d2, np.float32(-np.inf)))]
    ctx = make_ctx()
    ctx.set_cloud_p(P, delta)
    check_radius(ctx, P, rs, mns=[1, 2, 8, 64])


def test_full_size_sample(make_ctx):  # noqa: F811
    """1M points (cfg2, delta = 0.003), k = 16: 20 000 sampled mean distances against the port's rows, mu / sigma /
    the kept set against the port's reductions of the GPU's mean distances; radius counts at sampled rows against the
    range query's list lengths"""
    n, delta = 1_000_000, 0.003
    P = common.scenario(n, 0.3, delta, seed=42)["P"]
    ctx = make_ctx()
    ctx.set_cloud_p(P, delta)
    sub = np.sort(np.random.RandomState(0).choice(n, 20000, replace=False))
    keep, mean, mu, sigma = ctx.statistical_outliers(16, 1.0)
    assert np.array_equal(bits(mean[sub]), bits(oo.mean_rows(P, 16, sub)))
    wmu, wsigma = oo.moments(mean)
    assert bits(mu) == bits(wmu) and bits(sigma) == bits(wsigma)
    assert np.array_equal(keep, np.nonzero(oo.flags(mean, mu, sigma, 1.0))[0])
    assert 0.5 * n < len(keep) < n
    for r, mn in ((delta * delta, 4), (9 * delta * delta, 16)):
        keep, counts = ctx.radius_outliers(r, mn)
        off, _, _ = ctx.range_query(P[sub], r)
        assert np.array_equal(counts[sub], np.minimum(np.diff(off) - 1, mn))
        assert np.isin(sub[counts[sub] >= mn], keep).all() and not np.isin(sub[counts[sub] < mn], keep).any()


def test_dev_form_equals_host_form(make_ctx):  # noqa: F811
    import torch
    P = common.scenario(20000, 0.4, 0.01, seed=5)["P"]
    ctx = make_ctx()
    ctx.set_cloud_p(P, 0.01)
    n = len(P)
    dev = lambda dt: torch.full((n,), 7, dtype=dt, device="cuda")  # noqa: E731
    for k in (1, 16, 64):
        for r in (-0.5, 1.0):
            want = ctx.statistical_outliers(k, r)
            keep, nk, mean, out2 = dev(torch.int32), torch.zeros(1, dtype=torch.int64, device="cuda"), \
                dev(torch.float64), torch.zeros(2, dtype=torch.float64, device="cuda")
            torch.cuda.synchronize()
            ctx.statistical_outliers_dev(k, r, keep.data_ptr(), nk.data_ptr(), mean.data_ptr(), out2.data_ptr())
            ctx.synchronize()
            m = int(nk.item())
            assert np.array_equal(keep[:m].cpu().numpy(), want[0])
            assert np.array_equal(bits(mean.cpu().numpy()), bits(want[1]))
            assert np.array_equal(bits(out2.cpu().numpy()), bits([want[2], want[3]]))
            ctx.statistical_outliers_dev(k, r, keep.data_ptr(), nk.data_ptr())       # mean_dist and out2 are optional
            ctx.synchronize()
            assert np.array_equal(keep[:int(nk.item())].cpu().numpy(), want[0])
    for r, mn in ((0.01 ** 2, 4), (9 * 0.01 ** 2, 64)):
        want = ctx.radius_outliers(r, mn)
        keep, nk, counts = dev(torch.int32), torch.zeros(1, dtype=torch.int64, device="cuda"), dev(torch.int32)
        torch.cuda.synchronize()
        ctx.radius_outliers_dev(r, mn, keep.data_ptr(), nk.data_ptr(), counts.data_ptr())
        ctx.synchronize()
        assert np.array_equal(keep[:int(nk.item())].cpu().numpy(), want[0])
        assert np.array_equal(counts.cpu().numpy(), want[1])
        ctx.radius_outliers_dev(r, mn, keep.data_ptr(), nk.data_ptr(), None)
        ctx.synchronize()
        assert np.array_equal(keep[:int(nk.item())].cpu().numpy(), want[0])


def test_error_codes(s4g_lib):
    from super4pcs_b200 import Context
    with Context(0) as ctx:
        L, h = ctx._L, ctx.h
        keep, cnt, mean, out2 = np.empty(100, np.int32), np.empty(100, np.int32), np.empty(100), np.empty(2)
        nk = C.c_int64(0)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        assert L.s4g_statistical_outliers(h, 8, 1.0, p(keep), C.byref(nk), None, None) == S4G_ERR_STATE
        assert "s4g_set_cloud_p" in L.s4g_error_string(h).decode()
        assert L.s4g_statistical_outliers_dev(h, 8, 1.0, p(keep), C.byref(nk), None, None) == S4G_ERR_STATE
        assert L.s4g_radius_outliers(h, 1.0, 4, p(keep), C.byref(nk), None) == S4G_ERR_STATE
        assert L.s4g_radius_outliers_dev(h, 1.0, 4, p(keep), C.byref(nk), None) == S4G_ERR_STATE
        ctx.set_cloud_p(np.random.RandomState(0).rand(100, 3).astype(np.float32), 0.05)
        for k in (0, 65, -1):
            assert L.s4g_statistical_outliers(h, k, 1.0, p(keep), C.byref(nk), None, None) == S4G_ERR_ARG
            assert "k" in L.s4g_error_string(h).decode()
            assert L.s4g_statistical_outliers_dev(h, k, 1.0, p(keep), C.byref(nk), None, None) == S4G_ERR_ARG
        for r in (float("nan"), float("inf"), -float("inf")):
            assert L.s4g_statistical_outliers(h, 8, r, p(keep), C.byref(nk), None, None) == S4G_ERR_ARG
        assert L.s4g_statistical_outliers(h, 8, 1.0, None, C.byref(nk), None, None) == S4G_ERR_ARG
        assert L.s4g_statistical_outliers(h, 8, 1.0, p(keep), None, None, None) == S4G_ERR_ARG
        assert L.s4g_statistical_outliers(None, 8, 1.0, p(keep), C.byref(nk), None, None) == S4G_ERR_ARG
        assert L.s4g_radius_outliers(h, float("nan"), 4, p(keep), C.byref(nk), None) == S4G_ERR_ARG
        for mn in (0, -3):
            assert L.s4g_radius_outliers(h, 1.0, mn, p(keep), C.byref(nk), None) == S4G_ERR_ARG
            assert L.s4g_radius_outliers_dev(h, 1.0, mn, p(keep), C.byref(nk), None) == S4G_ERR_ARG
        assert L.s4g_radius_outliers(h, 1.0, 4, None, C.byref(nk), None) == S4G_ERR_ARG
        assert L.s4g_radius_outliers(None, 1.0, 4, p(keep), C.byref(nk), None) == S4G_ERR_ARG
        assert L.s4g_statistical_outliers(h, 64, 0.0, p(keep), C.byref(nk), p(mean), p(out2)) == S4G_OK
        assert L.s4g_radius_outliers(h, 0.0, 1, p(keep), C.byref(nk), p(cnt)) == S4G_OK   # radius 0: every point alone
        assert nk.value == 0 and (cnt == 0).all()
        with pytest.raises(Exception):
            ctx.radius_outliers(1.0, 0)


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = tout.build(tmp_path_factory.mktemp("outliers"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


def attributes(n, seed):
    rng = np.random.RandomState(seed)
    return rng.normal(0, 1, (n, 3)).astype(np.float32), rng.uniform(0, 1, (n, 3)).astype(np.float32)


@pytest.mark.parametrize("mode,a,b", [("statistical", 16, 1.0), ("statistical", 5, -0.25), ("radius", 0.02, 4),
                                      ("radius", float("inf"), 30000), ("radius", 0.0, 1)])
def test_cpp_functions_equal_context(program, make_ctx, tmp_path, mode, a, b):  # noqa: F811
    """Utils::RemoveStatisticalOutliers / RemoveRadiusOutliers on the real library: the Context filter on the same cloud
    at the functions' grid delta; the survivors keep their order, normals and colours"""
    d = tout.labelled_pair(20000, seed=3)
    P = d["P"]
    normals, rgb = attributes(len(P), 1)
    got = tout.run(program, tmp_path, P, normals, rgb, mode, a, b)
    assert got is not None
    ctx = make_ctx()
    if mode == "statistical":
        ctx.set_cloud_p(P, tout.grid_delta(P, a))
        keep = ctx.statistical_outliers(a, b)[0]
    else:
        ctx.set_cloud_p(P, tout.radius_delta(P, a, b))
        keep = ctx.radius_outliers(float(np.float32(a) * np.float32(a)), b)[0]
    assert got[0] == len(P) - len(keep)
    assert np.array_equal(common.bits(got[1]), common.bits(tout.held(P, normals, rgb)[keep]))


def test_labelled_pair_filtered_on_gpu_registers_as_reference(s4g_lib, tmp_path):
    """cfg3-style pair (20 000 points each, 20 % uniform outliers, labels known): the GPU's statistical filter (k = 16,
    std_ratio = 1) keeps what the port keeps; then normals on the GPU and the registration of the C++ layer on the real
    library equal the compiled reference's on the same filtered clouds, bit for bit"""
    from super4pcs_b200 import Context, build_cpp
    if not _build.build_ref() or build_cpp.build_all()["lib"] is None or _build.build_dropin_harness() is None:
        pytest.skip("oracle/_ref or the C++ layer not present")
    d = tout.labelled_pair()
    out = {}
    for key in ("P", "Q"):
        X = d[key]
        with Context(0) as ctx:
            ctx.set_cloud_p(X, tout.grid_delta(X, 16))
            keep = ctx.statistical_outliers(16, 1.0)[0]
            assert np.array_equal(keep, oo.statistical(X, 16, 1.0)[0])
            Xf = np.ascontiguousarray(X[keep])
            ctx.set_cloud_p(Xf, tout.grid_delta(Xf, 16))
            out[key], out[key + "n"] = Xf, ctx.normals(16)[0]
    same_registration(*register_both(out["P"], out["Q"], out["Pn"], out["Qn"], tmp_path))
