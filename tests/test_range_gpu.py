"""s4g_range on the GPU: every P point within a radius of arbitrary query points.

Values: offsets, indices and sq_dist are bit-equal to the port's brute force (oracle/range_port.cc) at every radius, with
and without T, over the grid regimes the Verify tests use (4- and 8-cell bricks, widened cells, coarse blocks of 2^3
cells), off-centre clouds, planar, single-point, duplicated and line P, ragged query counts, for queries inside the
cloud, on its decision faces (d^2 exactly delta^2, and a few floats either side), far outside and NaN.  Against
s4g_nearest: a list is non-empty exactly when the nearest point lies strictly inside the radius, and its smallest
(d^2, j) is that point.  At delta^2 the non-empty lists are the inliers s4g_verify counts, less the exact ties."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import range as orange
from tests import common, range as trange
from tests import edges as E
from tests.test_decision_edges_gpu import cloud

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S4G_OK, S4G_ERR_ARG, S4G_ERR_STATE = 0, 2, 3   # include/s4g.h


@pytest.fixture
def make_ctx(s4g_lib, monkeypatch):
    from super4pcs_b200 import Context
    made = []

    def make(cshift_min=None, sort_window=None):
        for var, v in (("S4G_CSHIFT_MIN", cshift_min), ("S4G_RANGE_SORT_WINDOW", sort_window)):
            if v is None:
                monkeypatch.delenv(var, raising=False)
            else:
                monkeypatch.setenv(var, str(v))
        made.append(Context(0))
        return made[-1]
    yield make
    for c in made:
        c.close()


def same(a, b):
    assert np.array_equal(a[0], b[0]), np.nonzero(a[0] != b[0])[0][:5]
    assert np.array_equal(a[1], b[1])
    assert np.array_equal(common.bits(a[2]), common.bits(b[2]))


def radii(delta, extent):
    """0, (0.1 delta)^2, delta^2, (3 delta)^2, MeanDistance's squared radius 0.2 x extent, +inf"""
    return [0.0, (0.1 * delta) ** 2, delta * delta, (3 * delta) ** 2, float(np.float32(extent) * np.float32(0.2)), np.inf]


def queries(P, delta, rng, n_in=300, n_edge=80, n_far=80, far_cells=1000):
    """jittered P points, points on the faces of the cloud's box, points up to `far_cells` cell widths outside, NaN"""
    lo, hi = P.min(0).astype(np.float64), P.max(0).astype(np.float64)
    c = 0.5 * (lo + hi)
    pick = P[rng.randint(0, len(P), n_in)] + rng.normal(0, 2 * delta, (n_in, 3))
    edge = rng.uniform(lo, hi, (n_edge, 3))
    ax = rng.randint(0, 3, n_edge)
    edge[np.arange(n_edge), ax] = np.where(rng.rand(n_edge) < 0.5, lo[ax], hi[ax])
    d = rng.normal(0, 1, (n_far, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    far = c + d * (0.5 * np.abs(hi - lo).max() + rng.uniform(1, far_cells, (n_far, 1)) * 2.02 * delta)
    nan = np.array([[np.nan, 0, 0], [0, np.nan, 0], [np.nan] * 3])
    return np.concatenate([pick, edge, far, nan]).astype(np.float32)


def check_all(ctx, P, X, delta, T16s):
    """every radius x T: bit-equal to the brute force; returns the entries seen"""
    extent = float(np.abs(P.max(0) - P.min(0)).max()) + delta
    total = 0
    for T16 in T16s:
        for r in radii(delta, extent):
            got = ctx.range_query(X, r, T16)
            same(got, orange.bruteforce(P, X, r, T16))
            total += int(got[0][-1])
    return total


@pytest.mark.parametrize("name,cshift_min", [("centred", None), ("centred", 3), ("brick8", None), ("widened", None),
                                             ("offcentre1e3", None)])
def test_bit_equal_to_bruteforce_over_grid_regimes(make_ctx, name, cshift_min):
    delta = E.REGIMES[name][0]
    P, cases, g = cloud(name, cshift_min=cshift_min or 1)
    ctx = make_ctx(cshift_min)
    ctx.set_cloud_p(P, delta)
    rng = np.random.RandomState(len(P))
    X = np.concatenate([np.asarray([c["t"] for c in cases], np.float32), queries(P, delta, rng)])
    R = E.rotations(1, rng)[0]
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = R
    T[:3, 3] = P.mean(0) - R @ P.mean(0)                       # a rotation about the cloud's centre
    assert check_all(ctx, P, X, delta, [None, T.T.reshape(16)]) > 0


@pytest.mark.parametrize("kind", ["planar", "single", "duplicates", "line"])
def test_bit_equal_to_bruteforce_on_degenerate_clouds(make_ctx, kind):
    rng = np.random.RandomState(11)
    delta = 0.01
    if kind == "planar":
        P = np.concatenate([rng.uniform(-0.3, 0.3, (4000, 2)), np.zeros((4000, 1))], 1)
    elif kind == "single":
        P = np.array([[0.1, -0.2, 0.3]])
    elif kind == "duplicates":
        P0 = rng.uniform(-0.2, 0.2, (2000, 3))
        P = np.concatenate([P0, P0[::3], P0[::2]])
    else:
        P = np.concatenate([rng.uniform(-0.5, 0.5, (3000, 1)), np.zeros((3000, 2))], 1)
    P = P.astype(np.float32)
    ctx = make_ctx()
    ctx.set_cloud_p(P, delta)
    X = queries(P, delta, rng, 200, 40, 40)
    if kind != "single":
        X = np.concatenate([X, P[:100]])                       # on the points themselves (d^2 = 0)
    assert check_all(ctx, P, X, delta, [None]) > 0


@pytest.mark.parametrize("n", [0, 1, 31, 129, 1000, 4097])
def test_ragged_query_counts(make_ctx, n):
    sc = common.scenario(5000, 0.4, 0.01, seed=3)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], 0.01)
    X = queries(sc["P"], 0.01, np.random.RandomState(n), n, 0, 0)[:n]
    for r in (0.01 ** 2, (0.05) ** 2):
        got = ctx.range_query(X, r)
        same(got, orange.bruteforce(sc["P"], X, r))
        assert len(got[0]) == n + 1 and got[0][0] == 0


def test_multi_chunk_sort_equals_single(make_ctx):
    """the per-list sort in windows (the path of results over 2^31 entries, here forced by a small window): the same
    lists as one window"""
    sc = common.scenario(20000, 0.4, 0.01, seed=6)
    X = queries(sc["P"], 0.01, np.random.RandomState(5), 2000, 100, 100)
    r = 0.08 ** 2
    want = orange.bruteforce(sc["P"], X, r)
    assert want[0][-1] > 80000
    for window in (None, 997, 40000):
        ctx = make_ctx(sort_window=window)
        ctx.set_cloud_p(sc["P"], 0.01)
        same(ctx.range_query(X, r), want)


@pytest.mark.parametrize("n,delta", [(3000, 0.02), (20000, 0.01), (20000, 0.0004)])   # the last: widened cells
def test_against_nearest_and_verify(make_ctx, n, delta):
    """the same radius for s4g_nearest: a list is non-empty exactly when the nearest d^2 is strictly below it, and its
    smallest (d^2, j) is the nearest answer.  At delta^2 under the candidates: the non-empty lists are s4g_verify's count
    less the queries whose nearest d^2 is exactly delta^2"""
    sc = common.scenario(n, 0.4, delta, seed=5)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], delta)
    ctx.set_cloud_q(sc["Q"])
    T16 = common.candidates_colmajor(sc, 6, seed=9, n_near=3)
    counts = ctx.verify(T16)
    sq_eps = float(np.float32(delta) * np.float32(delta))
    for k in range(len(T16)):
        for r in (sq_eps, (3 * delta) ** 2):
            off, idx, sq = ctx.range_query(sc["Q"], r, T16[k])
            ni, ns = ctx.nearest(sc["Q"], r, T16[k])
            nonempty = np.diff(off) > 0
            assert np.array_equal(nonempty, (ni >= 0) & (ns < np.float32(r)))
            rows = np.nonzero(nonempty)[0]
            seg = np.repeat(np.arange(len(rows)), np.diff(off)[rows])
            order = np.lexsort((idx, sq.view(np.int32), seg))                  # by list, then (d^2, j)
            first = order[np.searchsorted(seg[order], np.arange(len(rows)))]
            assert np.array_equal(idx[first], ni[rows]) and np.array_equal(common.bits(sq[first]), common.bits(ns[rows]))
            if r == sq_eps:
                ties = int(((ni >= 0) & (ns == np.float32(r))).sum())
                assert int(nonempty.sum()) == counts[k] - ties
    assert counts[:3].min() > 0


@pytest.mark.parametrize("which", ["delta", "mean_distance"])
def test_full_size_sample(make_ctx, which):
    """1M x 1M (cfg2, delta = 0.003) against the brute force: 20K sampled-P points and 20K T q under a near-ground-truth
    T at delta^2; at MeanDistance's squared radius (0.2 x extent) each list holds ~20 % of P, so 200 queries"""
    n, delta = 1_000_000, 0.003
    sc = common.scenario(n, 0.3, delta, seed=42)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], delta)
    if which == "delta":
        sub = np.random.RandomState(0).choice(n, 20000, replace=False)
        r = float(np.float32(delta) * np.float32(delta))
        T = common.candidates_colmajor(sc, 1, seed=7, n_near=1)[0]
        for X, T16 in ((sc["P"][sub], None), (sc["Q"][sub], T)):
            got = ctx.range_query(X, r, T16)
            same(got, orange.bruteforce(sc["P"], X, r, T16))
            assert got[0][-1] > 0
    else:
        sub = np.random.RandomState(1).choice(n, 200, replace=False)
        r = float(np.float32(np.abs(sc["P"].max(0) - sc["P"].min(0)).max()) * np.float32(0.2))
        got = ctx.range_query(sc["P"][sub], r)
        same(got, orange.bruteforce(sc["P"], sc["P"][sub], r))
        assert got[0][-1] > 200 * 10000


def test_dev_form_equals_host_form(make_ctx):
    import torch
    sc = common.scenario(20000, 0.4, 0.01, seed=5)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], 0.01)
    X = queries(sc["P"], 0.01, np.random.RandomState(1), 3000)
    T16 = common.candidates_colmajor(sc, 1, n_near=1)[0]
    n = len(X)
    dX, dT = torch.from_numpy(X).cuda(), torch.from_numpy(T16.copy()).cuda()
    for r in (0.01 ** 2, 0.04 ** 2):
        for T, dTp in ((None, None), (T16, dT.data_ptr())):
            want = ctx.range_query(X, r, T)
            d_off = torch.full((n + 1,), -7, dtype=torch.int64, device="cuda")
            torch.cuda.synchronize()
            ctx.range_count_dev(dX.data_ptr(), n, d_off.data_ptr(), r, dTp)
            ctx.synchronize()
            total = int(d_off[n].item())
            d_idx = torch.full((max(total, 1),), -7, dtype=torch.int32, device="cuda")
            d_sq = torch.zeros(max(total, 1), dtype=torch.float32, device="cuda")
            for with_sq in (True, False):
                ctx.range_fill_dev(dX.data_ptr(), n, d_off.data_ptr(), total, d_idx.data_ptr(),
                                   d_sq.data_ptr() if with_sq else None, r, dTp)
                ctx.synchronize()
                same((d_off.cpu().numpy(), d_idx.cpu().numpy()[:total], d_sq.cpu().numpy()[:total]), want)


def test_error_codes(s4g_lib):
    from super4pcs_b200 import Context
    with Context(0) as ctx:
        L, h = ctx._L, ctx.h
        X = np.zeros((4, 3), np.float32)
        off = np.full(5, -1, np.int64)
        tot = C.c_int64(-1)
        idx = np.empty(64, np.int32)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        assert L.s4g_get_range(h, p(idx), None) == S4G_ERR_STATE                        # before any s4g_range
        assert L.s4g_range(h, p(X), 4, None, 1.0, p(off), C.byref(tot)) == S4G_ERR_STATE   # before s4g_set_cloud_p
        assert L.s4g_range_count_dev(h, p(X), 0, None, 1.0, None) == S4G_ERR_STATE
        assert L.s4g_range_fill_dev(h, p(X), 0, None, 1.0, None, 0, None, None) == S4G_ERR_STATE
        ctx.set_cloud_p(np.random.RandomState(0).rand(100, 3).astype(np.float32), 0.05)
        assert L.s4g_get_range(h, p(idx), None) == S4G_ERR_STATE                        # still no result
        assert L.s4g_range(h, p(X), -1, None, 1.0, p(off), C.byref(tot)) == S4G_ERR_ARG
        assert L.s4g_range(h, None, 4, None, 1.0, p(off), C.byref(tot)) == S4G_ERR_ARG
        assert L.s4g_range(h, p(X), 4, None, 1.0, None, C.byref(tot)) == S4G_ERR_ARG
        assert L.s4g_range(h, p(X), 4, None, 1.0, p(off), None) == S4G_ERR_ARG
        assert L.s4g_range(h, p(X), 4, None, float("nan"), p(off), C.byref(tot)) == S4G_ERR_ARG
        assert L.s4g_range(None, p(X), 4, None, 1.0, p(off), C.byref(tot)) == S4G_ERR_ARG
        assert L.s4g_range_count_dev(h, None, 4, None, 1.0, None) == S4G_ERR_ARG
        assert L.s4g_range_count_dev(h, p(X), -1, None, 1.0, p(off)) == S4G_ERR_ARG
        assert L.s4g_range_count_dev(h, p(X), 4, None, float("nan"), p(off)) == S4G_ERR_ARG
        assert L.s4g_range_fill_dev(h, p(X), 4, None, 1.0, p(off), -1, p(idx), None) == S4G_ERR_ARG
        assert L.s4g_range_fill_dev(h, p(X), 4, None, 1.0, p(off), 3, None, None) == S4G_ERR_ARG
        assert L.s4g_range_fill_dev(h, p(X), 4, None, float("nan"), p(off), 0, None, None) == S4G_ERR_ARG
        assert L.s4g_range_count_dev(h, None, 0, None, 1.0, None) == S4G_OK             # n == 0: no-op
        assert L.s4g_range_fill_dev(h, None, 0, None, 1.0, None, 0, None, None) == S4G_OK
        off[0] = -1
        assert L.s4g_range(h, None, 0, None, 1.0, p(off), C.byref(tot)) == S4G_OK       # writes offsets[0] = 0
        assert off[0] == 0 and tot.value == 0
        assert L.s4g_get_range(h, None, None) == S4G_OK                                 # an empty result
        assert L.s4g_range(h, p(X), 4, None, float("inf"), p(off), C.byref(tot)) == S4G_OK
        assert tot.value == 400 and list(off) == [0, 100, 200, 300, 400]
        assert L.s4g_get_range(h, None, None) == S4G_ERR_ARG
        big = np.empty(400, np.int32)
        assert L.s4g_get_range(h, p(big), None) == S4G_OK
        assert np.array_equal(big, np.tile(np.arange(100, dtype=np.int32), 4))
        assert L.s4g_range(h, p(X), 4, None, 0.0, p(off), C.byref(tot)) == S4G_OK       # sq_radius 0: empty lists
        assert tot.value == 0 and (off == 0).all()
        assert L.s4g_range(h, p(X), 4, None, float("nan"), p(off), C.byref(tot)) == S4G_ERR_ARG
        assert L.s4g_get_range(h, p(big), None) == S4G_ERR_STATE                        # a failed call leaves none


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = trange.build(tmp_path_factory.mktemp("range"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


@pytest.mark.parametrize("which", ["hippo", "synthetic"])
def test_cpp_get_neighbors_equals_bruteforce(program, tmp_path, which):
    """getNeighbors of the C++ layer on the real library: the brute force's lists under the transform that was found"""
    if which == "hippo":
        h = np.load(os.path.join(ROOT, "tests", "golden", "hippo.npz"))
        P, Q, overlap, n = h["P"], h["Q"], 0.7, 200
    else:
        d = common.scenario(30000, 0.5, 0.01, seed=12)["raw"]
        P, Q, overlap, n = d["P"], d["Q"], 0.5, 1000
    r = trange.run(program, tmp_path, P, Q, 0.01, overlap, n)
    assert r["threw_before"] == 1
    for dist, got in zip(r["max_distance"], r["lists"]):
        same(got, orange.bruteforce(r["sP"], r["sQ"], np.float32(dist) * np.float32(dist), r["C"]))
    assert r["lists"][0][0][-1] > 0
