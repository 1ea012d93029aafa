"""s4g_knn on the GPU: the k nearest P points within a radius, for arbitrary query points.

Values: index and sq_dist are bit-equal to the port's brute force (oracle/knn_port.cc) for k in {1, 2, 5, 16, 33, 64} --
every k-instance of the kernel (8, 16, 32 and 64 slots) -- at radii 0, (0.1 delta)^2, delta^2, 9 delta^2, MeanDistance's
and +inf, with and without exclusion, without T and under a rotation, a wrong rigid T and a huge non-rigid one, over the
grid regimes the Verify tests use (4- and 8-cell bricks, widened cells, coarse blocks of 2^3 cells, clouds off-centre at
1e3 and 1.2e4), degenerate clouds (every point identical, planar, line, duplicates, a single point, fewer points than k),
ragged query counts, and queries inside the cloud, on its faces, far outside and NaN.  The brute force's row for k is the
first k of its row for 64, so each case runs it once.  Against the other queries: k = 1 is s4g_nearest, a finite radius
gives the s4g_range-derived prefix, and at delta^2 under T the rows with a neighbour are s4g_verify's count."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import knn as oknn
from tests import common, knn as tknn
from tests import edges as E
from tests.test_decision_edges_gpu import cloud

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S4G_OK, S4G_ERR_ARG, S4G_ERR_STATE = 0, 2, 3   # include/s4g.h
KS = [1, 2, 5, 16, 33, 64]


@pytest.fixture
def make_ctx(s4g_lib, monkeypatch):
    from super4pcs_b200 import Context
    made = []

    def make(cshift_min=None):
        if cshift_min is None:
            monkeypatch.delenv("S4G_CSHIFT_MIN", raising=False)
        else:
            monkeypatch.setenv("S4G_CSHIFT_MIN", str(cshift_min))
        made.append(Context(0))
        return made[-1]
    yield make
    for c in made:
        c.close()


def same(a, b, what=""):
    assert np.array_equal(a[0], b[0]), (what, np.argwhere(a[0] != b[0])[:5])
    assert np.array_equal(common.bits(a[1]), common.bits(b[1])), what


def radii(delta, extent):
    """0, (0.1 delta)^2, delta^2, 9 delta^2, MeanDistance's squared radius 0.2 x extent, +inf"""
    return [0.0, (0.1 * delta) ** 2, delta * delta, 9 * delta * delta, float(np.float32(extent) * np.float32(0.2)), np.inf]


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


def transforms(P, rng):
    """column-major 4x4s: a rotation about the cloud's centre, a wrong rigid motion (another rotation and a shift of a
    third of the extent), and a non-rigid one with coefficients ~1e3"""
    c = P.mean(0).astype(np.float64)
    extent = float(np.abs(P.max(0) - P.min(0)).max())
    out = []
    for R, shift in ((E.rotations(1, rng)[0], 0.0), (E.rotations(1, rng)[0], extent / 3)):
        T = np.eye(4)
        T[:3, :3] = R
        T[:3, 3] = c - R @ c + shift
        out.append(T)
    H = np.eye(4)
    H[:3, :3] = rng.uniform(-1e3, 1e3, (3, 3))
    H[:3, 3] = rng.uniform(-1e3, 1e3, 3)
    out.append(H)
    return [np.ascontiguousarray(T.T).reshape(16).astype(np.float32) for T in out]


def check_all(ctx, P, X, delta, T16s, rng, ks=KS):
    """every radius x T x exclusion x k: bit-equal to the brute force; returns the non-padding entries seen"""
    excl = rng.randint(-1, len(P), len(X)).astype(np.int32)
    extent = float(np.abs(P.max(0) - P.min(0)).max()) + delta
    held = 0
    for T16 in T16s:
        for r in radii(delta, extent):
            for ex in (None, excl):
                want = oknn.bruteforce(P, X, max(ks), r, T16, ex)
                for k in ks:
                    got = ctx.knn(X, k, r, T16, ex)
                    same(got, (want[0][:, :k], want[1][:, :k]), (r, k, T16 is None, ex is None))
                held += int((want[0] >= 0).sum())
    return held


@pytest.mark.parametrize("name,cshift_min", [("centred", None), ("centred", 3), ("brick8", None), ("widened", None),
                                             ("offcentre1e3", None), ("offcentre1e4", None)])
def test_bit_equal_to_bruteforce_over_grid_regimes(make_ctx, name, cshift_min):
    delta = E.REGIMES[name][0]
    P, cases, g = cloud(name, cshift_min=cshift_min or 1)
    ctx = make_ctx(cshift_min)
    ctx.set_cloud_p(P, delta)
    rng = np.random.RandomState(len(P))
    X = np.concatenate([np.asarray([c["t"] for c in cases], np.float32), queries(P, delta, rng)])
    assert check_all(ctx, P, X, delta, [None] + transforms(P, rng), rng) > 0


@pytest.mark.parametrize("kind", ["identical", "planar", "line", "duplicates", "single", "fewer_than_k"])
def test_bit_equal_to_bruteforce_on_degenerate_clouds(make_ctx, kind):
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
        P = np.concatenate([P0, P0[::3], P0[::2]])
    elif kind == "single":
        P = np.array([[0.1, -0.2, 0.3]])
    else:
        P = rng.uniform(-0.05, 0.05, (20, 3))
    P = P.astype(np.float32)
    ctx = make_ctx()
    ctx.set_cloud_p(P, delta)
    X = queries(P, delta, rng, 200, 40, 40)
    X = np.concatenate([X, P[:100]])                           # on the points themselves (d^2 = 0)
    assert check_all(ctx, P, X, delta, [None], rng) > 0
    idx, sq = ctx.knn(X, 64)
    if kind == "identical":                                    # every d^2 ties: the 64 smallest indices
        on = len(X) - 100
        assert (idx[on:] == np.arange(64)).all() and (sq[on:] == 0).all()
    if len(P) < 64:                                            # fewer points than k: padded rows
        assert (idx[:, len(P):] == -1).all() and np.isinf(sq[:, len(P):]).all()


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 127, 128, 129, 1000, 4097])
def test_ragged_query_counts(make_ctx, n):
    sc = common.scenario(5000, 0.4, 0.01, seed=3)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], 0.01)
    X = queries(sc["P"], 0.01, np.random.RandomState(n), n, 0, 0)[:n]
    for k, r in ((5, 0.01 ** 2), (33, np.inf)):
        got = ctx.knn(X, k, r)
        assert got[0].shape == got[1].shape == (n, k)
        same(got, oknn.bruteforce(sc["P"], X, k, r))


def test_far_queries_unbounded(make_ctx):
    """queries 1e3 cell widths outside the grid, unbounded radius: the brute force's rows, no padding"""
    sc = common.scenario(20000, 0.4, 0.005, seed=8)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], 0.005)
    h = ctx.grid_stats()["cell_edge"]
    rng = np.random.RandomState(4)
    d = rng.normal(0, 1, (500, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    lo, hi = sc["P"].min(0), sc["P"].max(0)
    X = (0.5 * (lo + hi) + d * (0.5 * np.abs(hi - lo).max() + 1000 * h)).astype(np.float32)
    X[::5, 0] = hi[0] + 1000 * h                               # straight off a face
    for k in (16, 64):
        got = ctx.knn(X, k)
        assert (got[0] >= 0).all()
        same(got, oknn.bruteforce(sc["P"], X, k))


@pytest.mark.parametrize("n,delta", [(3000, 0.02), (20000, 0.01), (20000, 0.0004)])   # the last: widened cells
def test_consistent_with_nearest_range_and_verify(make_ctx, n, delta):
    """k = 1 is s4g_nearest bit for bit; a finite radius gives the first k of the s4g_range list at the next float,
    exclusion removed; at delta^2 under T the rows with a neighbour are s4g_verify's count"""
    sc = common.scenario(n, 0.4, delta, seed=5)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], delta)
    ctx.set_cloud_q(sc["Q"])
    T16 = common.candidates_colmajor(sc, 6, seed=9, n_near=3)
    counts = ctx.verify(T16)
    sq_eps = float(np.float32(delta) * np.float32(delta))
    ex = np.random.RandomState(1).randint(-1, len(sc["P"]), len(sc["Q"])).astype(np.int32)
    for t in range(len(T16)):
        for r in (sq_eps, 9 * delta * delta, np.inf):
            for e in (None, ex):
                same(ctx.knn(sc["Q"], 1, r, T16[t], e), tuple(a[:, None] for a in ctx.nearest(sc["Q"], r, T16[t], e)))
        for r in (sq_eps, 9 * delta * delta):
            lists = ctx.range_query(sc["Q"], oknn.range_radius(r), T16[t])
            for k in (1, 8, 33):
                for e in (None, ex):
                    same(ctx.knn(sc["Q"], k, r, T16[t], e), oknn.from_range(lists, k, e), (t, r, k))
        idx, _ = ctx.knn(sc["Q"], 5, sq_eps, T16[t])
        assert int((idx[:, 0] >= 0).sum()) == counts[t]
    assert counts[:3].min() > 0


@pytest.mark.parametrize("which", ["self", "near_gt", "wrong"])
def test_full_size_sample(make_ctx, which):
    """1M x 1M (cfg2, delta = 0.003), unbounded: 20K sampled-P points each excluding itself (the normal-estimation
    query), and 20K T q under a near-ground-truth and a wrong T, against the brute force"""
    n, delta = 1_000_000, 0.003
    sc = common.scenario(n, 0.3, delta, seed=42)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], delta)
    sub = np.random.RandomState(0).choice(n, 20000, replace=False)
    if which == "self":
        X, T, ex, k = sc["P"][sub], None, sub.astype(np.int32), 16
    else:
        T16 = common.candidates_colmajor(sc, 2, seed=7, n_near=1)
        X, T, ex, k = sc["Q"][sub], T16[0 if which == "near_gt" else 1], None, 8
    got = ctx.knn(X, k, np.inf, T, ex)
    same(got, oknn.bruteforce(sc["P"], X, k, np.inf, T, ex))
    assert (got[0] >= 0).all()
    if which == "self":
        assert (got[0] != sub[:, None]).all()


def test_dev_and_stats_forms_equal_host_form(make_ctx):
    import torch
    sc = common.scenario(20000, 0.4, 0.01, seed=5)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], 0.01)
    X = queries(sc["P"], 0.01, np.random.RandomState(1), 3000)
    T16 = common.candidates_colmajor(sc, 1, n_near=1)[0]
    ex = np.random.RandomState(2).randint(-1, len(sc["P"]), len(X)).astype(np.int32)
    n = len(X)
    dX, dT, dE = torch.from_numpy(X).cuda(), torch.from_numpy(T16.copy()).cuda(), torch.from_numpy(ex).cuda()
    for k in (1, 9, 64):
        for r in (0.01 ** 2, np.inf):
            for T, dTp in ((None, None), (T16, dT.data_ptr())):
                for e, dEp in ((None, None), (ex, dE.data_ptr())):
                    want = ctx.knn(X, k, r, T, e)
                    d_index = torch.full((n, k), 7, dtype=torch.int32, device="cuda")
                    d_sq = torch.zeros((n, k), dtype=torch.float32, device="cuda")
                    torch.cuda.synchronize()
                    ctx.knn_dev(dX.data_ptr(), n, k, d_index.data_ptr(), d_sq.data_ptr(), r, dTp, dEp)
                    ctx.synchronize()
                    same((d_index.cpu().numpy(), d_sq.cpu().numpy()), want)
                    si, ss, st = ctx.knn(X, k, r, T, e, stats=True)
                    same((si, ss), want)
                    assert st["tested"] >= int((want[0] >= 0).sum()) and st["blocks"] > 0
    d_index = torch.full((n, 4), 7, dtype=torch.int32, device="cuda")
    ctx.knn_dev(dX.data_ptr(), n, 4, d_index.data_ptr(), None)   # sq_dist is optional
    ctx.synchronize()
    assert np.array_equal(d_index.cpu().numpy(), ctx.knn(X, 4)[0])


def test_error_codes(s4g_lib):
    from super4pcs_b200 import Context
    with Context(0) as ctx:
        L, h = ctx._L, ctx.h
        X = np.zeros((4, 3), np.float32)
        idx = np.empty((4, 64), np.int32)
        out2 = np.zeros(2, np.uint64)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        assert L.s4g_knn(h, p(X), 4, None, 4, 1.0, None, p(idx), None) == S4G_ERR_STATE   # before s4g_set_cloud_p
        assert "s4g_set_cloud_p" in L.s4g_error_string(h).decode()
        assert L.s4g_knn_dev(h, p(X), 0, None, 4, 1.0, None, p(idx), None) == S4G_ERR_STATE
        assert L.s4g_knn_probe_stats(h, p(X), 4, None, 4, 1.0, None, p(idx), None, p(out2)) == S4G_ERR_STATE
        ctx.set_cloud_p(np.random.RandomState(0).rand(100, 3).astype(np.float32), 0.05)
        for k in (0, 65, -1):
            assert L.s4g_knn(h, p(X), 4, None, k, 1.0, None, p(idx), None) == S4G_ERR_ARG
            assert "k" in L.s4g_error_string(h).decode()
            assert L.s4g_knn_dev(h, p(X), 4, None, k, 1.0, None, p(idx), None) == S4G_ERR_ARG
        assert L.s4g_knn(h, p(X), 4, None, 4, float("nan"), None, p(idx), None) == S4G_ERR_ARG
        assert "NaN" in L.s4g_error_string(h).decode()
        assert L.s4g_knn(h, None, 4, None, 4, 1.0, None, p(idx), None) == S4G_ERR_ARG
        assert L.s4g_knn(h, p(X), 4, None, 4, 1.0, None, None, None) == S4G_ERR_ARG
        assert L.s4g_knn(h, p(X), -1, None, 4, 1.0, None, p(idx), None) == S4G_ERR_ARG
        assert L.s4g_knn_dev(h, None, 4, None, 4, 1.0, None, None, None) == S4G_ERR_ARG
        assert L.s4g_knn_probe_stats(h, p(X), 4, None, 4, 1.0, None, p(idx), None, None) == S4G_ERR_ARG
        assert L.s4g_knn(None, p(X), 4, None, 4, 1.0, None, p(idx), None) == S4G_ERR_ARG
        assert L.s4g_knn(h, None, 0, None, 4, 1.0, None, None, None) == S4G_OK          # n == 0: no-op
        assert L.s4g_knn_dev(h, None, 0, None, 64, float("inf"), None, None, None) == S4G_OK
        assert L.s4g_knn(h, p(X), 4, None, 64, float("inf"), None, p(idx), None) == S4G_OK
        assert (idx[:, :64] >= 0).all()
        with pytest.raises(Exception):
            ctx.knn(X, 0)


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = tknn.build(tmp_path_factory.mktemp("knn"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


@pytest.mark.parametrize("which", ["hippo", "synthetic"])
def test_cpp_get_k_nearest_equals_bruteforce(program, tmp_path, which):
    """getKNearest of the C++ layer on the real library: the brute force's rows under the transform that was found"""
    if which == "hippo":
        h = np.load(os.path.join(ROOT, "tests", "golden", "hippo.npz"))
        P, Q, overlap, n = h["P"], h["Q"], 0.7, 200
    else:
        d = common.scenario(30000, 0.5, 0.01, seed=12)["raw"]
        P, Q, overlap, n = d["P"], d["Q"], 0.5, 1000
    r = tknn.run(program, tmp_path, P, Q, 0.01, overlap, n)
    assert r["threw_before"] == 1
    for (k, dist), got in zip(r["runs"], r["rows"]):
        same(got, oknn.bruteforce(r["sP"], r["sQ"], k, np.float32(dist) * np.float32(dist), r["C"]))
    assert (r["rows"][0][0] >= 0).any()
