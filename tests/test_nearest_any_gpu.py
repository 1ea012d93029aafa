"""s4g_nearest on the GPU: the restricted closest-point query at any radius, for arbitrary query points.

Values: index and sq_dist are bit-equal to the port's brute force (oracle/nearest_any_port.cc) at every radius, with and
without exclusion and T, over the grid regimes the Verify tests use (4- and 8-cell bricks, widened cells, coarse blocks
of 2^3 cells, clouds off-centre at 1e3 and 1.2e4, planar, single-point and duplicated P, ragged query counts), for
queries inside the cloud, on its decision faces, far outside and NaN.  At delta^2 with T the answer is
s4g_verify_nearest's.  The C++ layer's MeanDistance equals the reference's P_mean_distance_."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import nearest_any as ona
from tests import common, nearest_any
from tests import edges as E
from tests.test_decision_edges_gpu import cloud

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S4G_OK, S4G_ERR_ARG, S4G_ERR_STATE = 0, 2, 3   # include/s4g.h


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


def radii(delta, extent):
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


def check_all(ctx, P, X, delta, T16s, rng):
    """every radius x T x exclusion: bit-equal to the brute force"""
    excl = rng.randint(-1, len(P), len(X)).astype(np.int32)
    extent = float(np.abs(P.max(0) - P.min(0)).max()) + delta
    hits = 0
    for T16 in T16s:
        for r in radii(delta, extent):
            for ex in (None, excl):
                index, sq = ctx.nearest(X, r, T16, ex)
                pi, ps = ona.bruteforce(P, X, r, T16, ex)
                assert np.array_equal(index, pi), (r, ex is None, np.nonzero(index != pi)[0][:5])
                assert np.array_equal(common.bits(sq), common.bits(ps)), r
                hits += int((index >= 0).sum())
    return hits


@pytest.mark.parametrize("name,cshift_min", [("centred", None), ("centred", 3), ("brick8", None), ("widened", None),
                                             ("offcentre1e3", None), ("offcentre1e4", None)])
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
    assert check_all(ctx, P, X, delta, [None, T.T.reshape(16)], rng) > 0


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
    X = queries(P, delta, rng)
    if kind != "single":
        X = np.concatenate([X, P[:200]])                       # on the points themselves (ties at d^2 = 0)
    assert check_all(ctx, P, X, delta, [None], rng) > 0
    if kind == "duplicates":                                   # self-exclusion finds the copy at 0
        index, sq = ctx.nearest(P, np.inf, None, np.arange(len(P), dtype=np.int32))
        pi, ps = ona.bruteforce(P, P, np.inf, None, np.arange(len(P), dtype=np.int32))
        assert np.array_equal(index, pi) and (sq[:2000:3] == 0).all()


@pytest.mark.parametrize("n", [1, 31, 129, 1000, 4097])
def test_ragged_query_counts(make_ctx, n):
    sc = common.scenario(5000, 0.4, 0.01, seed=3)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], 0.01)
    X = queries(sc["P"], 0.01, np.random.RandomState(n), n, 0, 0)[:n]
    for r in (0.01 ** 2, np.inf):
        index, sq = ctx.nearest(X, r)
        pi, ps = ona.bruteforce(sc["P"], X, r)
        assert np.array_equal(index, pi) and np.array_equal(common.bits(sq), common.bits(ps))
    assert [len(a) for a in ctx.nearest(np.zeros((0, 3), np.float32))] == [0, 0]


@pytest.mark.parametrize("n,delta", [(3000, 0.02), (20000, 0.01), (20000, 0.0004)])   # the last: widened cells
def test_equals_verify_nearest_at_delta(make_ctx, n, delta):
    """sq_radius = delta^2, T, the sampled Q as queries: s4g_verify_nearest's answer bit for bit, s4g_verify's count"""
    sc = common.scenario(n, 0.4, delta, seed=5)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], delta)
    ctx.set_cloud_q(sc["Q"])
    T16 = common.candidates_colmajor(sc, 8, seed=9, n_near=4)
    vi, vs, vc = ctx.verify_nearest(T16)
    counts = ctx.verify(T16)
    sq_eps = float(np.float32(delta) * np.float32(delta))
    for k in range(len(T16)):
        index, sq = ctx.nearest(sc["Q"], sq_eps, T16[k])
        assert np.array_equal(index, vi[k]) and np.array_equal(common.bits(sq), common.bits(vs[k]))
        assert (index >= 0).sum() == counts[k] == vc[k]
    assert counts[:4].min() > 0


def test_far_queries_unbounded(make_ctx):
    """queries 1e3 cell widths outside the grid, unbounded radius: the brute force's nearest point"""
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
    index, sq = ctx.nearest(X)
    pi, ps = ona.bruteforce(sc["P"], X)
    assert (index >= 0).all()
    assert np.array_equal(index, pi) and np.array_equal(common.bits(sq), common.bits(ps))


@pytest.mark.parametrize("exclude_self", [False, True])
def test_full_size_sample(make_ctx, exclude_self):
    """1M x 1M (cfg2, delta = 0.003): 20K queries -- sampled-P points (self-excluded or not) at MeanDistance's radius, and
    T q unbounded under a near-ground-truth and a wrong transform -- against the brute force"""
    n, delta = 1_000_000, 0.003
    sc = common.scenario(n, 0.3, delta, seed=42)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], delta)
    sub = np.random.RandomState(0).choice(n, 20000, replace=False)
    X = sc["P"][sub]
    ex = sub.astype(np.int32) if exclude_self else None
    r = float(np.float32(np.abs(sc["P"].max(0) - sc["P"].min(0)).max()) * np.float32(0.2))
    index, sq = ctx.nearest(X, r, None, ex)
    pi, ps = ona.bruteforce(sc["P"], X, r, None, ex)
    assert np.array_equal(index, pi) and np.array_equal(common.bits(sq), common.bits(ps))
    if exclude_self:
        assert (index != sub).all() and (sq > 0).mean() > 0.5
    else:
        assert np.array_equal(index, sub) or (sq == 0).all()
    T16 = common.candidates_colmajor(sc, 2, seed=7, n_near=1)
    for T in T16:
        index, sq = ctx.nearest(sc["Q"][sub], np.inf, T, ex)
        pi, ps = ona.bruteforce(sc["P"], sc["Q"][sub], np.inf, T, ex)
        assert np.array_equal(index, pi) and np.array_equal(common.bits(sq), common.bits(ps))


def test_dev_form_equals_host_form(make_ctx):
    import torch
    sc = common.scenario(20000, 0.4, 0.01, seed=5)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], 0.01)
    X = queries(sc["P"], 0.01, np.random.RandomState(1), 3000)
    T16 = common.candidates_colmajor(sc, 1, n_near=1)[0]
    ex = np.random.RandomState(2).randint(-1, len(sc["P"]), len(X)).astype(np.int32)
    n = len(X)
    dX, dT, dE = torch.from_numpy(X).cuda(), torch.from_numpy(T16.copy()).cuda(), torch.from_numpy(ex).cuda()
    for r in (0.01 ** 2, np.inf):
        for T, dTp in ((None, None), (T16, dT.data_ptr())):
            for e, dEp in ((None, None), (ex, dE.data_ptr())):
                index, sq = ctx.nearest(X, r, T, e)
                d_index = torch.full((n,), 7, dtype=torch.int32, device="cuda")
                d_sq = torch.zeros(n, dtype=torch.float32, device="cuda")
                torch.cuda.synchronize()
                ctx.nearest_dev(dX.data_ptr(), n, d_index.data_ptr(), d_sq.data_ptr(), r, dTp, dEp)
                ctx.synchronize()
                assert np.array_equal(d_index.cpu().numpy(), index)
                assert np.array_equal(common.bits(d_sq.cpu().numpy()), common.bits(sq))
    d_index = torch.full((n,), 7, dtype=torch.int32, device="cuda")
    ctx.nearest_dev(dX.data_ptr(), n, d_index.data_ptr(), None)   # sq_dist is optional
    ctx.synchronize()
    assert np.array_equal(d_index.cpu().numpy(), ctx.nearest(X)[0])


def test_error_codes(s4g_lib):
    from super4pcs_b200 import Context
    with Context(0) as ctx:
        L, h = ctx._L, ctx.h
        X = np.zeros((4, 3), np.float32)
        idx = np.empty(4, np.int32)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        assert L.s4g_nearest(h, p(X), 4, None, 1.0, None, p(idx), None) == S4G_ERR_STATE   # before s4g_set_cloud_p
        assert L.s4g_nearest_dev(h, p(X), 0, None, 1.0, None, p(idx), None) == S4G_ERR_STATE
        ctx.set_cloud_p(np.random.RandomState(0).rand(100, 3).astype(np.float32), 0.05)
        assert L.s4g_nearest(h, p(X), -1, None, 1.0, None, p(idx), None) == S4G_ERR_ARG
        assert L.s4g_nearest(h, None, 4, None, 1.0, None, p(idx), None) == S4G_ERR_ARG
        assert L.s4g_nearest(h, p(X), 4, None, 1.0, None, None, None) == S4G_ERR_ARG
        assert L.s4g_nearest(h, p(X), 4, None, float("nan"), None, p(idx), None) == S4G_ERR_ARG
        assert L.s4g_nearest_dev(h, None, 4, None, 1.0, None, None, None) == S4G_ERR_ARG
        assert L.s4g_nearest(h, None, 0, None, 1.0, None, None, None) == S4G_OK           # n == 0: no-op
        assert L.s4g_nearest_dev(h, None, 0, None, float("inf"), None, None, None) == S4G_OK
        assert L.s4g_nearest(None, p(X), 4, None, 1.0, None, p(idx), None) == S4G_ERR_ARG
        assert L.s4g_nearest(h, p(X), 4, None, float("inf"), None, p(idx), None) == S4G_OK
        assert (idx >= 0).all()


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = nearest_any.build(tmp_path_factory.mktemp("nearest_any"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


def check_program(r):
    sP, sQ = r["sP"], r["sQ"]
    self_ = np.arange(len(sP), dtype=np.int32)
    pi, _ = ona.bruteforce(sP, sP, np.float32(r["diameter"]) * np.float32(0.2), None, self_)
    assert common.bits(r["mean_distance"]) == common.bits(ona.mean_distance(sP, pi))
    for k, dist in enumerate(r["max_distance"]):
        qi, qs = ona.bruteforce(sP, sQ, np.float32(dist) * np.float32(dist), r["C"])
        assert np.array_equal(r["nearest"][k], qi) and np.array_equal(common.bits(r["sq"][k]), common.bits(qs))
    assert np.array_equal(r["nearest"][0], r["nearest_delta"])
    assert np.array_equal(common.bits(r["sq"][0]), common.bits(r["sq_delta"]))


@pytest.mark.parametrize("which", ["hippo", "synthetic"])
def test_cpp_mean_distance_equals_reference(program, tmp_path, which):
    """MeanDistance() of the C++ layer on the real library = the reference's P_mean_distance_ (its init, the same
    options), and the getCorrespondences overload = the brute force"""
    if which == "hippo":
        h = np.load(os.path.join(ROOT, "tests", "golden", "hippo.npz"))
        P, Q, overlap, n = h["P"], h["Q"], 0.7, 200
    else:
        d = common.scenario(30000, 0.5, 0.01, seed=12)["raw"]
        P, Q, overlap, n = d["P"], d["Q"], 0.5, 1000
    r = nearest_any.run(program, tmp_path, P, Q, 0.01, overlap, n)
    assert r["threw_before"] == 1
    check_program(r)
    if ona.ref_available():
        m = ona.RefNearestAny(P, Q, 0.01, overlap=overlap, sample_size=n)
        diameter, want = m.diameter_and_mean_distance()
        assert common.bits(r["diameter"]) == common.bits(np.float32(diameter))
        assert common.bits(r["mean_distance"]) == common.bits(np.float32(want))
