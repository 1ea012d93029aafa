"""s4g_find_quads and s4g_try_bases where the quad search's decisions flip, against the restatement of tests/quads.py: on
uploaded lists (in the fixture's order and permuted), on extracted lists, and through the batched chain, whose quad
counts and winners must equal the per-base chain's.  Then the batched chain's limits: an extraction of 2^25 .. 2^26 pairs
is accepted and equals the per-base chain, one of 2^26 pairs or more is refused with S4G_ERR_ARG, and a batch of more
than 2^32 quads with S4G_ERR_NOMEM."""
import numpy as np
import pytest

from tests import quads as T

pytestmark = pytest.mark.gpu
ERR_ARG, ERR_NOMEM = 2, 4                                   # S4G_ERR_ARG, S4G_ERR_NOMEM


@pytest.fixture(scope="module")
def ctx(s4g_lib):
    from super4pcs_b200 import Context
    c = Context(0)
    yield c
    c.close()


def _set_cloud(ctx, Q):
    key = Q.tobytes()
    if getattr(ctx, "_qe_cloud", None) != key:
        ctx.set_cloud_p(Q, 0.01)
        ctx.set_cloud_q(Q)
        ctx._qe_cloud = key
        gc, ratio = ctx.q_normalization()
        wgc, wratio = T.normalization(Q)
        assert np.array_equal(gc, wgc) and np.float32(ratio) == wratio


def _supported(fx):
    return 0 <= T.grid(fx["thr2"], T.normalization(fx["Q"])[1])[0] <= 18


def _quads(ctx, fx, p1, p2):
    ctx.set_pairs(0, p1)
    ctx.set_pairs(1, p2)
    return ctx.find_quads(fx["inv1"], fx["inv2"], fx["thr2"], fx["base"])


def _want(fx, p1, p2):
    gc, ratio = T.normalization(fx["Q"])
    return T.find_quads(fx["Q"], gc, ratio, p1, p2, fx["inv1"], fx["inv2"], fx["thr2"], fx["base"])


@pytest.mark.parametrize("family", list(T.FAMILIES))
def test_uploaded_lists_equal_the_restatement(ctx, family):
    from super4pcs_b200 import S4GError
    rng = np.random.RandomState(1)
    bad = []
    for fx in T.fixtures(family):
        _set_cloud(ctx, fx["Q"])
        if not _supported(fx):
            with pytest.raises(S4GError):
                _quads(ctx, fx, fx["pairs1"], fx["pairs2"])
            continue
        for p1, p2 in ((fx["pairs1"], fx["pairs2"]),
                       (fx["pairs1"][rng.permutation(len(fx["pairs1"]))], fx["pairs2"][rng.permutation(len(fx["pairs2"]))])):
            got, want = _quads(ctx, fx, p1, p2), _want(fx, p1, p2)
            if not np.array_equal(got, want):
                bad.append((fx["name"], len(got), len(want)))
    assert not bad, bad


def _all_pairs(Q):
    """d = 0 and eps = 2.5 ratio: every ordered pair passes the pair query"""
    return 0.0, float(2.5 * T.normalization(Q)[1])


@pytest.mark.parametrize("family", list(T.FAMILIES))
def test_extracted_lists_equal_the_restatement(ctx, family):
    bad = []
    for fx in T.fixtures(family):
        if not _supported(fx):
            continue
        _set_cloud(ctx, fx["Q"])
        d, eps = _all_pairs(fx["Q"])
        n = len(fx["Q"])
        ctx.extract_pairs(d, 0.0, eps, slot=0, fetch=False)
        p = ctx.extract_pairs(d, 0.0, eps, slot=1)
        assert len(p) == n * (n - 1)
        got, want = ctx.find_quads(fx["inv1"], fx["inv2"], fx["thr2"], fx["base"]), _want(fx, p, p)
        if not np.array_equal(got, want):
            bad.append((fx["name"], len(got), len(want)))
    assert not bad, bad


def _batches():
    """fixtures that share a cloud and thr2, 64 at most per batch"""
    groups = {}
    for fx in T.all_fixtures():
        if _supported(fx):
            groups.setdefault((fx["Q"].tobytes(), float(fx["thr2"])), []).append(fx)
    for fxs in groups.values():
        for s in range(0, len(fxs), 64):
            yield fxs[s:s + 64]


def test_try_bases_equals_the_per_base_chain(ctx):
    """every fixture as one base (every ordered pair in both extractions): n_quads and the winner's key, index and
    transform bits equal the per-base chain's; grid depths beyond 14 are refused with S4G_ERR_ARG"""
    from super4pcs_b200 import S4GError
    n_batches = n_multi = 0
    for fxs in _batches():
        Q = fxs[0]["Q"]
        _set_cloud(ctx, Q)
        d, eps = _all_pairs(Q)
        thr2 = float(fxs[0]["thr2"])
        bases = [dict(d1=d, d2=d, na1=0.0, na2=0.0, inv1=float(fx["inv1"]), inv2=float(fx["inv2"]), bxp=fx["base"],
                      b9=np.concatenate([fx["base"], np.zeros((4, 3), np.float32), -np.ones((4, 3), np.float32)], 1))
                 for fx in fxs]
        if T.grid(thr2, T.normalization(Q)[1])[0] > 14:
            with pytest.raises(S4GError, match="too small for the batched"):
                ctx.try_bases(bases, eps, thr2, eps)
            continue
        got = ctx.try_bases(bases, eps, thr2, eps)
        n_batches += 1
        n_multi += len(bases) > 1
        for fx, b, g in zip(fxs, bases, got):
            n1 = ctx.extract_pairs(d, 0.0, eps, slot=0, fetch=False)
            n2 = ctx.extract_pairs(d, 0.0, eps, slot=1, fetch=False)
            assert g["n_pairs"] == [n1, n2]
            nq = ctx.find_quads(b["inv1"], b["inv2"], thr2, fx["base"], fetch=False)
            assert g["n_quads"] == nq, fx["name"]
            if nq == 0:
                assert g["tcs"]["best_index"] == -1, fx["name"]
                continue
            w = ctx.try_congruent_set_resident(b["bxp"], eps)
            t = g["tcs"]
            for k in ("key", "best_count", "best_index", "n_gate_pass"):
                assert t[k] == w[k], (fx["name"], k)
            assert np.array_equal(t["T"].view(np.uint32), w["T"].view(np.uint32)), fx["name"]
    assert n_batches > 10 and n_multi > 3


# ---- the batched chain's limits ----------------------------------------------------------------------------------------
def _ball(n, seed=0, radius=0.05):
    rng = np.random.RandomState(seed)
    u = rng.standard_normal((n, 3))
    u *= radius * rng.uniform(0, 1, (n, 1)) ** (1 / 3) / np.linalg.norm(u, axis=1, keepdims=True)
    return u.astype(np.float32)


def _desc(base, d1, d2, inv=0.5):
    base = np.asarray(base, np.float32)
    return dict(d1=d1, d2=d2, na1=0.0, na2=0.0, inv1=inv, inv2=inv, bxp=base,
                b9=np.concatenate([base, np.zeros((4, 3), np.float32), -np.ones((4, 3), np.float32)], 1))


def test_an_extraction_of_2_25_to_2_26_pairs_equals_the_per_base_chain(s4g_lib):
    """7000 points in a ball of radius 0.05 (48,993,000 ordered pairs in slot 0, P-pair indices up to 2^25.5) and a
    Q-pair of length 10 through its centre; the quads' ids span the whole list"""
    from super4pcs_b200 import Context
    Q = np.concatenate([_ball(7000), np.array([[-5, 0.001, 0.002], [5, -0.001, 0.0]], np.float32)]).astype(np.float32)
    base = np.array([[0, 0, 0], [0.08, 0, 0], [0, 0, 0], [0.08 * np.cos(0.4), 0.08 * np.sin(0.4), 0]], np.float32)
    eps = 1.0
    ratio = T.normalization(Q)[1]
    thr2 = float(ratio * 0.75 * 2.0 ** -10)                        # grid depth 10
    b = _desc(base, 0.0, 10.0)
    with Context(0) as c:
        c.set_cloud_p(Q, 0.01)
        c.set_cloud_q(Q)
        got = c.try_bases([b], eps, thr2, eps)[0]
        n1 = c.extract_pairs(0.0, 0.0, eps, slot=0, fetch=False)
        n2 = c.extract_pairs(10.0, 0.0, eps, slot=1, fetch=False)
        assert 2 ** 25 < n1 < 2 ** 26 and n2 == 2
        assert got["n_pairs"] == [n1, n2]
        quads = c.find_quads(0.5, 0.5, thr2, base)
        assert got["n_quads"] == len(quads) > 1000
        w = c.try_congruent_set_resident(base, eps)
    a, b2 = quads[:, 0].astype(np.int64), quads[:, 1].astype(np.int64)
    assert (a < 7000).all() and (b2 < 7000).all()
    ids = a * 6999 + b2 - (b2 > a)                                  # index in the sorted list of the ball's pairs
    assert ids.max() > 2 ** 25                                      # matching P-pairs beyond index 2^25
    for k in ("key", "best_count", "best_index", "n_gate_pass"):
        assert got["tcs"][k] == w[k], k
    assert np.array_equal(got["tcs"]["T"].view(np.uint32), w["T"].view(np.uint32))


def test_an_extraction_of_2_26_pairs_is_refused(s4g_lib):
    """8200 points in a ball: 67,231,800 ordered pairs >= 2^26 in slot 0 -> S4G_ERR_ARG (the per-base chain takes it)"""
    from super4pcs_b200 import Context, S4GError
    Q = _ball(8200, seed=1)
    base = np.array([[0, 0, 0], [0.08, 0, 0], [0, 0, 0], [0, 0.08, 0]], np.float32)
    with Context(0) as c:
        c.set_cloud_p(Q, 0.01)
        c.set_cloud_q(Q)
        with pytest.raises(S4GError, match="error %d: .*2\\^26 or more pairs" % ERR_ARG):
            c.try_bases([_desc(base, 0.0, 5.0)], 1.0, 0.5 * T.normalization(Q)[1], 1.0)
        assert c.count_pairs(0.0, 1.0) == 8200 * 8199 >= 2 ** 26


@pytest.fixture(scope="module")
def built(s4g_lib):
    from oracle import _build
    from super4pcs_b200 import build_cpp
    if build_cpp.build_all()["lib"] is None or _build.build_dropin_harness() is None:
        pytest.skip("C++ layer not available")


def test_the_cpp_layer_falls_back_to_the_per_base_chain_beyond_2_26_pairs(built):
    """ComputeTransformation on a line of 8200 points against a 4-point P whose bases have one diagonal of 0.5 (with
    delta 0.25 its band holds all 67,231,800 ordered pairs) and one of 1.5 (none): with batches of 8 allowed up to
    100000 sampled Q points, s4g_try_bases refuses every batch (S4G_ERR_ARG) and the result is the per-base chain's"""
    from tests.test_host_logic_cpu import run_driver
    per_base = run_driver("bigpairs", "dropin", extra_env={"S4PCS_BATCH": "1"}, timeout=600)
    batched = run_driver("bigpairs", "dropin", extra_env={"S4PCS_BATCH": "8", "S4PCS_BATCH_MAX_Q": "100000"}, timeout=600)
    assert batched == per_base


def test_a_batch_of_more_than_2_32_quads_is_refused(s4g_lib):
    """310 collinear points 0.01 long, every ordered pair in both extractions, base segments 3 degrees apart and
    thr2 / ratio = 0.75 (grid depth 0): each Q-pair matches the 47,895 P-pairs of its orientation, 4.59e9 quads in all.
    Only the counting passes run.  Each (the batched one, then the per-base one) has 95,790 threads, each walking the
    95,790 entries of the one cell: 9.2e9 key loads, broadcast within a warp, and 4.6e9 distance tests, of the order of
    10-100 ms on an H100 (the keys fit in L2); estimated from the code, not measured."""
    from super4pcs_b200 import Context, S4GError
    n = 310
    Q = np.zeros((n, 3), np.float32)
    Q[:, 0] = np.linspace(-0.005, 0.005, n, dtype=np.float32)
    ratio = T.normalization(Q)[1]
    thr2 = float(np.float32(0.75) * ratio)
    a = np.deg2rad(3.0)
    base = np.array([[0, 0, 0], [1, 0, 0], [0, 0, 0], [np.cos(a), np.sin(a), 0]], np.float32)
    pairs = n * (n - 1)
    with Context(0) as c:
        c.set_cloud_p(Q, 0.001)
        c.set_cloud_q(Q)
        with pytest.raises(S4GError, match="error %d: .*2\\^31-1 quads" % ERR_NOMEM):
            c.try_bases([_desc(base, 0.0, 0.0)], 1.0, thr2, 1.0)
        # the per-base chain counts in 64 bits and refuses the same set
        assert c.extract_pairs(0.0, 0.0, 1.0, slot=0, fetch=False) == pairs
        assert c.extract_pairs(0.0, 0.0, 1.0, slot=1, fetch=False) == pairs
        with pytest.raises(S4GError, match="error %d: .*2\\^32-2 quads" % ERR_NOMEM):
            c.find_quads(0.5, 0.5, thr2, base, fetch=False)
