"""Verify and the pair query where their decisions flip (tests/edges.py builds the cases, its fp32 oracle decides them).

Every shortcut in front of Verify's fp32 point test -- tile cull, delta-field, 2x2x2 probe block -- has a margin, and
random clouds almost never put a decision near one.  Here every (query, candidate) pair is built to sit within ulps of
fl(delta^2), or on a voxel / sub-voxel / cell / brick / coarse-block / outer face, in each grid layout, and most counts
are a single decision (one query, one target per candidate), compared one to one with the oracle and the port.
"""
import functools

import numpy as np
import pytest

from oracle import port as oport
from tests import edges as E

pytestmark = pytest.mark.gpu

f32 = np.float32


@pytest.fixture
def context(s4g_lib, monkeypatch):
    from super4pcs_b200 import Context

    def make(cshift_min=None, patches=None):
        for var, val in (("S4G_CSHIFT_MIN", cshift_min), ("S4G_VERIFY_PATCHES", patches)):
            if val is None:
                monkeypatch.delenv(var, raising=False)
            else:
                monkeypatch.setenv(var, str(val))
        return Context(0)
    return make


@functools.lru_cache(maxsize=None)
def cloud(name, cshift_min=1):
    return E.regime_cloud(name, cshift_min=cshift_min)


def check_grid(ctx, g):
    """the host's grid (tests/edges.py) is the one s4g_set_cloud_p built"""
    gs = ctx.grid_stats()
    assert gs["cell_edge"] == float(f32(g["h"]))
    assert gs["brick_edge"] == 1 << g["bshift"]
    assert gs["cells"] == g["cells"]
    return gs


def one_query_candidates(targets, path, g, rng):
    """(Q, T34): one query q and one candidate [R | m3] per target with fl(R q + m3) = the target.  fast: q = 0, so the
    translation column is the target.  robust: the same, plus a far query that makes every candidate's rounding bound
    E exceed vslack (that query maps far outside the cloud)."""
    R = E.rotations(len(targets), rng)
    T34 = np.concatenate([R, np.asarray(targets, f32)[:, :, None]], 2)
    Q = np.zeros((1, 3), f32)
    if path == "robust":
        far = 1024.0
        while 2.0 ** -20 * far <= 4 * float(g["vslack"]):
            far *= 2
        Q = np.array([[0, 0, 0], [far, far, far]], f32)
    return Q, T34


def expected_counts(P, Q, T34, delta):
    t = E.fp32_tq_all(T34, Q)                                  # (K, N, 3)
    return E.fp32_inlier(P, t.reshape(-1, 3), delta).reshape(len(T34), len(Q)).sum(1)


@pytest.mark.parametrize("path", ["fast", "robust"])
@pytest.mark.parametrize("name,cshift_min", [("centred", 1), ("centred", 3), ("brick8", 1), ("widened", 1),
                                             ("offcentre1e3", 1), ("offcentre1e4", 1)])
def test_one_query_one_decision_per_candidate(context, name, cshift_min, path):
    delta = E.REGIMES[name][0]
    P, cases, g = cloud(name, cshift_min)
    ulps, inl = E.coverage(P, cases, delta, lattice_only=name.startswith("offcentre"))
    Q, T34 = one_query_candidates([c["t"] for c in cases], path, g, np.random.RandomState(len(cases)))
    # every candidate takes the path it is meant to test
    qabs = np.abs(Q).max(0)
    for M in T34:
        _, Eb, s, fast = E.verify_record(M, g, qabs)
        assert fast == (path == "fast"), (Eb, s, g["vslack"])
    T16 = E.colmajor(T34)
    with context(cshift_min if cshift_min > 1 else None) as ctx:
        ctx.set_cloud_p(P, delta)
        check_grid(ctx, g)
        ctx.set_cloud_q(Q)
        counts = ctx.verify(T16)
    want = expected_counts(P, Q, T34, delta)
    assert np.array_equal(E.fp32_tq_all(T34, Q)[:, 0], np.array([c["t"] for c in cases]))
    assert np.array_equal(want, inl.astype(np.int64))          # the far query of the robust path is never an inlier
    _, good, _ = oport.Port(P, Q, delta).verify_batch(T16, 0.0, nthreads=oport.num_threads())
    assert np.array_equal(good, want)
    bad = np.nonzero(counts != want)[0]
    assert len(bad) == 0, [(cases[i]["kind"], cases[i]["k"], int(ulps[i]), int(counts[i]), int(want[i])) for i in bad[:10]]


@pytest.mark.parametrize("shape", ["planar", "single", "duplicates"])
def test_degenerate_clouds(context, shape):
    delta = 0.01
    rng = np.random.RandomState(7)
    if shape == "single":
        P = np.array([[0.1, -0.2, 0.05]], f32)
    else:
        P = rng.uniform(-0.3, 0.3, (40, 3)).astype(f32)
        P = P[np.argsort(P[:, 0])]
        P = P[np.r_[True, np.diff(P[:, 0]) > 8 * delta]]
        if shape == "planar":
            P[:, 2] = f32(0.125)
        else:
            P = np.concatenate([P, P[::2]])
    targets = []
    for p in P[:12]:
        for u in E.directions(rng, n_random=1):
            targets += [t for k, t in E.walk_targets(p, u, delta).items()]
    Q, T34 = one_query_candidates(targets, "fast", None, rng)
    T16 = E.colmajor(T34)
    with context() as ctx:
        ctx.set_cloud_p(P, delta)
        check_grid(ctx, E.grid_layout(P, delta))
        ctx.set_cloud_q(Q)
        counts = ctx.verify(T16)
    want = expected_counts(P, Q, T34, delta)
    assert 0 < want.sum() < len(want)
    assert np.array_equal(counts, want)
    _, good, _ = oport.Port(P, Q, delta).verify_batch(T16, 0.0, nthreads=oport.num_threads())
    assert np.array_equal(good, want)


@pytest.mark.parametrize("name", ["centred", "brick8", "offcentre1e4"])
def test_pairs_in_the_field_margin_reach_the_exact_test(context, name):
    """a pair whose distance is within md + slack of delta can be decided by neither delta-field level: it must reach
    the exact test (points read); and some pairs just outside that band are decided by the field (it is active here)"""
    delta = E.REGIMES[name][0]
    P, cases, g = cloud(name)
    band = g["md"] + g["slack"]
    rng = np.random.RandomState(11)
    targets, inside = [], []
    anchors = P[8:]
    for p in anchors[rng.choice(len(anchors), 6, replace=False)]:
        for u in E.directions(rng, n_random=1)[::2]:
            for s in (0.0, 0.5, 0.99, -0.5, -0.99):
                targets.append((p + (delta + s * band) * u).astype(f32))
                inside.append(True)
            for j in (1, 2, 4, 6):
                for sg in (1, -1):
                    s = delta + sg * (band + j * g["v"] / 8)
                    if s > 0:
                        targets.append((p + s * u).astype(f32))
                        inside.append(False)
    t = np.array(targets, f32)
    _, dist = E.margin_ulps(P, t, delta)
    inside = np.abs(dist - float(f32(delta))) <= band
    Q, T34 = one_query_candidates(t, "fast", g, rng)
    want = expected_counts(P, Q, T34, delta)
    T16 = E.colmajor(T34)
    reached = np.zeros(len(t), bool)
    with context() as ctx:
        ctx.set_cloud_p(P, delta)
        ctx.set_cloud_q(Q)
        assert np.array_equal(ctx.verify(T16), want)
        for i in range(len(t)):
            st = ctx.verify_probe_stats(T16[i:i + 1])
            reached[i] = st["points_tested"] > 0 or st["ranges_read"] > 0
    # the probe statistics show the exact test only when it reads points: when the P point lies in the 2x2x2 cell block
    # around the target, which holds within half a cell (far from the origin the band is several cells wide)
    seen = inside & (dist < 0.4999 * g["h"])
    assert seen.sum() >= 15
    assert reached[seen].all(), np.nonzero(seen & ~reached)[0]
    if name != "offcentre1e4":      # there the band (slack ~ 0.09) is wider than every target's distance from delta
        assert (~reached[~inside]).any()


@pytest.mark.parametrize("patches", [None, 3])
def test_many_queries_many_candidates(context, patches):
    """all generated targets of the centred regime plus queries jittered around the P points as Q (a tile dense with
    pairs that go to the exact test), candidates the identity and small exact translations: verify and verify_best"""
    delta = E.REGIMES["centred"][0]
    P, cases, g = cloud("centred")
    rng = np.random.RandomState(5)
    t = np.array([c["t"] for c in cases], f32)
    jit = (P[rng.randint(0, len(P), 3000)] + rng.standard_normal((3000, 3)) * delta * 0.6).astype(f32)
    Q = np.concatenate([t, jit])
    K = 40
    T34 = np.zeros((K, 3, 4), f32)
    T34[:, :, :3] = np.eye(3, dtype=f32)
    T34[1:, :, 3] = (rng.randint(-64, 65, (K - 1, 3)) * 2.0 ** -24).astype(f32)
    T16 = E.colmajor(T34)
    want = expected_counts(P, Q, T34, delta)
    with context(patches=patches) as ctx:
        ctx.set_cloud_p(P, delta)
        ctx.set_cloud_q(Q)
        counts = ctx.verify(T16)
        st = ctx.verify_probe_stats(T16)
        c2, key = ctx.verify_best(T16)
    _, good, _ = oport.Port(P, Q, delta).verify_batch(T16, 0.0, nthreads=oport.num_threads())
    assert np.array_equal(good, want)
    assert np.array_equal(counts, want) and np.array_equal(c2, want)
    best = int(np.argmax(want))
    assert key == (int(want[best]) << 32) | (0xFFFFFFFF - best)
    assert st["points_tested"] > len(Q)                        # the exact test ran for many pairs (queues flushed)


def test_offcentre_coarse_face_cull_keeps_inliers(context):
    """Regression: a cloud at 1.2e4 with P points on coarse-block faces and queries delta across them.  With the tile
    cull's fixed 0.52-cell pad some of these exact inliers were culled (the centre's FMA chain rounds at ~3e6 voxels);
    the pad now carries vslack / h."""
    delta = E.REGIMES["offcentre1e4"][0]
    P, q, T34, g = E.coarse_face_cull_cases()
    culled_before = 0
    for M in T34:
        V, _, s, _ = E.verify_record(M, g, np.abs(q))
        culled_before += not E.tile_live(g, V, q, f32(1e-7), s, pad=f32(0.52))
    assert culled_before > 0
    T16 = E.colmajor(T34)
    with context() as ctx:
        ctx.set_cloud_p(P, delta)
        check_grid(ctx, g)
        ctx.set_cloud_q(q[None])
        counts = ctx.verify(T16)
    want = expected_counts(P, q[None], T34, delta)
    assert (want == 1).all()
    _, good, _ = oport.Port(P, q[None], delta).verify_batch(T16, 0.0, nthreads=oport.num_threads())
    assert np.array_equal(good, want)
    assert np.array_equal(counts, want), int((counts != want).sum())


@pytest.mark.parametrize("unit_binding", [False, True])
def test_pair_band_edges_all_modes(context, unit_binding):
    """pairs at d -+ eps exactly, +-1 and +-2 floats around, fl(sq) around the squared pre-filter bounds, d - eps <= 0,
    and the unit-cube test's own edge: every k_pairs mode against the fp32 emulation and the port, pair by pair"""
    Q, queries, kinds = E.pair_cloud(unit_binding)
    pt = oport.Port(Q[:1], Q, 0.01)
    with context() as ctx:
        ctx.set_cloud_p(Q, 0.01)
        ctx.set_cloud_q(Q)
        for d, eps in queries:
            want = E.pair_set(Q, d, eps)
            assert np.array_equal(pt.extract_pairs(d, 0.0, eps), want)
            got = ctx.extract_pairs(d, 0.0, eps)                                    # mode 1
            assert np.array_equal(got, want), (d, eps, len(got), len(want))
            assert ctx.count_pairs(d, eps) == len(want)                             # mode 0
            total, rows = ctx.count_pairs_rows(d, eps)                              # mode 2
            assert total == len(want)
            assert np.array_equal(rows, np.bincount(want[:, 0], minlength=len(Q)))
            b9 = np.tile(np.array([0, 0, 0, 0, 0, 0, -1, -1, -1], f32), (4, 1))
            base = dict(d1=d, d2=d, b9=b9, bxp=Q[:4], inv1=0.5, inv2=0.5)
            got3 = ctx.try_bases([base], eps, eps, eps)                             # mode 3
            assert got3[0]["n_pairs"] == [len(want), len(want)]
