"""The decision-edge construction of tests/edges.py and its fp32 oracle, checked without a GPU: on every generated case
the oracle agrees with the port (grid search and brute force), and the cases reach what the GPU tests rely on -- exact
ties, +-1 and +-2 ulps of fl(delta^2) with both outcomes, every face kind, the pair band's edges."""
import numpy as np
import pytest

from oracle import port as oport
from tests import edges as E


@pytest.mark.parametrize("name", list(E.REGIMES))
def test_oracle_agrees_with_the_port_on_every_edge_case(name):
    delta = E.REGIMES[name][0]
    P, cases, g = E.regime_cloud(name)
    lattice = name.startswith("offcentre")          # coordinates ~1e3 / 1e4: d^2 moves in steps of many ulps
    ulps, inl = E.coverage(P, cases, delta, lattice_only=lattice)
    kinds = {c["kind"] for c in cases}
    assert {"generic", "outer"} | {"p_on_" + k for k in E.FACE_KINDS} | {"t_on_" + k for k in E.FACE_KINDS} <= kinds
    t = np.array([c["t"] for c in cases], np.float32)
    # one query at the origin, one candidate per target: T q = the translation column, exactly
    T34 = np.zeros((len(t), 3, 4), np.float32)
    T34[:, :, :3] = np.eye(3, dtype=np.float32)
    T34[:, :, 3] = t
    assert np.array_equal(E.fp32_tq(T34, np.zeros(3, np.float32)), t)
    pt = oport.Port(P, np.zeros((1, 3), np.float32), delta)
    T16 = E.colmajor(T34)
    _, good, _ = pt.verify_batch(T16, 0.0, nthreads=oport.num_threads())
    assert np.array_equal(good.astype(bool), inl)
    assert np.array_equal(pt.verify_bruteforce(T16).astype(bool), inl)
    # the host grid is the one the GPU tests compare with grid_stats()
    if name == "brick8":
        assert g["bshift"] == 3
    elif name == "widened":
        assert g["widened"] and g["h"] > 2.02 * delta
    else:
        assert g["bshift"] == 2 and not g["widened"]
    if name == "offcentre1e4":
        assert g["slack"] > 0.02 * g["v"] * 100      # the slack comes from the size of the coordinates


def test_fp32_oracle_is_the_reference_order():
    """d^2 = dx^2 + (dy^2 + dz^2) and T q = ((m0 x + m1 y) + m2 z) + m3, not a fused or reassociated form: cases where
    the orders differ in float32"""
    rng = np.random.RandomState(0)
    x = rng.uniform(-1, 1, (20000, 3)).astype(np.float32)
    d2 = E.fp32_d2(x, np.zeros((1, 3), np.float32))[:, 0]
    left = (x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2]
    assert (d2 != left).any()
    assert np.array_equal(d2, x[:, 0] * x[:, 0] + (x[:, 1] * x[:, 1] + x[:, 2] * x[:, 2]))
    T = rng.uniform(-1, 1, (2000, 3, 4)).astype(np.float32)
    q = rng.uniform(-1, 1, 3).astype(np.float32)
    tq = E.fp32_tq(T, q)
    ref = np.einsum("krc,c->kr", T.astype(np.float64), np.append(q, 1).astype(np.float64))
    assert np.abs(tq - ref).max() < 1e-6 and (tq != ref.astype(np.float32)).any()


def test_walk_targets_reach_each_ulp():
    rng = np.random.RandomState(1)
    seen = set()
    for _ in range(4):
        p = rng.uniform(-0.4, 0.4, 3).astype(np.float32)
        for u in E.directions(rng):
            got = E.walk_targets(p, u, 0.01)
            for k in E.KS:
                if k in got:
                    u_, _ = E.margin_ulps(p[None], got[k][None], 0.01)
                    assert u_[0] == k
                    seen.add(k)
            assert E.margin_ulps(p[None], got["in"][None], 0.01)[0][0] <= 0
            assert E.margin_ulps(p[None], got["out"][None], 0.01)[0][0] > 0
    assert seen == set(E.KS)


def test_coarse_face_cases_reach_the_old_cull():
    """the off-centre cull cases: every one is an exact inlier on the fast path, the tile cull with the fixed 0.52-cell
    pad culls some of them (the bug the GPU test keeps fixed), the pad carrying vslack culls none"""
    P, q, T, g = E.coarse_face_cull_cases()
    delta = E.REGIMES["offcentre1e4"][0]
    t = np.array([E.fp32_tq(M, q)[0] for M in T])
    assert E.fp32_inlier(P, t, delta).all()
    old = new = 0
    for M in T:
        V, _, s, fast = E.verify_record(M, g, np.abs(q))
        assert fast
        old += not E.tile_live(g, V, q, np.float32(1e-7), s, pad=np.float32(0.52))
        new += not E.tile_live(g, V, q, np.float32(1e-7), s, pad=E.cull_pad(g))
    assert old > 0 and new == 0


@pytest.mark.parametrize("unit_binding", [False, True])
def test_pair_emulation_agrees_with_the_port(unit_binding):
    Q, queries, kinds = E.pair_cloud(unit_binding)
    pt = oport.Port(Q[:1], Q, 0.01)
    for d, eps in queries:
        want = E.pair_set(Q, d, eps)
        got = pt.extract_pairs(d, 0.0, eps)
        assert np.array_equal(got, want), (d, eps)
    if unit_binding:
        # the exact ties pass the world test and fail the strict unit-cube test
        d, eps = queries[0]
        tie = np.nonzero(kinds == "tie")[0].reshape(-1, 2)
        sep = np.abs(Q[tie[:, 1], 0] - Q[tie[:, 0], 0])
        on_tie = np.isin(sep, np.float32([d - eps, d + eps]))
        assert on_tie.any()
        accepted = {tuple(p) for p in E.pair_set(Q, d, eps).tolist()}
        assert not any((a, b) in accepted for a, b in tie[on_tie].tolist())
        assert len(accepted) > 0
    else:
        # both sides of every tie, and fl(sq) on both sides of the squared pre-filter bounds with the distance in band
        for d, eps in queries:
            lo_sq, hi_sq, lo, hi = E.prefilter_bounds(d, eps)
            pre = np.nonzero(kinds == "prefilter")[0].reshape(-1, 2)
            if lo > 0:
                a, b = Q[pre[:, 0]], Q[pre[:, 1]]
                dq = b - a
                sq = dq[:, 0] * dq[:, 0] + (dq[:, 1] * dq[:, 1] + dq[:, 2] * dq[:, 2])
                near = np.abs(E.ordinal(sq) - E.ordinal(np.float32(lo * lo))) <= 3
                assert near.any()
