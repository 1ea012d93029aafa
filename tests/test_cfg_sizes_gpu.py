"""GPU parity at the sizes BASELINE.json names for cfg3 and cfg4 (VERDICT round 1, item 1c):

  cfg3  200K-point pair + Gaussian noise (sigma 0.005) + 20 % outliers, normals on (30 deg), |sampled_Q| = 3000 / 10000:
        pairs (both slots, normal filter), quads and TryCongruentSet of one base against the oracle port, bit-exact;
  cfg4  10M-point cloud, counting-only shell query at eps = 2e-4 (SURVEY.md 8(d)): the list cannot be materialised
        (2.6e10 pairs), so the per-point rows of the query (s4g_count_pairs_rows) are checked against brute force on
        sampled rows (the reference's own criterion, tests/pair_extraction.cc:172-194), and their sum against the total.
"""
import numpy as np
import pytest

import bench
from oracle import port as oport
from super4pcs_b200 import synth

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cfg3():
    d = synth.make_pair(200_000, 0.4, seed=43, noise_sigma=0.005, outlier_frac=0.2, with_normals=True)
    P, _ = synth.center(d["P"])
    Q, _ = synth.center(d["Q"])
    return d, P, Q


@pytest.mark.parametrize("ns,patches", [pytest.param(3000, None, id="3000"), pytest.param(10000, None, id="10000"),
                                        pytest.param(10000, 10, id="10000-patches10")])   # one super-tile per Verify patch
def test_cfg3_base_matches_oracle(s4g_lib, monkeypatch, cfg3, ns, patches):
    from super4pcs_b200 import Context, PairFilters
    if patches is not None:
        monkeypatch.setenv("S4G_VERIFY_PATCHES", str(patches))
    d, P, Q = cfg3
    delta = 0.01
    rng = np.random.RandomState(ns)
    sel = rng.choice(len(Q), ns, replace=False)
    Qs = np.ascontiguousarray(Q[sel])
    Qn = (d["Qn"][sel] / np.linalg.norm(d["Qn"][sel], axis=1, keepdims=True)).astype(np.float32)
    sub = rng.choice(len(P), 20000, replace=False)
    diameter = float(np.linalg.norm(P[sub].max(0) - P[sub].min(0)))
    filt = (30.0, -1.0, -1.0, -1.0)
    pt = oport.Port(P, Qs, delta, Qn=Qn)
    with Context(0) as ctx:
        ctx.set_cloud_p(P, delta)
        ctx.set_cloud_q(Qs, normals=Qn)
        tested = 0
        for _ in range(12):                                   # a few bases until one has congruent quads
            ids, inv1, inv2 = bench.select_base(P[sub], rng, diameter)
            pid = sub[ids]
            bx = P[pid]
            bn = (d["Pn"][pid] / np.linalg.norm(d["Pn"][pid], axis=1, keepdims=True)).astype(np.float32)
            b9 = [np.concatenate([bx[i], bn[i], [-1, -1, -1]]).astype(np.float32) for i in range(4)]
            d1, d2 = bench._eigen_norm(bx[0] - bx[1]), bench._eigen_norm(bx[2] - bx[3])
            na1, na2 = bench._eigen_norm(bn[0] - bn[1]), bench._eigen_norm(bn[2] - bn[3])
            got1 = ctx.extract_pairs(d1, na1, 2 * delta, b9[0], b9[1], PairFilters(*filt), slot=0)
            got2 = ctx.extract_pairs(d2, na2, 2 * delta, b9[2], b9[3], PairFilters(*filt), slot=1)
            want1 = pt.extract_pairs(d1, na1, 2 * delta, b9[0], b9[1], filt)
            want2 = pt.extract_pairs(d2, na2, 2 * delta, b9[2], b9[3], filt)
            assert np.array_equal(got1, want1) and np.array_equal(got2, want2)      # ordered pair sets, bit-exact
            assert len(want1) > 0 and len(want2) > 0
            quads = ctx.find_quads(inv1, inv2, 2 * delta, bx)
            wantq = pt.find_quads(inv1, inv2, 2 * delta, bx, want1, want2)
            assert np.array_equal(quads, wantq)                                      # same quads, same order
            if len(wantq) == 0:
                continue
            r = ctx.try_congruent_set_resident(bx, 2 * delta)
            w = pt.try_congruent_set(pid.astype(np.int32), wantq, best_lcp_in=0.0)
            assert r["n_gate_pass"] == w["n_gate"] and r["best_index"] == w["best_index"]
            if w["best_index"] >= 0:
                assert np.float32(r["best_count"]) / np.float32(r["n_q"]) == np.float32(w["best_lcp"])
                assert np.array_equal(r["T"].view(np.uint32), w["T"].view(np.uint32))
                tested += 1
            if tested >= 2:
                break
        assert tested >= 1


def test_cfg4_counting_query_rows(s4g_lib):
    from super4pcs_b200 import Context
    n, dist, eps = 10_000_000, 1.0, 2e-4
    d = synth.make_pair(n, 0.2, seed=44)
    Q, _ = synth.center(d["Q"])
    del d
    with Context(0) as ctx:
        ctx.set_cloud_q(Q)
        total = ctx.count_pairs(dist, eps)
        total2, rows = ctx.count_pairs_rows(dist, eps)
    assert total == total2 == int(rows.sum(dtype=np.int64)) and total > 10 ** 9
    # sampled rows against brute force in the reference's arithmetic: float distance in Eigen's order, double compare
    for a in np.random.RandomState(4).choice(n, 12, replace=False):
        df = (Q - Q[a]).astype(np.float32)
        dd = np.sqrt(df[:, 0] * df[:, 0] + (df[:, 1] * df[:, 1] + df[:, 2] * df[:, 2]))
        want = np.count_nonzero(np.abs(dd.astype(np.float64) - np.float64(np.float32(dist))) <= np.float64(np.float32(eps)))
        want -= int(abs(0.0 - float(np.float32(dist))) <= float(np.float32(eps)))      # the point itself (distance 0)
        assert int(rows[a]) == want
