"""s4g_verify_nearest on the GPU: the nearest P point within delta of every transformed Q point.

Count invariant: the number of index >= 0 (and `counts`) equals s4g_verify's count for the same T, over the transform
families and grid regimes the Verify tests use (near-GT / random candidates, NaN, huge and non-rigid 4x4, widened cells,
off-centre clouds, queries on the delta-sphere and on the field / cell / brick lattices).  Values: index and sq_dist are
bit-equal to the port's brute force (oracle/port.cc), and to the compiled reference's kd-tree up to its tie order."""
import os

import numpy as np
import pytest

from oracle import nearest as onear
from tests import common, correspondences
from tests import edges as E
from tests.test_decision_edges_gpu import cloud, one_query_candidates
from tests.test_verify_nearest_cpu import check_against_reference

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def ctx(s4g_lib):
    from super4pcs_b200 import Context
    c = Context(0)
    yield c
    c.close()


def nearest_checked(ctx, T16):
    """verify_nearest, with its count invariant against verify"""
    index, sq, counts = ctx.verify_nearest(T16)
    want = ctx.verify(T16)
    assert np.array_equal(counts, want)
    assert np.array_equal((index >= 0).sum(1), want)
    assert (index < ctx.nP).all() and (index >= -1).all()
    assert np.isinf(sq[index < 0]).all() and (sq[index >= 0] <= np.float32(ctx.delta) * np.float32(ctx.delta)).all()
    return index, sq, counts


def equal_to_port(P, Q, delta, T16, index, sq):
    pi, ps, pc = onear.bruteforce(P, Q, delta, T16)
    assert np.array_equal(index, pi)
    assert np.array_equal(common.bits(sq), common.bits(ps))


def transform_families(sc, seed=9):
    """near-GT and random candidates, then scaled / sheared / anisotropic / huge versions of near-GT ones (the robust path),
    far away, NaN and Inf"""
    T = common.candidates_colmajor(sc, 24, seed=seed, n_near=8)
    base = T[:8].reshape(-1, 4, 4).transpose(0, 2, 1).astype(np.float64)
    rng = np.random.RandomState(seed)
    extra = []
    for k, M in enumerate(base):
        A = np.eye(4)
        A[:3, :3] = [np.eye(3) * (1 + 0.2 * rng.random_sample()), np.eye(3) + np.eye(3, k=1) * 0.3,
                     np.diag([1.3, 0.8, 1.1]), np.eye(3) * 1e4][k % 4]
        extra.append((M @ A).astype(np.float32).T.reshape(16))
    far = np.eye(4, dtype=np.float32)
    far[:3, 3] = 1000.0
    extra += [far.T.reshape(16), np.full(16, np.nan, np.float32), np.full(16, np.inf, np.float32)]
    return np.concatenate([T, np.asarray(extra, np.float32)])


@pytest.mark.parametrize("n,delta", [(3000, 0.02), (20000, 0.01), (20000, 0.0004)])   # the last: widened cells
def test_count_invariant_and_port_on_transform_families(ctx, n, delta):
    sc = common.scenario(n, 0.4, delta, seed=5)
    ctx.set_cloud_p(sc["P"], delta)
    ctx.set_cloud_q(sc["Q"])
    if delta < 0.001:
        assert ctx.grid_stats()["cell_edge"] > 2.02 * delta * 1.05
    T16 = transform_families(sc)
    index, sq, counts = nearest_checked(ctx, T16)
    assert counts[:8].max() > 0 and counts[-3:].max() == 0
    sub = np.arange(n) if n <= 3000 else np.random.RandomState(1).choice(n, 2000, replace=False)   # brute force: a sample
    equal_to_port(sc["P"], sc["Q"][sub], delta, T16, index[:, sub], sq[:, sub])
    if onear.ref_available() and n == 3000:
        m = onear.RefNearest(sc["raw"]["P"], sc["raw"]["Q"], delta)
        sP, sQ = m.sampled()
        ctx.set_cloud_p(sP, delta)
        ctx.set_cloud_q(sQ)
        index, sq, _ = nearest_checked(ctx, T16[:24])
        ri, rs = m.query(T16[:24])
        check_against_reference(sP, index, sq, ri, rs, T16[:24], sQ)


@pytest.mark.parametrize("path", ["fast", "robust"])
@pytest.mark.parametrize("name", ["centred", "brick8", "widened", "offcentre1e3", "offcentre1e4"])
def test_decision_edges(s4g_lib, name, path):
    """one query per candidate on the delta-sphere, the voxel / sub-voxel / cell / brick / coarse faces (tests/edges.py)"""
    from super4pcs_b200 import Context
    delta = E.REGIMES[name][0]
    P, cases, g = cloud(name)
    Q, T34 = one_query_candidates([c["t"] for c in cases], path, g, np.random.RandomState(len(cases)))
    T16 = E.colmajor(T34)
    with Context(0) as c:
        c.set_cloud_p(P, delta)
        c.set_cloud_q(Q)
        index, sq, counts = nearest_checked(c, T16)
    assert 0 < counts.sum() < len(T16)
    equal_to_port(P, Q, delta, T16, index, sq)


@pytest.mark.parametrize("nP,nQ", [(1, 1), (2, 2), (129, 129), (1000, 1000), (1000, 129), (2, 1000)])
def test_small_and_ragged_clouds_bit_equal_to_port(ctx, nP, nQ):
    sc = common.scenario(3000, 0.4, 0.02)
    P, Q = sc["P"][:nP], sc["Q"][:nQ]
    ctx.set_cloud_p(P, 0.05)
    ctx.set_cloud_q(Q)
    T16 = np.concatenate([common.candidates_colmajor(sc, 37), np.eye(4, dtype=np.float32).reshape(1, 16)])
    index, sq, _ = nearest_checked(ctx, T16)
    equal_to_port(P, Q, 0.05, T16, index, sq)
    # empty result: nothing within delta of anything
    far = np.eye(4, dtype=np.float32)
    far[:3, 3] = 50.0
    index, sq, counts = nearest_checked(ctx, far.T.reshape(1, 16))
    assert counts[0] == 0 and (index == -1).all() and np.isinf(sq).all()
    assert [len(a) for a in ctx.verify_nearest(np.zeros((0, 16), np.float32))] == [0, 0, 0]


def test_full_size_count_invariant_and_port_sample(ctx):
    """1M x 1M (cfg2): the count invariant for 16 transforms, and a 20K-query sample of rows against the port"""
    n, delta = 1_000_000, 0.003
    sc = common.scenario(n, 0.3, delta, seed=42)
    ctx.set_cloud_p(sc["P"], delta)
    ctx.set_cloud_q(sc["Q"])
    T16 = common.candidates_colmajor(sc, 16, n_near=8)
    index, sq, counts = nearest_checked(ctx, T16)
    assert (counts[:8] > 0.05 * n).all()
    sub = np.random.RandomState(0).choice(n, 20000, replace=False)
    two = T16[[0, 8]]                                          # one near-GT, one random transform
    equal_to_port(sc["P"], sc["Q"][sub], delta, two, index[[0, 8]][:, sub], sq[[0, 8]][:, sub])


def test_dev_form_equals_host_form(ctx):
    import torch
    sc = common.scenario(20000, 0.4, 0.01, seed=5)
    ctx.set_cloud_p(sc["P"], 0.01)
    ctx.set_cloud_q(sc["Q"])
    T16 = common.candidates_colmajor(sc, 20, n_near=6)
    index, sq, counts = ctx.verify_nearest(T16)
    K, nQ = T16.shape[0], ctx.nQ
    dT = torch.from_numpy(T16).cuda()
    d_index = torch.full((K, nQ), 7, dtype=torch.int32, device="cuda")
    d_sq = torch.zeros((K, nQ), dtype=torch.float32, device="cuda")
    d_counts = torch.full((K,), 99, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.verify_nearest_dev(dT.data_ptr(), K, d_index.data_ptr(), d_sq.data_ptr(), d_counts.data_ptr())
    ctx.synchronize()
    assert np.array_equal(d_index.cpu().numpy(), index)
    assert np.array_equal(common.bits(d_sq.cpu().numpy()), common.bits(sq))
    assert np.array_equal(d_counts.cpu().numpy().astype(np.uint32), counts)
    d_index.fill_(7)
    torch.cuda.synchronize()
    ctx.verify_nearest_dev(dT.data_ptr(), K, d_index.data_ptr(), None, None)   # sq_dist and counts are optional
    ctx.synchronize()
    assert np.array_equal(d_index.cpu().numpy(), index)
    L = ctx._L
    import ctypes as C
    out = np.empty((K, nQ), np.int32)
    assert L.s4g_verify_nearest(ctx.h, T16.ctypes.data_as(C.c_void_p), K, out.ctypes.data_as(C.c_void_p), None, None) == 0
    assert np.array_equal(out, index)
    assert L.s4g_verify_nearest(ctx.h, T16.ctypes.data_as(C.c_void_p), K, None, None, None) != 0   # index is required


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = correspondences.build(tmp_path_factory.mktemp("corr"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


def test_get_correspondences_hippo_golden(program, tmp_path):
    h = np.load(os.path.join(ROOT, "tests", "golden", "hippo.npz"))
    g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
    r = correspondences.run(program, tmp_path, h["P"], h["Q"], 0.01, 0.7, 200)
    assert r["threw_before"] == 1
    assert r["score"] == g["score"] == np.float32(0.64)
    assert np.array_equal(common.bits(r["T"]), common.bits(g["T_colmajor"]))
    assert (r["nearest"] >= 0).sum() == 128
    pi, ps, _ = onear.bruteforce(r["sP"], r["sQ"], 0.01, r["C"])
    assert np.array_equal(r["nearest"], pi[0]) and np.array_equal(common.bits(r["sq"]), common.bits(ps[0]))
    assert np.array_equal(r["nearest2"], r["nearest"])


def test_get_correspondences_synthetic_count_is_lcp(program, tmp_path):
    d = common.scenario(30000, 0.5, 0.01, seed=12)["raw"]
    r = correspondences.run(program, tmp_path, d["P"], d["Q"], 0.01, 0.5, 1000)
    count = int((r["nearest"] >= 0).sum())
    assert count > 0 and np.float32(count) / np.float32(len(r["sQ"])) == r["score"]
    pi, ps, _ = onear.bruteforce(r["sP"], r["sQ"], 0.01, r["C"])
    assert np.array_equal(r["nearest"], pi[0]) and np.array_equal(common.bits(r["sq"]), common.bits(ps[0]))
