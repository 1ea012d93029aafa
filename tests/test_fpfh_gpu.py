"""s4g_fpfh and s4g_fpfh_match on the GPU: every output bit equal to the port (oracle/fpfh_port.cc) from 1 to 10^6
points at k = 1, 16 and 64, with a finite and an infinite radius, on s4g_normals' normals unoriented and oriented by
s4g_orient_normals, and on pairs built so that their f1, f2, f3 and swap decisions lie within double rounding of a face; two calls bit-identical;
the _dev form chained after s4g_normals_dev -> s4g_orient_normals_dev with no host round trip; the match bit-equal to the
port with ties, NaN rows, mutual and the _dev form; the error codes; Utils::ComputeFPFH / Utils::MatchFPFH against
Context; and one end-to-end check: a bumpy surface and a rigidly moved copy, oriented -> FPFH -> mutual match.

Up to 20 000 points the port builds its own rows by brute force.  Above, it is given the rows and d^2 of s4g_knn with
self-exclusion, which tests/test_knn_gpu.py holds to the brute force bit for bit."""
import numpy as np
import pytest

from oracle import fpfh as ofpfh
from tests import common, fpfh as tf

pytestmark = pytest.mark.gpu

S4G_OK, S4G_ERR_ARG, S4G_ERR_STATE = 0, 2, 3   # include/s4g.h
_f = np.float32
VIEW = np.float32([0.3, -2.0, 1.5])


def same(got, want, what=""):
    assert np.array_equal(common.bits(got), common.bits(want)), (what, np.argwhere(common.bits(got) != common.bits(want))[:5])


@pytest.fixture(scope="module")
def ctx(s4g_lib):
    from super4pcs_b200 import Context
    with Context(0) as c:
        yield c


def delta_of(n):
    return float(2.0 * np.sqrt(16.0 / max(n, 1)))


def normals_of(ctx, oriented):
    N, _ = ctx.normals(16)
    return ctx.orient_normals(N, 16, viewpoint=VIEW)[0] if oriented else N


@pytest.mark.parametrize("n", [1, 2, 3, 100, 5000, 20_000])
@pytest.mark.parametrize("k", [1, 16, 64])
def test_bit_equal_to_port_small(ctx, n, k):
    P = tf.surface(n, seed=n + k)
    ctx.set_cloud_p(P, delta_of(n))
    for oriented in (False, True):
        N = normals_of(ctx, oriented)
        for r in (np.inf, 16.0 / n):
            same(ctx.fpfh(N, k, r), ofpfh.port(P, N, k, r), (oriented, r))


@pytest.mark.parametrize("k", [16, 64])
def test_bit_equal_to_port_million(ctx, k):
    n = 1_000_000
    P = tf.surface(n, seed=k)
    ctx.set_cloud_p(P, delta_of(n))
    N = normals_of(ctx, True)
    for r in (np.inf, 4e-6):
        rows, sq = ctx.knn(P, k, r, exclude=np.arange(n, dtype=np.int32))
        same(ctx.fpfh(N, k, r), ofpfh.port(P, N, k, r, rows=rows, sq=sq), r)


def test_pairs_on_faces(ctx):
    """tests/fpfh.py's face_pairs: rows whose f1 face test lies within about 1e-14 of zero, and rows whose f2, f3 or swap
    decision lies exactly on its face, so that only the rounding of the double arithmetic decides; on these a kernel that
    takes f1 from atan2, reassociates a dot product or swaps on |a1| <= |a2| gives other bins
    (tests/test_fpfh_cpu.py::test_pairs_on_faces shows each on the same inputs)"""
    P, N, kind = tf.face_pairs()
    m = len(kind)
    _, margin = tf.contract_pairs_np(P[:m], N[:m], P[m:], N[m:])
    assert (margin["f1"][kind == 1] < 1e-14).sum() >= 200
    assert all((margin[name][kind == k] < 1e-15).all() for k, name in ((2, "f2"), (3, "f3"), (4, "swap")))
    ctx.set_cloud_p(P, 8.0)
    for r in (np.inf, 300.0):
        same(ctx.fpfh(N, 1, r), ofpfh.port(P, N, 1, r), r)
    same(ctx.fpfh(-N, 1), ofpfh.port(P, -N, 1))
    same(ctx.fpfh(N, 4), ofpfh.port(P, N, 4))


def ofpfh_rows(P, k):
    from oracle import knn as oknn
    return oknn.bruteforce(P, P, k, np.inf, exclude=np.arange(len(P), dtype=np.int32))


def test_special_normals(ctx):
    P = tf.surface(3000, seed=7)
    ctx.set_cloud_p(P, delta_of(3000))
    N = normals_of(ctx, True).copy()
    N[::11] *= 7.0
    N[1::13] = 0
    N[2::17] = [np.nan, 0, 1]
    N[3::19] = [0, -np.inf, 0]
    got = ctx.fpfh(N, 16)
    same(got, ofpfh.port(P, N, 16))
    assert not got[1::13].any()


def test_repeatable(ctx):
    P = tf.surface(200_000, seed=1)
    ctx.set_cloud_p(P, delta_of(200_000))
    N = normals_of(ctx, True)
    a = ctx.fpfh(N, 32)
    b = ctx.fpfh(N, 32)
    same(a, b)


def test_dev_chained(ctx):
    import torch
    n = 100_000
    P = tf.surface(n, seed=12)
    ctx.set_cloud_p(P, delta_of(n))
    dN = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    out2 = torch.empty(2, dtype=torch.int64, device="cuda")
    dF = torch.full((n, 33), np.nan, dtype=torch.float32, device="cuda")
    ctx.normals_dev(16, dN.data_ptr())
    ctx.orient_normals_dev(dN.data_ptr(), 16, dN.data_ptr(), out2.data_ptr(), viewpoint=VIEW)
    ctx.fpfh_dev(dN.data_ptr(), 24, dF.data_ptr(), 1e-3)
    torch.cuda.synchronize()
    N = normals_of(ctx, True)
    same(dF.cpu().numpy(), ctx.fpfh(N, 24, 1e-3))
    same(dN.cpu().numpy(), N)


def descriptors(n, seed):
    rng = np.random.RandomState(seed)
    return rng.uniform(0, 60, (n, 33)).astype(_f)


@pytest.mark.parametrize("na, nb", [(1, 1), (1, 1000), (1000, 1), (1000, 1000), (1, 100_000), (100_000, 1),
                                    (1000, 100_000), (100_000, 1000)])
def test_match_bit_equal_to_port(ctx, na, nb):
    A, B = descriptors(na, na + 1), descriptors(nb, nb + 2)
    if nb > 10:
        B[5] = B[3]                                  # a tie: the smaller index wins
        B[7] = np.nan                                # never wins
        B[8, 4] = np.inf
    if na > 10:
        A[2] = np.nan                                # no finite d^2: -1, +inf
        A[4] = B[min(5, nb - 1)]
        A[6] = B[min(5, nb - 1)]                     # two a-rows on one b-row: mutual keeps the first
    for mutual in (False, True):
        got = ctx.fpfh_match(A, B, mutual)
        want = ofpfh.match_port(A, B, mutual)
        assert np.array_equal(got[0], want[0]), mutual
        same(got[1], want[1])


def test_match_empty(ctx):
    A = descriptors(10, 1)
    idx, sq = ctx.fpfh_match(A, A[:0], True)
    assert (idx == -1).all() and np.isinf(sq).all()
    idx, sq = ctx.fpfh_match(A[:0], A, True)
    assert len(idx) == 0


def test_match_dev(ctx):
    import torch
    A, B = descriptors(20_000, 3), descriptors(30_000, 4)
    B[:5000] = A[:5000] + 0.01
    dA, dB = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    di = torch.empty(len(A), dtype=torch.int32, device="cuda")
    ds = torch.empty(len(A), dtype=torch.float32, device="cuda")
    for mutual in (False, True):
        ctx.fpfh_match_dev(dA.data_ptr(), len(A), dB.data_ptr(), len(B), di.data_ptr(), ds.data_ptr(), mutual=mutual)
        torch.cuda.synchronize()
        got = ctx.fpfh_match(A, B, mutual)
        assert np.array_equal(di.cpu().numpy(), got[0])
        same(ds.cpu().numpy(), got[1])
    ctx.fpfh_match_dev(dA.data_ptr(), len(A), dB.data_ptr(), len(B), di.data_ptr(), None, mutual=True)
    torch.cuda.synchronize()
    assert np.array_equal(di.cpu().numpy(), got[0])


def test_error_codes(s4g_lib):
    import ctypes as C
    from super4pcs_b200 import Context, s4g
    L = s4g.load_library()
    with Context(0) as c:
        N = np.zeros((10, 3), _f)
        F = np.zeros((10, 33), _f)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        assert L.s4g_fpfh(c.h, p(N), 8, float("inf"), p(F)) == S4G_ERR_STATE
        c.set_cloud_p(tf.surface(10, 1), 0.5)
        for k, r in ((0, np.inf), (65, np.inf), (8, -1.0), (8, np.nan)):
            assert L.s4g_fpfh(c.h, p(N), k, float(r), p(F)) == S4G_ERR_ARG, (k, r)
            assert L.s4g_fpfh_dev(c.h, None, k, float(r), None) == S4G_ERR_ARG
        assert L.s4g_fpfh(c.h, None, 8, float("inf"), p(F)) == S4G_ERR_ARG
        assert L.s4g_fpfh(c.h, p(N), 8, float("inf"), None) == S4G_ERR_ARG
        assert L.s4g_fpfh(c.h, p(N), 8, float("inf"), p(F)) == S4G_OK
        I = np.zeros(10, np.int32)
        assert L.s4g_fpfh_match(c.h, p(F), -1, p(F), 10, 0, p(I), None) == S4G_ERR_ARG
        assert L.s4g_fpfh_match(c.h, p(F), 10, p(F), 2 ** 31, 0, p(I), None) == S4G_ERR_ARG
        assert L.s4g_fpfh_match(c.h, None, 10, p(F), 10, 0, p(I), None) == S4G_ERR_ARG
        assert L.s4g_fpfh_match(c.h, p(F), 10, None, 10, 0, p(I), None) == S4G_ERR_ARG
        assert L.s4g_fpfh_match(c.h, p(F), 10, p(F), 10, 0, None, None) == S4G_ERR_ARG
        assert L.s4g_fpfh_match(c.h, p(F), 0, p(F), 10, 0, p(I), None) == S4G_OK
        assert L.s4g_fpfh_match(c.h, p(F), 10, p(F), 10, 1, p(I), None) == S4G_OK


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = tf.build(tmp_path_factory.mktemp("fpfh"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


def test_cpp_functions(ctx, program, tmp_path):
    from tests import normals as tnormals
    P = tf.surface(20_000, seed=8)
    ctx.set_cloud_p(P, delta_of(20_000))
    N = normals_of(ctx, True)
    held = tnormals.set_normal(N)
    got = tf.run_compute(program, tmp_path, P, N, 32, 0.05)
    ctx.set_cloud_p(P, tnormals.grid_delta(P, 32))
    same(got, ctx.fpfh(held, 32, np.float32(0.05) * np.float32(0.05)))
    idx = tf.run_match(program, tmp_path, got[:5000], got[5000:12000], True)
    assert np.array_equal(idx, ctx.fpfh_match(got[:5000], got[5000:12000], True)[0])


def moved(P, seed):
    rng = np.random.RandomState(seed)
    R, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    if np.linalg.det(R) < 0:
        R[:, 0] *= -1
    t = np.array([0.3, -0.2, 0.5])
    perm = rng.permutation(len(P))
    return (P.astype(np.float64) @ R.T + t).astype(_f)[perm], perm, R, t


def test_end_to_end_correspondences(ctx):
    """a bumpy surface and a rigidly moved, permuted copy: estimate -> orient (viewpoints that move with the cloud) ->
    FPFH (k = 32) -> mutual match.  On this input the port (computable on the CPU: tests/fpfh.py's restatements) matches
    49.5 % of the points mutually, and 99.96 % of those matches are the true correspondences; the GPU gives the same
    matches bit for bit"""
    from oracle import normals as onormals, orient_normals as oon
    n = 5000
    P = tf.surface(n, seed=21, bumps=8)
    Q, perm, R, t = moved(P, 5)
    vp = np.float32([0, 0, 5])
    vq = (vp.astype(np.float64) @ R.T + t).astype(_f)

    def gpu(X, v):
        ctx.set_cloud_p(X, delta_of(n))
        N, _ = ctx.normals(16)
        return ctx.fpfh(ctx.orient_normals(N, 16, viewpoint=v)[0], 32)

    def port(X, v):
        N = onormals.port(X, 16)[0]
        return ofpfh.port(X, oon.port(X, N, 16, viewpoint=v)[0], 32)

    FP, FQ = gpu(P, vp), gpu(Q, vq)
    same(FP, port(P, vp))
    same(FQ, port(Q, vq))
    idx, _ = ctx.fpfh_match(FP, FQ, True)
    assert np.array_equal(idx, ofpfh.match_port(FP, FQ, True)[0])
    inv = np.empty(n, np.int64)
    inv[perm] = np.arange(n)
    ok = idx >= 0
    assert ok.mean() > 0.45 and (idx[ok] == inv[ok]).mean() > 0.99
