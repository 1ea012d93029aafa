"""s4g_orient_normals on the GPU: the oriented normals, root, out2 and the forest bit-equal to the port
(oracle/orient_normals_port.cc: Kruskal and a breadth-first walk) from 2 to 10^6 points at k = 1, 8, 16 and 64, on normals
from s4g_normals and on random ones, with and without a viewpoint, and at a radius that leaves many components; two calls
bit-identical; the _dev form in place and chained after s4g_normals_dev with no host round trip; its -1 sentinel; the
error codes; Utils::OrientNormals against Context; and the motivation end to end: a dense sphere's normals averaged by
s4g_voxel_grid agree with the analytic normal only once they are oriented.

Up to 20 000 points the port builds its own rows by brute force.  Above, it is given the rows of s4g_knn with
self-exclusion, which tests/test_knn_gpu.py holds to the brute force bit for bit; a sample of them is checked here too."""
import ctypes as C

import numpy as np
import pytest

from oracle import knn as oknn, orient_normals as oon
from tests import common, orient_normals as ton

pytestmark = pytest.mark.gpu

S4G_OK, S4G_ERR_ARG, S4G_ERR_STATE = 0, 2, 3   # include/s4g.h
_f = np.float32
VIEW = np.float32([0.3, -2.0, 1.5])


def same(got, want, what=""):
    assert got[2] == want[2], (what, got[2], want[2])
    assert np.array_equal(common.bits(got[0]), common.bits(want[0])), (what, np.argwhere(got[0] != want[0])[:5])
    assert np.array_equal(got[1], want[1]), what
    assert np.array_equal(got[3], want[3]), (what, len(got[3]), len(want[3]))


@pytest.fixture(scope="module")
def ctx(s4g_lib):
    from super4pcs_b200 import Context
    with Context(0) as c:
        yield c


def cloud(n, seed):
    """a sampled surface (a wavy sheet with a bump) and a few stray points, so that s4g_normals gives real normals"""
    rng = np.random.RandomState(seed)
    uv = rng.uniform(-1, 1, (n, 2))
    z = 0.2 * np.sin(3 * uv[:, 0]) * np.cos(2 * uv[:, 1]) + 0.3 * np.exp(-8 * (uv ** 2).sum(1))
    P = np.concatenate([uv, z[:, None]], 1)
    stray = rng.rand(n) < 0.01
    P[stray] += rng.normal(0, 0.2, (stray.sum(), 3))
    return P.astype(_f)


def delta_of(n):
    return float(2.0 * np.sqrt(16.0 / max(n, 1)))


def rows_of(ctx, P, k, sq_radius):
    n = len(P)
    return ctx.knn(P, k, sq_radius, exclude=np.arange(n, dtype=np.int32))[0]


def inputs(ctx, P, kind, seed):
    if kind == "estimated":
        N, _ = ctx.normals(16)
        return N
    rng = np.random.RandomState(seed)
    N = rng.normal(0, 1, (len(P), 3)).astype(_f)
    N[rng.rand(len(P)) < 0.02] = 0                     # points without a normal
    return N


@pytest.mark.parametrize("n", [2, 3, 100, 1000, 20_000])
@pytest.mark.parametrize("k", [1, 8, 16, 64])
def test_bit_equal_to_port_small(ctx, n, k):
    P = cloud(n, n + k)
    ctx.set_cloud_p(P, delta_of(n))
    for kind in ("estimated", "random"):
        N = inputs(ctx, P, kind, n)
        for r in (np.inf, 4.0 / n):                       # unbounded, and a radius that leaves many components
            for vp in (None, VIEW):
                same(ctx.orient_normals(N, k, r, vp), oon.port(P, N, k, r, vp), (kind, r, vp is None))


@pytest.mark.parametrize("n,k", [(200_000, 1), (200_000, 64), (1_000_000, 1), (1_000_000, 8), (1_000_000, 16),
                                 (1_000_000, 64)])
def test_bit_equal_to_port_large(ctx, n, k):
    P = cloud(n, 7)
    ctx.set_cloud_p(P, delta_of(n))
    kinds = ("estimated", "random") if n <= 200_000 or k == 16 else (("estimated",) if k != 1 else ("random",))
    for kind in kinds:
        N = inputs(ctx, P, kind, k)
        for r in ((np.inf, 4.0 / n) if k != 64 else (np.inf,)):
            rows = rows_of(ctx, P, k, r)
            pick = np.random.RandomState(k).choice(n, 300, replace=False)
            want_rows, _ = oknn.bruteforce(P, P[pick], k, r, exclude=pick.astype(np.int32))
            assert np.array_equal(rows[pick], want_rows)
            vp = VIEW if kind == "estimated" else None
            got = ctx.orient_normals(N, k, r, vp)
            want = oon.port(P, N, k, r, vp, rows=rows)
            same(got, want, (kind, r))
            assert len(got[3]) == int(((N != 0).any(1)).sum()) - got[2]


def test_repeatable(ctx):
    n = 300_000
    P = cloud(n, 3)
    ctx.set_cloud_p(P, delta_of(n))
    N = inputs(ctx, P, "random", 3)
    a = ctx.orient_normals(N, 16, viewpoint=VIEW)
    for _ in range(3):
        same(ctx.orient_normals(N, 16, viewpoint=VIEW), a)


def test_dev_in_place_and_chained_after_normals_dev(ctx):
    import torch
    n, k = 100_000, 16
    P = cloud(n, 5)
    ctx.set_cloud_p(P, delta_of(n))
    d_n = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    d_root = torch.empty(n, dtype=torch.int32, device="cuda")
    d_out2 = torch.zeros(2, dtype=torch.int64, device="cuda")
    d_tree = torch.empty((n - 1, 2), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.normals_dev(16, d_n.data_ptr(), viewpoint=VIEW)
    ctx.orient_normals_dev(d_n.data_ptr(), k, d_n.data_ptr(), d_out2.data_ptr(), d_root.data_ptr(), d_tree.data_ptr(),
                           viewpoint=VIEW)
    ctx.synchronize()
    N, _ = ctx.normals(16, viewpoint=VIEW)
    want = ctx.orient_normals(N, k, viewpoint=VIEW)
    nc, nt = [int(x) for x in d_out2.cpu()]
    same((d_n.cpu().numpy(), d_root.cpu().numpy(), nc, d_tree.cpu().numpy()[:nt]), want)
    # without root and the forest, into a second buffer
    d_o = torch.empty_like(d_n)
    d_in = torch.from_numpy(N).cuda()
    torch.cuda.synchronize()
    ctx.orient_normals_dev(d_in.data_ptr(), k, d_o.data_ptr(), d_out2.data_ptr(), viewpoint=VIEW)
    ctx.synchronize()
    assert np.array_equal(common.bits(d_o.cpu().numpy()), common.bits(want[0]))
    assert np.array_equal(common.bits(d_in.cpu().numpy()), common.bits(N))        # the input is left as it was
    # the sentinel of a non-finite normal
    N[77, 1] = np.inf
    d_in = torch.from_numpy(N).cuda()
    torch.cuda.synchronize()
    ctx.orient_normals_dev(d_in.data_ptr(), k, d_o.data_ptr(), d_out2.data_ptr())
    ctx.synchronize()
    assert int(d_out2[0].item()) == -1


def test_error_codes(s4g_lib):
    from super4pcs_b200 import Context
    L = s4g_lib
    with Context(0) as c:
        h = c.h
        n = 200
        P = np.random.RandomState(0).rand(n, 3).astype(_f)
        N = np.random.RandomState(1).normal(size=(n, 3)).astype(_f)
        out, root, tree = np.empty((n, 3), _f), np.empty(n, np.int32), np.empty(2 * n, np.int32)
        out2 = np.zeros(2, np.int64)
        p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)  # noqa: E731

        def call(nrm=N, k=8, r=np.inf, vp=None, o=out, o2=out2):
            return L.s4g_orient_normals(h, p(nrm), k, r, p(vp), p(o), p(root), p(o2), p(tree))

        assert call() == S4G_ERR_STATE                  # before s4g_set_cloud_p
        assert "set_cloud_p" in L.s4g_error_string(h).decode()
        c.set_cloud_p(P, 0.1)
        assert call() == S4G_OK and out2[0] >= 1
        for k in (0, 65, -1):
            assert call(k=k) == S4G_ERR_ARG
        for r in (float("nan"), -1.0):
            assert call(r=r) == S4G_ERR_ARG
        assert call(nrm=None) == S4G_ERR_ARG
        assert call(o=None) == S4G_ERR_ARG
        assert call(o2=None) == S4G_ERR_ARG
        for bad in (np.nan, np.inf):
            assert call(vp=np.float32([0, bad, 0])) == S4G_ERR_ARG
            M = N.copy()
            M[13, 2] = bad
            assert call(nrm=M) == S4G_ERR_ARG
            assert "finite" in L.s4g_error_string(h).decode()
        assert L.s4g_orient_normals(None, p(N), 8, np.inf, None, p(out), None, p(out2), None) == S4G_ERR_ARG
        assert L.s4g_orient_normals(h, p(N), 8, np.inf, None, p(out), None, p(out2), None) == S4G_OK  # root, tree NULL
        assert L.s4g_orient_normals_dev(h, None, 8, np.inf, None, None, None, None, None) == S4G_ERR_ARG
        M = N.copy()
        assert L.s4g_orient_normals(h, p(M), 8, 0.01, None, p(M), None, p(out2), None) == S4G_OK   # in place
        assert np.array_equal(common.bits(M), common.bits(oon.port(P, N, 8, 0.01)[0]))
        with pytest.raises(Exception):
            c.orient_normals(N[:10], 8)


def test_sphere_voxel_grid_needs_orientation(ctx):
    """the dense sphere -> s4g_normals -> s4g_voxel_grid with normals: unoriented, some voxel averages are off the
    analytic normal by more than 10 degrees; oriented first (viewpoint outside), none is"""
    X, _ = ton.sphere(400_000, 2)
    ctx.set_cloud_p(X, delta_of(len(X)))
    N, _ = ctx.normals(16)
    leaf = 0.05

    def worst(normals):
        xyz, nrm, _, counts, _, _ = ctx.voxel_grid(X, leaf, normals=normals)
        truth = xyz / np.linalg.norm(xyz, axis=1, keepdims=True)
        ok = np.linalg.norm(nrm, axis=1) > 0
        cos = np.where(ok, (nrm * truth).sum(1), -1.0)
        return np.degrees(np.arccos(np.clip(cos, -1, 1)))

    before = worst(N)
    assert (before > 10).sum() > 100, (before > 10).sum()
    oriented, _, n_comp, _ = ctx.orient_normals(N, 16, viewpoint=[0.0, 0.0, 5.0])
    assert n_comp == 1
    after = worst(oriented)
    assert after.max() < 10, after.max()


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = ton.build(tmp_path_factory.mktemp("orient_normals"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


@pytest.mark.parametrize("vp", [None, (0.0, 0.0, 5.0)])
def test_cpp_function_equals_context(program, ctx, tmp_path, vp):
    from tests import normals as tnormals
    X, T = ton.torus(100_000, 4)
    N = ton.scramble(T, 4)
    held = tnormals.set_normal(N)
    threw, count, got = ton.run(program, tmp_path, X, N, 16, viewpoint=vp)
    assert not threw
    ctx.set_cloud_p(X, delta_of(len(X)))
    want = ctx.orient_normals(held, 16, viewpoint=None if vp is None else np.float32(vp))
    assert count == want[2]
    assert np.array_equal(common.bits(got), common.bits(ton.expected_held(held, want[0])))
    if vp is not None:
        assert ((got * T).sum(1) > 0).all()
    threw, _, got = ton.run(program, tmp_path, X, N, 0)
    assert threw and np.array_equal(common.bits(got), common.bits(held))
