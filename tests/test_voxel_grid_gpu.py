"""Voxel-grid downsampling on the GPU (s4g_voxel_grid): every output bit-equal to the port (oracle/voxel_grid_port.cc)
from 1 to 10^7 points, at leaves giving about 1, 10 and over 2000 points per voxel and min_points 1 and above; `first`
equal to s4g_voxel_sample at min_points = 1, on ordinary and georeferenced clouds; the _dev form equal to the host form
and its -1 sentinel; two calls bit-identical; the error codes; and Utils::VoxelGridFilter on the real library."""
import ctypes as C

import numpy as np
import pytest

from oracle import voxel_grid as ovg
from tests import common, voxel_grid as tvg

pytestmark = pytest.mark.gpu

S4G_OK, S4G_ERR_ARG = 0, 2   # include/s4g.h
_f = np.float32


def same(a, b):
    for x, y in zip(a, b):
        if x is None or y is None:
            assert x is None and y is None
            continue
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape, (x.shape, y.shape)
        if x.dtype == np.float32:
            bad = np.argwhere(common.bits(x) != common.bits(y))
            assert len(bad) == 0, (len(bad), bad[:5])
        else:
            bad = np.argwhere(x != y)
            assert len(bad) == 0, (len(bad), bad[:5])


@pytest.fixture(scope="module")
def ctx(s4g_lib):
    from super4pcs_b200 import Context
    with Context(0) as c:
        yield c


@pytest.mark.parametrize("n", [1, 2, 1000, 100_000, 1_000_000])
@pytest.mark.parametrize("ppv", [1, 10, 2500])
@pytest.mark.parametrize("min_points", [1, 4])
def test_bit_equal_to_port(ctx, n, ppv, min_points):
    X, N, R, leaf = tvg.cloud(n, ppv, seed=n + ppv)
    want = ovg.port(X, leaf, N, R, min_points)
    same(ctx.voxel_grid(X, leaf, N, R, min_points), want)
    same(ctx.voxel_grid(X, leaf, min_points=min_points), ovg.port(X, leaf, min_points=min_points))


@pytest.mark.parametrize("ppv,min_points", [(1, 1), (10, 3), (2500, 100)])
def test_bit_equal_to_port_at_ten_million(ctx, ppv, min_points):
    X, N, R, leaf = tvg.cloud(10_000_000, ppv, seed=7)
    same(ctx.voxel_grid(X, leaf, N, R, min_points), ovg.port(X, leaf, N, R, min_points))


@pytest.mark.parametrize("m", [1023, 1024, 1025, 2048, 2049, 100_000, 2_000_000])
def test_one_voxel(ctx, m):
    """all points in one voxel: one run, two runs, and many runs summed in order"""
    rng = np.random.RandomState(m)
    X = (rng.random_sample((m, 3)) * 0.9 + 0.05).astype(_f)
    N = rng.normal(0, 1, (m, 3)).astype(_f)
    R = rng.random_sample((m, 3)).astype(_f)
    got = ctx.voxel_grid(X, 1.0, N, R)
    same(got, ovg.port(X, 1.0, N, R))
    assert len(got[0]) == 1 and got[3][0] == m


def test_mixed_voxel_sizes(ctx):
    """voxels of 1 to 5000 points side by side, so that runs of multi-run voxels and single points share 1024-blocks"""
    rng = np.random.RandomState(5)
    sizes = np.concatenate([rng.randint(1, 5, 3000), rng.randint(1000, 5000, 40), [1024, 1025, 2048, 3072]])
    rng.shuffle(sizes)
    centres = rng.permutation(60 ** 3)[:len(sizes)]
    cell = np.stack([centres % 60, (centres // 60) % 60, centres // 3600], 1)
    X = np.concatenate([c + rng.uniform(0.01, 0.99, (k, 3)) for c, k in zip(cell, sizes)]).astype(_f)
    X = X[rng.permutation(len(X))]
    N = rng.normal(0, 1, X.shape).astype(_f)
    for mp in (1, 2, 1024, 1025, 4000):
        same(ctx.voxel_grid(X, 1.0, N, None, mp), ovg.port(X, 1.0, N, None, mp))


@pytest.mark.parametrize("offset", [0.0, 1e5, -3e5])
@pytest.mark.parametrize("ppv", [1, 30])
def test_first_equals_voxel_sample(ctx, offset, ppv):
    X, _, _, leaf = tvg.cloud(200_000, ppv, seed=11)
    X = (X.astype(np.float64) * 100 + offset).astype(_f)
    leaf *= 100
    got = ctx.voxel_grid(X, leaf)
    assert np.array_equal(got[4], ctx.voxel_sample(X, leaf))
    same(got, ovg.port(X, leaf))


def test_faces_negative_and_span_limit(ctx):
    leaf = 0.25
    base = np.array([-1.0, -0.5, -0.25, 0.0, 0.25, 0.5, 1.0], _f)
    v = np.concatenate([base, np.nextafter(base, _f(-np.inf)), np.nextafter(base, _f(np.inf))]).astype(_f)
    X = np.stack([v, np.roll(v, 3), -v], 1).astype(_f)
    same(ctx.voxel_grid(X, leaf), ovg.port(X, leaf))
    Z = np.zeros((3, 3), _f)
    Z[1, 2] = 2 ** 21 - 1
    same(ctx.voxel_grid(Z, 1.0), ovg.port(Z, 1.0))


def test_repeatable(ctx):
    X, N, R, leaf = tvg.cloud(2_000_000, 10, seed=13)
    a = ctx.voxel_grid(X, leaf, N, R, 2)
    b = ctx.voxel_grid(X, leaf, N, R, 2)
    same(a, b)


def test_dev_form_equals_host_form(ctx):
    import torch
    X, N, R, leaf = tvg.cloud(300_000, 10, seed=17)
    n = len(X)
    for mp in (1, 5):
        want = ctx.voxel_grid(X, leaf, N, R, mp)
        dx, dn, dr = (torch.from_numpy(a).cuda() for a in (X, N, R))
        ox, on, orr = (torch.full((n, 3), 7.0, dtype=torch.float32, device="cuda") for _ in range(3))
        cnt, fst, vof = (torch.full((n,), 7, dtype=torch.int32, device="cuda") for _ in range(3))
        m = torch.zeros(1, dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        ctx.voxel_grid_dev(dx.data_ptr(), n, leaf, ox.data_ptr(), m.data_ptr(), dn.data_ptr(), dr.data_ptr(),
                           on.data_ptr(), orr.data_ptr(), cnt.data_ptr(), fst.data_ptr(), vof.data_ptr(), min_points=mp)
        ctx.synchronize()
        k = int(m.item())
        same((ox[:k].cpu().numpy(), on[:k].cpu().numpy(), orr[:k].cpu().numpy(), cnt[:k].cpu().numpy(),
              fst[:k].cpu().numpy(), vof.cpu().numpy()), want)
        m.zero_()
        ctx.voxel_grid_dev(dx.data_ptr(), n, leaf, ox.data_ptr(), m.data_ptr(), min_points=mp)   # the rest optional
        ctx.synchronize()
        assert int(m.item()) == k
        assert np.array_equal(common.bits(ox[:k].cpu().numpy()), common.bits(want[0]))
    # the sentinel: a non-finite coordinate or too wide a span gives *d_n_out = -1
    for bad in (float("nan"), float("inf")):
        Y = X.copy()
        Y[12345, 1] = bad
        dy = torch.from_numpy(Y).cuda()
        ctx.voxel_grid_dev(dy.data_ptr(), n, leaf, ox.data_ptr(), m.data_ptr())
        ctx.synchronize()
        assert int(m.item()) == -1
    Y = X.copy()
    Y[5, 0] = 2 ** 22
    dy = torch.from_numpy(Y).cuda()
    ctx.voxel_grid_dev(dy.data_ptr(), n, 1.0, ox.data_ptr(), m.data_ptr())
    ctx.synchronize()
    assert int(m.item()) == -1
    m.fill_(5)
    ctx.voxel_grid_dev(dx.data_ptr(), 0, leaf, ox.data_ptr(), m.data_ptr())
    ctx.synchronize()
    assert int(m.item()) == 0


def test_error_codes(ctx):
    L, h = ctx._L, ctx.h
    X = np.random.RandomState(0).rand(100, 3).astype(_f)
    out, cnt = np.empty((100, 3), _f), np.empty(100, np.int32)
    m = C.c_int64(5)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    call = lambda xyz, n, leaf, mp, nrm=None, nout=None, o=p(out), nn=C.byref(m): L.s4g_voxel_grid(  # noqa: E731
        h, xyz, nrm, None, n, leaf, mp, o, nout, None, None, None, None, nn)
    assert call(p(X), 100, 0.1, 1) == S4G_OK and 0 < m.value <= 100
    for leaf in (0.0, -0.5, float("nan"), float("inf")):
        assert call(p(X), 100, leaf, 1) == S4G_ERR_ARG
    assert "leaf" in L.s4g_error_string(h).decode()
    assert call(p(X), 100, 0.1, 0) == S4G_ERR_ARG
    assert call(p(X), -1, 0.1, 1) == S4G_ERR_ARG
    assert call(p(X), 2 ** 31, 0.1, 1) == S4G_ERR_ARG
    assert call(None, 100, 0.1, 1) == S4G_ERR_ARG
    assert call(p(X), 100, 0.1, 1, o=None) == S4G_ERR_ARG
    assert call(p(X), 100, 0.1, 1, nn=None) == S4G_ERR_ARG
    assert call(p(X), 100, 0.1, 1, nrm=p(X)) == S4G_ERR_ARG            # normals without normals_out
    assert call(p(X), 100, 0.1, 1, nout=p(out)) == S4G_ERR_ARG         # and the other way round
    assert L.s4g_voxel_grid(None, p(X), None, None, 100, 0.1, 1, p(out), None, None, None, None, None,
                            C.byref(m)) == S4G_ERR_ARG
    for bad in (np.nan, np.inf, -np.inf, 3e38):
        Y = X.copy()
        Y[42, 2] = bad
        assert call(p(Y), 100, 0.1, 1) == S4G_ERR_ARG
        assert "finite" in L.s4g_error_string(h).decode()
    Y = X.copy()
    Y[7, 0] = 2 ** 21
    assert call(p(Y), 100, 1.0, 1) == S4G_ERR_ARG
    assert "2^21" in L.s4g_error_string(h).decode()
    m.value = 5
    assert call(p(X), 0, 0.1, 1) == S4G_OK and m.value == 0
    assert L.s4g_voxel_grid(h, p(X), None, None, 100, 0.1, 1, p(out), None, None, p(cnt), None, None,
                            C.byref(m)) == S4G_OK
    assert cnt[:m.value].sum() == 100
    with pytest.raises(Exception):
        ctx.voxel_grid(X, -1.0)


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = tvg.build(tmp_path_factory.mktemp("voxel_grid"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


@pytest.mark.parametrize("colour", [True, False])
@pytest.mark.parametrize("ppv,min_points", [(1, 1), (10, 1), (10, 5)])
def test_cpp_function_equals_context(program, ctx, tmp_path, colour, ppv, min_points):
    X, N, R, leaf = tvg.cloud(200_000, ppv, seed=19)
    rgb = R if colour else None
    threw, count, pts = tvg.run(program, tmp_path, X, N, rgb, leaf, min_points)
    assert not threw
    held = tvg.held(X, N, rgb)
    want = ctx.voxel_grid(held[:, :3], leaf, held[:, 3:6], held[:, 6:] if colour else None, min_points)
    assert count == len(want[0]) == len(pts)
    assert np.array_equal(common.bits(pts), common.bits(tvg.expected_cloud(want)))


def test_cpp_function_throws_and_keeps_the_cloud(program, tmp_path):
    X, N, R, _ = tvg.cloud(1000, 1, seed=23)
    Y = X.copy()
    Y[3, 1] = np.inf
    for xyz, leaf in ((X, -1.0), (Y, 0.1)):
        threw, _, pts = tvg.run(program, tmp_path, xyz, N, R, leaf, 1)
        assert threw
        assert np.array_equal(common.bits(pts), common.bits(tvg.held(xyz, N, R)))
