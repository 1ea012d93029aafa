"""Voxel-grid downsampling (s4g_voxel_grid) without a GPU: the port (oracle/voxel_grid_port.cc) against an independent
numpy restatement of the contract, bit for bit, at the places its decisions and sums can go wrong (voxel faces, negative
and georeferenced coordinates, several runs of 1024 members, min_points, cancelling normals, empty and one-point clouds,
the argument errors), and Utils::VoxelGridFilter on the oracle stand-in.

Contract (include/s4g.h): voxel (floor(fl(x s)), ...), s = 1.0f / leaf; members in ascending index; sums in double over
runs of 1024 members left to right, then over the run sums; centroid and rgb = sum / m, normal = S / |S| or 0; voxels with
m < min_points dropped; output in order of each voxel's first member; voxel_of the output row or -1."""
import numpy as np
import pytest

from oracle import voxel_grid as ovg
from tests import build_shim, common, voxel_grid as tvg

_f = np.float32


def same(a, b):
    """bit equality of two port / restatement results (None for an array not computed)"""
    for x, y in zip(a, b):
        if x is None or y is None:
            assert x is None and y is None
            continue
        x, y = np.asarray(x), np.asarray(y)
        assert x.shape == y.shape, (x.shape, y.shape)
        if x.dtype == np.float32:
            assert np.array_equal(common.bits(x), common.bits(y)), np.argwhere(common.bits(x) != common.bits(y))[:5]
        else:
            assert np.array_equal(x, y)


def check(xyz, leaf, normals=None, rgb=None, min_points=1):
    got = ovg.port(xyz, leaf, normals, rgb, min_points)
    same(got, tvg.numpy_voxel_grid(xyz, leaf, normals, rgb, min_points))
    return got


@pytest.mark.parametrize("ppv", [1, 10, 2500])
@pytest.mark.parametrize("min_points", [1, 3])
def test_port_equals_numpy_restatement(ppv, min_points):
    X, N, R, leaf = tvg.cloud(20000, ppv, seed=ppv)
    out = check(X, leaf, N, R, min_points)
    assert out[3].sum() <= len(X) and (out[3] >= min_points).all()
    check(X, leaf)                                        # positions alone
    check(X, leaf, normals=N)
    check(X, leaf, rgb=R)


def test_points_on_voxel_faces_and_negative_coordinates():
    """x s an exact integer (the point opens the upper voxel), the float just below it, and negative coordinates, where
    floor and truncation differ: -0.25 lies in voxel -1, not 0"""
    leaf = 0.25                                           # s = 4 exactly
    base = np.array([-1.0, -0.5, -0.25, 0.0, 0.25, 0.5, 1.0], _f)
    below = np.nextafter(base, _f(-np.inf))
    above = np.nextafter(base, _f(np.inf))
    v = np.concatenate([base, below, above]).astype(_f)
    X = np.stack([v, np.roll(v, 3), -v], 1).astype(_f)
    out = check(X, leaf)
    C = np.floor(X * _f(4)).astype(np.int64)
    assert C[2, 0] == -1 and C[2 + 7, 0] == -2 and C[2 + 14, 0] == -1     # -0.25 on the face, below it, above it
    assert len(out[0]) == len(np.unique(C, axis=0))
    for i in range(len(X)):
        o = out[5][i]
        members = np.nonzero((C == C[i]).all(1))[0]
        assert out[3][o] == len(members) and out[4][o] == members[0]
    # a leaf whose reciprocal rounds: the voxel uses the float product, as s4g_voxel_sample
    check(X * _f(0.3), 0.1)


@pytest.mark.parametrize("offset", [1e5, -2.5e5])
def test_georeferenced_offsets(offset):
    """clouds far from the origin (UTM-like coordinates): the key is relative to the bounding-box voxel"""
    X, N, R, _ = tvg.cloud(5000, 1, seed=3, offset=0.0)
    X = (X.astype(np.float64) * 50 + offset).astype(_f)
    for leaf in (0.05, 0.5, 5.0):
        out = check(X, leaf, N, R)
        assert np.all(np.abs(out[0] - offset) < 60)


@pytest.mark.parametrize("m", [1024, 1025, 3000, 4096, 5000])
def test_one_voxel_with_several_runs(m):
    """every point in one voxel: runs of 1024 summed left to right, then the run sums; 1024 is one run, 1025 two"""
    rng = np.random.RandomState(m)
    X = (rng.random_sample((m, 3)) * 0.9 + 0.05).astype(_f)
    N = rng.normal(0, 1, (m, 3)).astype(_f)
    R = rng.random_sample((m, 3)).astype(_f)
    out = check(X, 1.0, N, R)
    assert len(out[0]) == 1 and out[3][0] == m and out[4][0] == 0 and (out[5] == 0).all()
    if m == 1024:                                        # one run: the plain left-to-right sum
        flat = np.array([np.cumsum(np.concatenate([[0.0], X[:, c].astype(np.float64)]))[-1] for c in range(3)])
        assert np.array_equal(common.bits((flat / m).astype(_f)), common.bits(out[0][0]))


def test_min_points_drops_voxels():
    """voxels of 1, 2, 3 and 5 points; min_points 1..6: the dropped voxels' points get voxel_of = -1, the survivors keep
    the order of their first points"""
    centres = np.array([[0.5, 0.5, 0.5], [3.5, 0.5, 0.5], [0.5, 2.5, 0.5], [1.5, 1.5, 4.5]], _f)
    sizes = [1, 2, 3, 5]
    rng = np.random.RandomState(0)
    X = np.concatenate([c + rng.uniform(-0.4, 0.4, (k, 3)) for c, k in zip(centres, sizes)]).astype(_f)
    perm = rng.permutation(len(X))
    X = X[perm]
    label = np.repeat(np.arange(4), sizes)[perm]
    for mp in range(1, 7):
        out = check(X, 1.0, min_points=mp)
        alive = [v for v in range(4) if sizes[v] >= mp]
        assert len(out[0]) == len(alive)
        assert sorted(out[3].tolist()) == sorted(sizes[v] for v in alive)
        assert ((out[5] == -1) == np.isin(label, [v for v in range(4) if v not in alive])).all()
        assert list(out[4]) == sorted(out[4])
        for i in np.nonzero(out[5] >= 0)[0]:
            assert out[3][out[5][i]] == sizes[label[i]]


def test_opposite_normals_cancel():
    X = np.array([[0.1, 0.1, 0.1], [0.2, 0.2, 0.2], [1.5, 0.1, 0.1], [1.6, 0.1, 0.1], [1.7, 0.1, 0.1]], _f)
    N = np.array([[0, 0, 1], [0, 0, -1], [1, 0, 0], [-1, 0, 0], [0, 0, 0]], _f)
    out = check(X, 1.0, normals=N)
    assert (out[1] == 0).all()                           # (0, 0, 0): "no normal"
    N2 = N.copy()
    N2[4] = [0, 2, 0]
    out = check(X, 1.0, normals=N2)
    assert (out[1][0] == 0).all() and np.array_equal(out[1][1], _f([0, 1, 0]))     # zero normals add nothing


def test_empty_and_single_point():
    out = check(np.zeros((0, 3), _f), 0.1)
    assert len(out[0]) == 0 and len(out[5]) == 0
    X = np.array([[-3.25, 7.5, 1e5]], _f)
    out = check(X, 0.5, np.array([[0, 3, 4]], _f), np.array([[0.2, 0.4, 0.6]], _f))
    assert np.array_equal(out[0], X) and np.array_equal(out[1], _f([[0, 0.6, 0.8]]))
    assert list(out[3]) == [1] and list(out[4]) == [0] and list(out[5]) == [0]
    assert len(ovg.port(X, 0.5, min_points=2)[0]) == 0


def test_errors():
    X = np.random.RandomState(1).rand(50, 3).astype(_f)
    for leaf in (0.0, -1.0, float("nan"), float("inf")):
        with pytest.raises(ovg.VoxelGridError):
            ovg.port(X, leaf)
    with pytest.raises(ovg.VoxelGridError):
        ovg.port(X, 0.1, min_points=0)
    for bad in (np.nan, np.inf, -np.inf):
        Y = X.copy()
        Y[17, 1] = bad
        with pytest.raises(ovg.VoxelGridError):
            ovg.port(Y, 0.1)
        with pytest.raises(ValueError):
            tvg.numpy_voxel_grid(Y, 0.1)
    Y = X.copy()
    Y[3, 0] = 3e38                                       # finite, but x s overflows the int32 range
    with pytest.raises(ovg.VoxelGridError):
        ovg.port(Y, 0.1)
    # span: 2^21 - 1 voxels is accepted, 2^21 is not
    leaf = 1.0
    Z = np.zeros((2, 3), _f)
    Z[1, 2] = 2 ** 21 - 1
    check(Z, leaf)
    Z[1, 2] = 2 ** 21
    with pytest.raises(ovg.VoxelGridError):
        ovg.port(Z, leaf)
    with pytest.raises(ValueError):
        tvg.numpy_voxel_grid(Z, leaf)


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    d = tmp_path_factory.mktemp("voxel_grid")
    exe = tvg.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


@pytest.mark.parametrize("colour", [True, False, "partial"])
@pytest.mark.parametrize("leaf,min_points", [(0.05, 1), (0.2, 1), (0.2, 20)])
def test_cpp_function_on_oracle_shim(program, tmp_path, colour, leaf, min_points):
    """the port's centroids and normals (the normal through set_normal once more), colours only when every point has
    one (an rgb other than the default (-1, -1, -1), which hasColor() does not tell apart); the returned size"""
    exe, shim = program
    X, N, R, _ = tvg.cloud(6000, 1, seed=4)
    rgb = R if colour else None
    if colour == "partial":
        rgb = R.copy()
        rgb[123] = -1                                    # one point with the default "no colour": none is averaged
    threw, count, pts = tvg.run(exe, tmp_path, X, N, rgb, leaf, min_points, preload=shim)
    assert not threw
    held = tvg.held(X, N, rgb)
    want = ovg.port(held[:, :3], leaf, held[:, 3:6], held[:, 6:] if colour is True else None, min_points)
    assert count == len(want[0]) == len(pts)
    assert np.array_equal(common.bits(pts), common.bits(tvg.expected_cloud(want)))
    assert (pts[:, 6:] == -1).all() == (colour is not True)


def test_cpp_function_throws_and_keeps_the_cloud(program, tmp_path):
    exe, shim = program
    X, N, R, _ = tvg.cloud(500, 1, seed=5)
    held = tvg.held(X, N, R)
    bad_x = X.copy()
    bad_x[7, 2] = np.nan
    wide = X.copy()
    wide[9, 0] = 3e6
    for xyz, leaf, mp in ((X, 0.0, 1), (X, -0.1, 1), (X, float("nan"), 1), (X, float("inf"), 1), (X, 0.1, 0),
                          (bad_x, 0.1, 1), (wide, 1.0, 1)):
        threw, _, pts = tvg.run(exe, tmp_path, xyz, N, R, leaf, mp, preload=shim)
        assert threw, (leaf, mp)
        assert np.array_equal(common.bits(pts), common.bits(tvg.held(xyz, N, R))), (leaf, mp)
    threw, count, pts = tvg.run(exe, tmp_path, X[:0], N[:0], R[:0], 0.1, 1, preload=shim)
    assert not threw and count == 0 and len(pts) == 0
    assert len(held) == 500
