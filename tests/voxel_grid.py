"""Builds and runs tests/cpp/voxel_grid_main.cc, the test program of Utils::VoxelGridFilter, for
tests/test_voxel_grid_cpu.py (on the oracle stand-in) and tests/test_voxel_grid_gpu.py (on the real library).  Also an
independent numpy restatement of the s4g_voxel_grid contract, and the clouds the tests share."""
import numpy as np

from tests import cpp_main, normals as tnormals

_f = np.float32


def build(outdir):
    return cpp_main.build("voxel_grid_main", outdir)


def run(exe, workdir, xyz, normals, rgb, leaf, min_points, preload=None):
    """rgb None: the points get no colour -> (threw, returned count, points [m, 9] float32: position, normal, rgb of each
    point of the cloud after the call, as Point3D holds them)"""
    xyz = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    has_rgb = rgb is not None
    rgb = np.zeros_like(xyz) if rgb is None else rgb
    blob = np.concatenate([xyz, np.asarray(normals, _f).reshape(-1, 3), np.asarray(rgb, _f).reshape(-1, 3)])
    payload = np.int32([len(xyz), int(has_rgb)]).tobytes() + np.ascontiguousarray(blob, _f).tobytes()
    r = cpp_main.Reader(cpp_main.run(exe, workdir, payload, [repr(float(leaf)), str(int(min_points))], preload))
    threw, count, m = r.take(np.int32, 3)
    return bool(threw), int(count), r.take(_f, 9 * int(m)).reshape(-1, 9)


def held(xyz, normals, rgb):
    """[n, 9] float32: what the program's Point3D hold (the normal through set_normal; rgb None: no colour)"""
    xyz = np.asarray(xyz, _f).reshape(-1, 3)
    rgb = np.full_like(xyz, -1) if rgb is None else np.asarray(rgb, _f).reshape(-1, 3)
    return np.concatenate([xyz, tnormals.set_normal(normals), rgb], 1)


def expected_cloud(out):
    """the cloud VoxelGridFilter leaves, [m, 9], from Context.voxel_grid's / the port's (centroids, normals, rgb, ...)
    of the held points: the normal once more through set_normal, no colour when rgb was not passed"""
    return held(out[0], out[1], out[2])


def numpy_voxel_grid(xyz, leaf, normals=None, rgb=None, min_points=1):
    """the s4g_voxel_grid contract restated in numpy, sharing no code with the port: np.floor of the float32 product,
    a stable lexicographic order of (voxel, index), and each sum as np.cumsum (strictly left to right) over the runs of
    1024 members, then over the run sums.  Raises ValueError where the contract gives S4G_ERR_ARG."""
    X = np.asarray(xyz, _f).reshape(-1, 3)
    n = len(X)
    s = _f(1) / _f(leaf)
    with np.errstate(over="ignore", invalid="ignore"):
        C = np.floor(X * s)
    if not ((C >= -2.0 ** 31) & (C < 2.0 ** 31)).all():
        raise ValueError("invalid coordinate")
    C = C.astype(np.int64)
    if n and ((C.max(0) - C.min(0)) >= 2 ** 21).any():
        raise ValueError("span")
    order = np.lexsort((np.arange(n), C[:, 2], C[:, 1], C[:, 0]))
    Cs = C[order]
    head = np.ones(n, bool)
    head[1:] = (Cs[1:] != Cs[:-1]).any(1)
    starts = np.nonzero(head)[0]
    ends = np.append(starts[1:], n)
    attrs = [a for a in (X, normals, rgb) if a is not None]
    keep = [(order[b], b, e) for b, e in zip(starts, ends) if e - b >= min_points]
    keep.sort()
    out = {k: [] for k in ("xyz", "n", "rgb", "counts", "first")}
    voxel_of = np.full(n, -1, np.int32)

    def ordered_sum(v):
        runs = [np.cumsum(np.concatenate([[0.0], v[r:r + 1024]]))[-1] for r in range(0, len(v), 1024)]
        return np.cumsum(np.concatenate([[0.0], runs]))[-1]

    for o, (first, b, e) in enumerate(keep):
        members = order[b:e]
        m = e - b
        S = [np.array([ordered_sum(np.asarray(a, _f).reshape(-1, 3)[members, c].astype(np.float64)) for c in range(3)])
             for a in attrs]
        out["xyz"].append((S[0] / m).astype(_f))
        if normals is not None:
            Sn = S[1]
            ln = np.sqrt((Sn[0] * Sn[0] + Sn[1] * Sn[1]) + Sn[2] * Sn[2])
            out["n"].append(np.zeros(3, _f) if ln == 0 else (Sn / ln).astype(_f))
        if rgb is not None:
            out["rgb"].append((S[-1] / m).astype(_f))
        out["counts"].append(m)
        out["first"].append(first)
        voxel_of[members] = o
    arr = lambda k: np.asarray(out[k], _f).reshape(-1, 3)  # noqa: E731
    return (arr("xyz"), arr("n") if normals is not None else None, arr("rgb") if rgb is not None else None,
            np.asarray(out["counts"], np.int32), np.asarray(out["first"], np.int32), voxel_of)


def cloud(n, points_per_voxel, seed=0, offset=0.0):
    """n points uniform in a cube, with the leaf that puts about points_per_voxel of them in a voxel; normals of random
    directions all in the upper hemisphere, rgb in [0, 1]: (xyz, normals, rgb, leaf)"""
    rng = np.random.RandomState(seed)
    X = (rng.random_sample((n, 3)) + offset).astype(_f)
    N = rng.normal(0, 1, (n, 3))
    N[:, 2] = np.abs(N[:, 2]) + 0.1
    N = (N / np.linalg.norm(N, axis=1, keepdims=True)).astype(_f)
    R = rng.random_sample((n, 3)).astype(_f)
    leaf = float((points_per_voxel / max(n, 1)) ** (1.0 / 3.0))
    return X, N, R, leaf
