"""Builds and runs tests/cpp/outliers_main.cc, the test program of Utils::RemoveStatisticalOutliers and
Utils::RemoveRadiusOutliers, for tests/test_outliers_cpu.py (on the oracle stand-in) and tests/test_outliers_gpu.py (on the
real library).  Also the rules of the grid delta of the two functions, and a cloud of surface points and uniform outliers whose labels are
known."""
import numpy as np

from tests import cpp_main, normals as tnormals

_f = np.float32


def build(outdir):
    return cpp_main.build("outliers_main", outdir)


def run(exe, workdir, xyz, normals, rgb, mode, a, b, preload=None):
    """mode 'statistical' (a = k, b = std_ratio) or 'radius' (a = radius, b = min_neighbors) -> None when the call threw,
    else (returned count, points [m, 9] float32: position, normal, rgb of each point left, as Point3D holds them)"""
    xyz = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    blob = np.concatenate([xyz, np.asarray(normals, _f).reshape(-1, 3), np.asarray(rgb, _f).reshape(-1, 3)])
    payload = np.int32(len(xyz)).tobytes() + np.ascontiguousarray(blob, _f).tobytes()
    r = cpp_main.Reader(cpp_main.run(exe, workdir, payload, [mode, repr(a), repr(b)], preload))
    if r.take(np.int32, 1)[0]:
        return None
    count, m = r.take(np.int32, 2)
    return int(count), r.take(_f, 9 * int(m)).reshape(-1, 9)


def held(xyz, normals, rgb):
    """[n, 9] float32: what the program's Point3D hold before any filter (the normal through set_normal)"""
    return np.concatenate([np.asarray(xyz, _f).reshape(-1, 3), tnormals.set_normal(normals), np.asarray(rgb, _f)], 1)


def grid_delta(xyz, k):
    """the delta of RemoveStatisticalOutliers' grid: EstimateNormals' rule"""
    return tnormals.grid_delta(xyz, k)


def radius_delta(xyz, radius, min_neighbors):
    """the delta of RemoveRadiusOutliers' grid: radius / 2.02 (float32), or EstimateNormals' rule with k = min_neighbors
    when that is not a positive finite number"""
    d = np.float32(radius) / np.float32(2.02)
    return float(d) if np.isfinite(d) and d > 0 else tnormals.grid_delta(xyz, min_neighbors)


def labelled_pair(n=20000, overlap=0.6, noise_sigma=0.005, outlier_frac=0.2, seed=43):
    """cfg3's recipe (synth.make_pair: Gaussian noise on Q, a share `outlier_frac` of each cloud uniform over its
    bounding box, shuffled) with the labels kept, which make_pair's shuffle loses: dict(P, Q, out_P, out_Q), out_* [n]
    bool = the point is one of the uniform outliers"""
    from super4pcs_b200 import synth
    rng = np.random.RandomState(seed)
    n_out = int(round(outlier_frac * n))
    d = synth.make_pair(n - n_out, overlap, seed=seed, noise_sigma=noise_sigma)
    out = {}
    for key in ("P", "Q"):
        X = d[key].astype(np.float64)
        lo, hi = X.min(0), X.max(0)
        X = np.concatenate([X, lo + rng.random_sample((n_out, 3)) * (hi - lo)])
        label = np.arange(n) >= n - n_out
        perm = rng.permutation(n)
        out[key], out["out_" + key] = X[perm].astype(_f), label[perm]
    return out
