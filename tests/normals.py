"""Builds and runs tests/cpp/normals_main.cc, the test program of Utils::EstimateNormals, for tests/test_normals_cpu.py
(on the oracle stand-in) and tests/test_normals_gpu.py (on the real library).  Also the float32 arithmetic of
Point3D::set_normal, which EstimateNormals stores its normals through, and the rule of its grid's delta."""
import numpy as np

from tests import cpp_main

ROOT = cpp_main.ROOT
_f = np.float32


def build(outdir):
    return cpp_main.build("normals_main", outdir)


def run(exe, workdir, xyz, k, max_distance=np.inf, viewpoint=None, preload=None):
    """-> None when EstimateNormals threw, else (returned count, normals [n, 3] float32 as the points hold them)"""
    xyz = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    args = [str(int(k)), repr(float(max_distance))]
    if viewpoint is not None:
        args += [repr(float(v)) for v in np.asarray(viewpoint, _f)]
    r = cpp_main.Reader(cpp_main.run(exe, workdir, np.int32(len(xyz)).tobytes() + xyz.tobytes(), args, preload))
    if r.take(np.int32, 1)[0]:
        return None
    return int(r.take(np.int32, 1)[0]), r.take(_f, 3 * len(xyz)).reshape(-1, 3)


def set_normal(n):
    """Point3D::set_normal (Eigen's normalized()) in float32: n / sqrt(x^2 + (y^2 + z^2)) when that is > 0, else n"""
    n = np.asarray(n, _f)
    sq = n[:, 0] * n[:, 0] + (n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2])
    out = n.copy()
    pos = sq > 0
    out[pos] = n[pos] / np.sqrt(sq[pos])[:, None]
    return out


def grid_delta(xyz, k):
    """the delta EstimateNormals builds its grid with: 0.5 E sqrt(k / n), E the largest edge of the bounding box; 1 when
    E is 0"""
    xyz = np.asarray(xyz, _f)
    E = float((xyz.max(0).astype(np.float64) - xyz.min(0).astype(np.float64)).max())
    d = np.float32(0.5 * E * np.sqrt(k / len(xyz)))
    return float(d) if d > 0 else 1.0
