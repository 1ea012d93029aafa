"""TEST INFRASTRUCTURE ONLY: the oracle of s4g_voxel_grid (include/s4g.h).

* `port` -- oracle/liboracle_voxel_grid.so (oracle/voxel_grid_port.cc): the contract restated operation for operation, so
            that it equals the device bit for bit.

The reference has no voxel-grid filter; its UniformDistSampler (s4g_voxel_sample) keeps the first point of the same
voxels, which is the `first` output at min_points = 1."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32


class VoxelGridError(ValueError):
    """the port's S4G_ERR_ARG: bad arguments, a non-finite or out-of-range coordinate, or too wide a span"""


def _L():
    L = _lib(_build.port_lib("voxel_grid"))
    L.voxel_grid_port.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_long, C.c_float, C.c_int] + [C.c_void_p] * 7
    L.voxel_grid_port.restype = C.c_int
    return L


def port(xyz, leaf, normals=None, rgb=None, min_points=1):
    """-> (centroids [m, 3], normals [m, 3] or None, rgb [m, 3] or None, counts [m], first [m], voxel_of [n]), as
    Context.voxel_grid; raises VoxelGridError where the device returns S4G_ERR_ARG"""
    X = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    N = None if normals is None else np.ascontiguousarray(normals, _f).reshape(-1, 3)
    R = None if rgb is None else np.ascontiguousarray(rgb, _f).reshape(-1, 3)
    n = len(X)
    out = np.empty((n, 3), _f)
    nout = None if N is None else np.empty((n, 3), _f)
    rout = None if R is None else np.empty((n, 3), _f)
    counts, first, voxel_of = np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n, np.int32)
    m = np.zeros(1, np.int64)
    rc = _L().voxel_grid_port(_p(X), _p(N), _p(R), n, float(leaf), int(min_points), _p(out), _p(nout), _p(rout),
                              _p(counts), _p(first), _p(voxel_of), _p(m))
    if rc != 0:
        raise VoxelGridError("voxel_grid_port: rc %d" % rc)
    k = int(m[0])
    cut = lambda a: None if a is None else a[:k].copy()  # noqa: E731
    return out[:k].copy(), cut(nout), cut(rout), counts[:k].copy(), first[:k].copy(), voxel_of
