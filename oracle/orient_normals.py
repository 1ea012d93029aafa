"""TEST INFRASTRUCTURE ONLY: the oracle of s4g_orient_normals (include/s4g.h), normals oriented consistently along the
minimum spanning forest of the k-nearest graph.

* `port` -- oracle/liboracle_orient_normals.so (oracle/orient_normals_port.cc + the brute force of oracle/knn_port.cc):
            the contract restated with Kruskal, a sequential union-find and a breadth-first walk, so that it equals the
            device bit for bit.  For clouds too large for the brute force, the rows can be given (e.g. s4g_knn's, which
            tests/test_knn_gpu.py holds to the brute force).

The reference has no normal estimation, so there is no reference-side library."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32


class OrientError(ValueError):
    """the port's S4G_ERR_ARG: bad arguments or a non-finite normal component"""


def port(P, normals, k, sq_radius=np.inf, viewpoint=None, rows=None, out=None):
    """-> (oriented [n, 3] float32, root [n] int32, n_components, tree_edges [n_tree, 2] int32), Context.orient_normals'
    form.  rows: [n, k] int32 knn rows with self-exclusion to use instead of the brute force.  out: the array to write the
    oriented normals to (may be `normals` itself: in place).  Raises OrientError where the contract gives S4G_ERR_ARG."""
    L = _lib(_build.port_lib("orient_normals"))
    L.orient_normals_port.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.orient_normals_port.restype = C.c_int
    P = np.ascontiguousarray(P, _f).reshape(-1, 3)
    n = len(P)
    N = normals if out is not None and out is normals else np.ascontiguousarray(normals, _f).reshape(-1, 3)
    if len(N) != n:
        raise OrientError("one normal per point")
    vp = None if viewpoint is None else np.ascontiguousarray(viewpoint, _f).reshape(3)
    R = None if rows is None else np.ascontiguousarray(rows, np.int32).reshape(n, int(k))
    res = np.empty((n, 3), _f) if out is None else out
    root = np.empty(n, np.int32)
    tree = np.empty((max(n - 1, 0), 2), np.int32)
    out2 = np.zeros(2, np.int64)
    rc = L.orient_normals_port(_p(P), n, _p(N), int(k), float(sq_radius), _p(vp), _p(R), _p(res), _p(root), _p(out2),
                               _p(tree))
    if rc == 2:
        raise OrientError("bad arguments or a non-finite normal")
    assert rc == 0, "the forest does not span the components"
    return res, root, int(out2[0]), tree[:int(out2[1])].copy()
