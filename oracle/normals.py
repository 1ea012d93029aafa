"""TEST INFRASTRUCTURE ONLY: the oracle of s4g_normals (include/s4g.h), PCA normals of k-nearest neighbourhoods.

* `port`  -- oracle/liboracle_normals.so (oracle/normals_port.cc + the brute force of oracle/knn_port.cc): the contract
             restated operation for operation, so that it equals the device bit for bit.
* `eigh`  -- an independent check of the same rows: numpy float64 np.linalg.eigh of their covariance.

The reference has no normal estimation (its kd-tree has no k-nearest query), so there is no reference-side library."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32


def port(P, k, sq_radius=np.inf, viewpoint=None, which=None, rows=False):
    """-> (normals [n, 3], eigenvalues [n, 3]) float32 of the P points `which` (default all, n = len(P)); rows=True: also
    their knn rows [n, k] int32"""
    L = _lib(_build.port_lib("normals"))
    L.normals_port.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                               C.c_void_p, C.c_void_p]
    P = np.ascontiguousarray(P, _f).reshape(-1, 3)
    which = None if which is None else np.ascontiguousarray(which, np.int64).reshape(-1)
    n = len(P) if which is None else len(which)
    vp = None if viewpoint is None else np.ascontiguousarray(viewpoint, _f).reshape(3)
    normals, eig = np.empty((n, 3), _f), np.empty((n, 3), _f)
    R = np.empty((n, k), np.int32) if rows else None
    L.normals_port(_p(P), len(P), _p(which), n, int(k), float(sq_radius), _p(vp), _p(normals), _p(eig), _p(R))
    return (normals, eig, R) if rows else (normals, eig)


def eigh(P, rows):
    """-> (eigenvalues [n, 3] ascending, eigenvectors [n, 3, 3] (columns), m [n]): float64 np.linalg.eigh of the
    covariance sum (p - c)(p - c)^T / m of each row's real entries"""
    P = np.asarray(P, np.float64)
    n, k = rows.shape
    m = (rows >= 0).sum(1)
    pts = P[np.where(rows >= 0, rows, 0)]
    w = (rows >= 0)[..., None].astype(np.float64)
    c = (pts * w).sum(1) / np.maximum(m, 1)[:, None]
    d = (pts - c[:, None, :]) * w
    cov = np.einsum("nki,nkj->nij", d, d) / np.maximum(m, 1)[:, None, None]
    val, vec = np.linalg.eigh(cov)
    return val, vec, m
