"""TEST INFRASTRUCTURE ONLY: the oracle of s4g_knn (include/s4g.h), the k nearest P points within a radius of any query
points.

* `bruteforce`   -- oracle/liboracle_knn.so (oracle/knn_port.cc): all P points, the contract of s4g.h;
* `from_range`   -- the contract restated on a range query's CSR lists: the first k of each list at
                    nextafterf(sq_radius, +inf), exclude removed, ordered by (d^2, index).  Given the lists of the
                    reference's own kd-tree (oracle.range.RefRange), it ties the brute force to the reference.

The reference's kd-tree has no k-nearest query, so there is no reference-side library here: the reference side reuses
oracle.range.RefRange and oracle.nearest_any.RefNearestAny."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32


def bruteforce(P, X, k, sq_radius=np.inf, T16=None, exclude=None):
    """-> (index [n, k] int32, sq_dist [n, k] float32): the s4g_knn contract over all of P"""
    L = _lib(_build.port_lib("knn"))
    L.knn_bruteforce.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_void_p, C.c_int, C.c_float, C.c_void_p,
                                 C.c_void_p, C.c_void_p]
    P, X = np.ascontiguousarray(P, _f).reshape(-1, 3), np.ascontiguousarray(X, _f).reshape(-1, 3)
    T16 = None if T16 is None else np.ascontiguousarray(T16, _f).reshape(16)
    exclude = None if exclude is None else np.ascontiguousarray(exclude, np.int32).reshape(len(X))
    index, sq = np.empty((len(X), k), np.int32), np.empty((len(X), k), _f)
    L.knn_bruteforce(_p(P), len(P), _p(X), len(X), _p(T16), int(k), float(sq_radius), _p(exclude), _p(index), _p(sq))
    return index, sq


def range_radius(sq_radius):
    """the range query's (strict) radius whose lists are the points with d^2 <= sq_radius: the next float above it"""
    return float(np.nextafter(np.float32(sq_radius), np.float32(np.inf)))


def from_range(lists, k, exclude=None):
    """(offsets, index, sq_dist) of a range query at range_radius(sq_radius) -> the (index [n, k], sq_dist [n, k]) rows of
    s4g_knn at sq_radius: each list without exclude[i], ordered by (d^2, index), its first k entries, padded with
    -1 / +inf"""
    off, idx, sq = lists
    n = len(off) - 1
    index, out = np.full((n, k), -1, np.int32), np.full((n, k), np.inf, _f)
    for i in range(n):
        j, d = idx[off[i]:off[i + 1]], sq[off[i]:off[i + 1]]
        if exclude is not None:
            keep = j != exclude[i]
            j, d = j[keep], d[keep]
        order = np.lexsort((j, d))[:k]
        index[i, :len(order)] = j[order]
        out[i, :len(order)] = d[order]
    return index, out
