"""TEST INFRASTRUCTURE ONLY: the oracles of s4g_range (include/s4g.h), the range query of the reference's kd-tree: every
P point closer than a radius to any query point.

* `bruteforce` -- oracle/liboracle_range.so (oracle/range_port.cc): all P points, the contract of s4g.h;
* `RefRange`   -- oracle/_ref/liboracle_ref_range.so (oracle/range_ref.cc): the UNMODIFIED reference's own kd-tree query
                  (doQueryDistIndices), each list sorted by index, linked against oracle/_ref/liboracle_ref.so; built where
                  the reference is present and travelling with oracle/_ref otherwise.

Both return CSR lists: (offsets [n + 1] int64, index [total] int32, sq_dist [total] float32)."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32


def ref_available():
    return _build.ref_lib("range") is not None


def bruteforce(P, X, sq_radius, T16=None):
    """-> (offsets, index, sq_dist): the s4g_range contract over all of P"""
    L = _lib(_build.port_lib("range"))
    args = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_void_p, C.c_float]
    L.range_bruteforce_count.argtypes = args + [C.c_void_p]
    L.range_bruteforce_fill.argtypes = args + [C.c_void_p, C.c_void_p, C.c_void_p]
    P, X = np.ascontiguousarray(P, _f).reshape(-1, 3), np.ascontiguousarray(X, _f).reshape(-1, 3)
    T16 = None if T16 is None else np.ascontiguousarray(T16, _f).reshape(16)
    offsets = np.zeros(len(X) + 1, np.int64)
    L.range_bruteforce_count(_p(P), len(P), _p(X), len(X), _p(T16), float(sq_radius), _p(offsets))
    index, sq = np.empty(int(offsets[-1]), np.int32), np.empty(int(offsets[-1]), _f)
    L.range_bruteforce_fill(_p(P), len(P), _p(X), len(X), _p(T16), float(sq_radius), _p(offsets), _p(index), _p(sq))
    return offsets, index, sq


class RefRange:
    """The reference's matcher after init(P, Q): `sampled()` = its centred clouds, `query(...)` = its kd-tree's range
    query.  sample_size <= 0 keeps every point; otherwise the reference's own sampler runs with that size and
    configureOverlap(overlap)."""

    def __init__(self, P, Q, delta, overlap=1.0, sample_size=0):
        path = _build.ref_lib("range")
        if path is None:
            raise RuntimeError("reference oracle not available (no reference sources and no prebuilt "
                               "oracle/_ref/liboracle_ref_range.so)")
        L = self._L = _lib(path)
        L.range_ref_create.restype = C.c_void_p
        L.range_ref_create.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_long]
        L.range_ref_destroy.argtypes = [C.c_void_p]
        L.range_ref_sizes.argtypes = [C.c_void_p, C.c_void_p]
        L.range_ref_sampled.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.range_ref_query.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_float, C.c_void_p]
        L.range_ref_get.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        P, Q = np.ascontiguousarray(P, _f).reshape(-1, 3), np.ascontiguousarray(Q, _f).reshape(-1, 3)
        self.h = L.range_ref_create(_p(P), len(P), _p(Q), len(Q), float(delta), float(overlap), int(sample_size))
        n = np.zeros(2, np.int64)
        L.range_ref_sizes(self.h, _p(n))
        self.nP, self.nQ = int(n[0]), int(n[1])

    def close(self):
        if self.h:
            self._L.range_ref_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sampled(self):
        P, Q = np.empty((self.nP, 3), _f), np.empty((self.nQ, 3), _f)
        self._L.range_ref_sampled(self.h, _p(P), _p(Q))
        return P, Q

    def query(self, X, sq_radius, T16=None):
        """-> (offsets, index, sq_dist) of the kd-tree, every list sorted by index"""
        X = np.ascontiguousarray(X, _f).reshape(-1, 3)
        T16 = None if T16 is None else np.ascontiguousarray(T16, _f).reshape(16)
        offsets = np.zeros(len(X) + 1, np.int64)
        self._L.range_ref_query(self.h, _p(X), len(X), _p(T16), float(sq_radius), _p(offsets))
        index, sq = np.empty(int(offsets[-1]), np.int32), np.empty(int(offsets[-1]), _f)
        self._L.range_ref_get(self.h, _p(index), _p(sq))
        return offsets, index, sq
