"""TEST INFRASTRUCTURE ONLY: the oracles of s4g_verify_nearest (include/s4g.h), the nearest P point within delta of every
transformed Q point.

* `bruteforce`  -- oracle/liboracle_nearest.so (oracle/nearest_port.cc): all P points, the contract of s4g.h;
* `RefNearest`  -- oracle/_ref/liboracle_ref_nearest.so (oracle/nearest_ref.cc): the UNMODIFIED reference's own kd-tree
                   query, linked against oracle/_ref/liboracle_ref.so; built where the reference is present and
                   travelling with oracle/_ref otherwise."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32


def bruteforce(P, Q, delta, T16):
    """-> (index [K, nQ] int32, sq_dist [K, nQ] float32, counts [K] uint32) over the centred clouds P, Q"""
    L = _lib(_build.port_lib("nearest"))
    L.nearest_bruteforce.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_float, C.c_void_p, C.c_long,
                                     C.c_void_p, C.c_void_p, C.c_void_p]
    P, Q = np.ascontiguousarray(P, _f).reshape(-1, 3), np.ascontiguousarray(Q, _f).reshape(-1, 3)
    T16 = np.ascontiguousarray(T16, _f).reshape(-1, 16)
    K = len(T16)
    index, sq, counts = np.empty((K, len(Q)), np.int32), np.empty((K, len(Q)), _f), np.empty(K, np.uint32)
    L.nearest_bruteforce(_p(P), len(P), _p(Q), len(Q), float(delta), _p(T16), K, _p(index), _p(sq), _p(counts))
    return index, sq, counts


def ref_available():
    return _build.ref_lib("nearest") is not None


class RefNearest:
    """The reference's matcher after init(P, Q) with every point kept; `sampled()` = its centred clouds, `query(T16)` =
    (index [K, nQ] int32, sq_dist [K, nQ] float32) of its kd-tree for the query Verify builds (-1 / +inf: none)"""

    def __init__(self, P, Q, delta):
        path = _build.ref_lib("nearest")
        if path is None:
            raise RuntimeError("reference oracle not available (no reference sources and no prebuilt "
                               "oracle/_ref/liboracle_ref_nearest.so)")
        L = self._L = _lib(path)
        L.nearest_ref_create.restype = C.c_void_p
        L.nearest_ref_create.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_float]
        L.nearest_ref_destroy.argtypes = [C.c_void_p]
        L.nearest_ref_sampled.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.nearest_ref_query.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_void_p]
        P, Q = np.ascontiguousarray(P, _f).reshape(-1, 3), np.ascontiguousarray(Q, _f).reshape(-1, 3)
        self.nP, self.nQ = len(P), len(Q)
        self.h = L.nearest_ref_create(_p(P), self.nP, _p(Q), self.nQ, float(delta))

    def close(self):
        if self.h:
            self._L.nearest_ref_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sampled(self):
        P, Q = np.empty((self.nP, 3), _f), np.empty((self.nQ, 3), _f)
        self._L.nearest_ref_sampled(self.h, _p(P), _p(Q))
        return P, Q

    def query(self, T16):
        T16 = np.ascontiguousarray(T16, _f).reshape(-1, 16)
        K = len(T16)
        index, sq = np.empty((K, self.nQ), np.int32), np.empty((K, self.nQ), _f)
        self._L.nearest_ref_query(self.h, _p(T16), K, _p(index), _p(sq))
        return index, sq
