"""TEST INFRASTRUCTURE ONLY: the oracles of s4g_nearest (include/s4g.h), the restricted closest-point query of the
reference's kd-tree at any radius, for arbitrary query points, and of Match4PCSBase::MeanDistance.

* `bruteforce`     -- oracle/liboracle_nearest_any.so (oracle/nearest_any_port.cc): all P points, the contract of s4g.h;
* `RefNearestAny`  -- oracle/_ref/liboracle_ref_nearest_any.so (oracle/nearest_any_ref.cc): the UNMODIFIED reference's
                      own kd-tree query and P_mean_distance_, linked against oracle/_ref/liboracle_ref.so; built where the
                      reference is present and travelling with oracle/_ref otherwise.
* `mean_distance`  -- the reference's MeanDistance restated on the brute force's indices."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32


def ref_available():
    return _build.ref_lib("nearest_any") is not None


def bruteforce(P, X, sq_radius=np.inf, T16=None, exclude=None):
    """-> (index [n] int32, sq_dist [n] float32): the s4g_nearest contract over all of P"""
    L = _lib(_build.port_lib("nearest_any"))
    L.nearest_any_bruteforce.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_void_p, C.c_float, C.c_void_p,
                                         C.c_void_p, C.c_void_p]
    P, X = np.ascontiguousarray(P, _f).reshape(-1, 3), np.ascontiguousarray(X, _f).reshape(-1, 3)
    T16 = None if T16 is None else np.ascontiguousarray(T16, _f).reshape(16)
    exclude = None if exclude is None else np.ascontiguousarray(exclude, np.int32).reshape(len(X))
    index, sq = np.empty(len(X), np.int32), np.empty(len(X), _f)
    L.nearest_any_bruteforce(_p(P), len(P), _p(X), len(X), _p(T16), float(sq_radius), _p(exclude), _p(index), _p(sq))
    return index, sq


def mean_distance(P, index):
    """MeanDistance (match4pcsBase.cc:158-182) from the neighbour of every sampled-P point: the fp32 norms
    sqrt(dx^2 + (dy^2 + dz^2)) of p_i - p_index[i], summed in index order in fp32, divided by their number (0/0 -> NaN)"""
    P = np.ascontiguousarray(P, _f).reshape(-1, 3)
    hit = np.nonzero(index >= 0)[0]
    d = (P[hit] - P[index[hit]]).astype(_f)
    norms = np.sqrt((d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])).astype(_f)).astype(_f)
    total = np.cumsum(norms, dtype=_f)[-1] if len(norms) else _f(0)
    with np.errstate(invalid="ignore", divide="ignore"):
        return _f(_f(total) / _f(len(norms)))


class RefNearestAny:
    """The reference's matcher after init(P, Q): `sampled()` = its centred clouds, `query(...)` = its kd-tree's
    restricted closest-point query, `diameter_and_mean_distance()` = (P_diameter_, P_mean_distance_).  sample_size <= 0
    keeps every point; otherwise the reference's own sampler runs with that size and configureOverlap(overlap)."""

    def __init__(self, P, Q, delta, overlap=1.0, sample_size=0):
        path = _build.ref_lib("nearest_any")
        if path is None:
            raise RuntimeError("reference oracle not available (no reference sources and no prebuilt "
                               "oracle/_ref/liboracle_ref_nearest_any.so)")
        L = self._L = _lib(path)
        L.nearest_any_ref_create.restype = C.c_void_p
        L.nearest_any_ref_create.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_long]
        L.nearest_any_ref_destroy.argtypes = [C.c_void_p]
        L.nearest_any_ref_sizes.argtypes = [C.c_void_p, C.c_void_p]
        L.nearest_any_ref_sampled.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.nearest_any_ref_mean_distance.argtypes = [C.c_void_p, C.c_void_p]
        L.nearest_any_ref_query.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p, C.c_float, C.c_void_p,
                                            C.c_void_p, C.c_void_p]
        P, Q = np.ascontiguousarray(P, _f).reshape(-1, 3), np.ascontiguousarray(Q, _f).reshape(-1, 3)
        self.h = L.nearest_any_ref_create(_p(P), len(P), _p(Q), len(Q), float(delta), float(overlap), int(sample_size))
        n = np.zeros(2, np.int64)
        L.nearest_any_ref_sizes(self.h, _p(n))
        self.nP, self.nQ = int(n[0]), int(n[1])

    def close(self):
        if self.h:
            self._L.nearest_any_ref_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def sampled(self):
        P, Q = np.empty((self.nP, 3), _f), np.empty((self.nQ, 3), _f)
        self._L.nearest_any_ref_sampled(self.h, _p(P), _p(Q))
        return P, Q

    def diameter_and_mean_distance(self):
        o = np.zeros(2, _f)
        self._L.nearest_any_ref_mean_distance(self.h, _p(o))
        return o[0], o[1]

    def query(self, X, sq_radius=np.inf, T16=None, exclude=None):
        X = np.ascontiguousarray(X, _f).reshape(-1, 3)
        T16 = None if T16 is None else np.ascontiguousarray(T16, _f).reshape(16)
        exclude = None if exclude is None else np.ascontiguousarray(exclude, np.int32).reshape(len(X))
        index, sq = np.empty(len(X), np.int32), np.empty(len(X), _f)
        self._L.nearest_any_ref_query(self.h, _p(X), len(X), _p(T16), float(sq_radius), _p(exclude), _p(index), _p(sq))
        return index, sq
