"""TEST INFRASTRUCTURE ONLY: the oracle of s4g_fpfh and s4g_fpfh_match (include/s4g.h), FPFH descriptors from k-nearest
neighbourhoods and the nearest descriptor.

* `port`       -- oracle/liboracle_fpfh.so (oracle/fpfh_port.cc + the brute force of oracle/knn_port.cc): the contract
                  restated operation for operation in double, compiled without contraction, so that it equals the device
                  bit for bit.  For clouds too large for the brute force, the rows and their d^2 can be given (e.g.
                  s4g_knn's, which tests/test_knn_gpu.py holds to the brute force).
* `match_port` -- the nearest descriptor by a plain loop over every pair.

The reference computes no descriptors, so there is no reference-side library."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32


class FPFHError(ValueError):
    """the port's S4G_ERR_ARG"""


def _L():
    L = _lib(_build.port_lib("fpfh"))
    L.fpfh_port.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                            C.c_void_p]
    L.fpfh_port.restype = C.c_int
    L.fpfh_match_port.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_void_p, C.c_void_p]
    L.fpfh_match_port.restype = None
    return L


def port(P, normals, k, sq_radius=np.inf, rows=None, sq=None, spfh=False):
    """-> fpfh [n, 33] float32 (and the SPFH [n, 33] float64 with spfh=True), Context.fpfh's form.  rows / sq: [n, k]
    knn rows with self-exclusion and their d^2 to use instead of the brute force.  Raises FPFHError where the contract
    gives S4G_ERR_ARG."""
    P = np.ascontiguousarray(P, _f).reshape(-1, 3)
    n = len(P)
    N = np.ascontiguousarray(normals, _f).reshape(-1, 3)
    if len(N) != n:
        raise FPFHError("one normal per point")
    R = None if rows is None else np.ascontiguousarray(rows, np.int32).reshape(n, int(k))
    S = None if sq is None else np.ascontiguousarray(sq, _f).reshape(n, int(k))
    out = np.empty((n, 33), _f)
    sp = np.empty((n, 33), np.float64) if spfh else None
    if _L().fpfh_port(_p(P), n, _p(N), int(k), float(sq_radius), _p(R), _p(S), _p(out), _p(sp)) == 2:
        raise FPFHError("bad arguments")
    return (out, sp) if spfh else out


def match_port(a, b, mutual=False):
    """-> (index [n_a] int32, sq_dist [n_a] float32), Context.fpfh_match's form"""
    A = np.ascontiguousarray(a, _f).reshape(-1, 33)
    B = np.ascontiguousarray(b, _f).reshape(-1, 33)
    index, sq = np.empty(len(A), np.int32), np.empty(len(A), _f)
    _L().fpfh_match_port(_p(A), len(A), _p(B), len(B), int(bool(mutual)), _p(index), _p(sq))
    return index, sq
