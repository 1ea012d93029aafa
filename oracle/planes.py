"""TEST INFRASTRUCTURE ONLY: the oracle of s4g_segment_planes (include/s4g.h).

* `planes`      -- oracle/liboracle_planes.so (oracle/planes_port.cc): the contract restated operation for operation --
                   the draws, the double-precision hypothesis planes, every hypothesis tested on every active point in
                   fp32, the fixed-order refit with s4g_normals' Jacobi, the final test, accept or stop -- so that it
                   equals the device bit for bit.  Context.segment_planes' form.
* `hypotheses`, `counts` -- one round's draws and planes, and the counts of given planes, on their own.

The reference has no plane segmentation, so there is no reference side."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32

# s4g_plane (include/s4g.h), as super4pcs_b200.s4g.PLANE_DTYPE
PLANE_DTYPE = np.dtype([("coefficients", np.float32, 4), ("hypothesis", np.float32, 4), ("hypothesis_index", np.int32),
                        ("sample", np.int32, 3), ("hypothesis_inliers", np.int64), ("n_inliers", np.int64)])


def _L():
    L = _lib(_build.port_lib("planes"))
    L.planes_hypotheses.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_long, C.c_uint64, C.c_void_p, C.c_void_p,
                                    C.c_void_p]
    L.planes_counts.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_long, C.c_void_p, C.c_float, C.c_void_p]
    L.planes_port.argtypes = [C.c_void_p, C.c_long, C.c_float, C.c_int, C.c_uint64, C.c_int, C.c_int, C.c_int64,
                              C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _cloud(P):
    return np.ascontiguousarray(P, _f).reshape(-1, 3)


def hypotheses(P, active, H, seed_r):
    """-> (sample [H, 3] int32, plane [H, 4] float32 (NaN: invalid), valid [H] bool) of one round over the ascending
    positions `active`"""
    P, act = _cloud(P), np.ascontiguousarray(active, np.int32)
    sample, plane, valid = np.empty((H, 3), np.int32), np.empty((H, 4), _f), np.empty(H, np.uint8)
    _L().planes_hypotheses(_p(P), _p(act), len(act), int(H), C.c_uint64(int(seed_r) % 2 ** 64), _p(sample), _p(plane),
                           _p(valid))
    return sample, plane, valid.astype(bool)


def counts(P, active, planes, threshold):
    """-> counts [H] uint32: the points of P[active] with |((a x + b y) + c z) + d| < threshold, per plane [H, 4]"""
    P, act = _cloud(P), np.ascontiguousarray(active, np.int32)
    planes = np.ascontiguousarray(planes, _f).reshape(-1, 4)
    out = np.empty(len(planes), np.uint32)
    _L().planes_counts(_p(P), _p(act), len(act), len(planes), _p(planes), float(threshold), _p(out))
    return out


def planes(P, threshold, n_hypotheses=1000, max_planes=1, min_inliers=1, seed=0, refine=True, hyp_counts=False):
    """-> (labels, planes, offsets, members[, counts]): the contract of s4g_segment_planes (Context.segment_planes' form)"""
    P = _cloud(P)
    n, H, R = len(P), int(n_hypotheses), int(max_planes)
    labels, members = np.empty(n, np.int32), np.empty(n, np.int32)
    out, offsets = np.zeros(R, PLANE_DTYPE), np.zeros(R + 1, np.int64)
    cnt = np.empty((R, H), np.uint32) if hyp_counts else None
    k = C.c_int(0)
    _L().planes_port(_p(P), n, float(threshold), H, C.c_uint64(int(seed) % 2 ** 64), 1 if refine else 0, R,
                     int(min_inliers), _p(labels), _p(out), C.byref(k), _p(offsets), _p(members), _p(cnt))
    k = k.value
    res = (labels, out[:k].copy(), offsets[:k + 1].copy(), members[:offsets[k]].copy())
    return res + (cnt,) if hyp_counts else res
