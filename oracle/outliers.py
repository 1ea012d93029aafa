"""TEST INFRASTRUCTURE ONLY: the oracle of s4g_statistical_outliers and s4g_radius_outliers (include/s4g.h).

* `statistical`, `radius` -- oracle/liboracle_outliers.so (oracle/outliers_port.cc + the brute force of
                             oracle/knn_port.cc): both contracts restated operation for operation, so that they equal the
                             device bit for bit.  `mean_rows`, `moments` and `flags` are the statistical filter's three
                             steps on their own, for clouds too large for a brute force over every row.
* `scipy_statistical`     -- an independent check of the statistical filter: scipy's cKDTree and numpy in float64.

The reference has no outlier removal; its kd-tree's range query (oracle.range.RefRange) is the reference side of the
radius filter's counts."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32


def _L():
    L = _lib(_build.port_lib("outliers"))
    L.outlier_mean_rows.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_int, C.c_void_p]
    L.outlier_moments.argtypes = [C.c_void_p, C.c_long, C.c_void_p]
    L.outlier_flags.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_double, C.c_void_p]
    L.radius_port.argtypes = [C.c_void_p, C.c_long, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _cloud(P):
    return np.ascontiguousarray(P, _f).reshape(-1, 3)


def mean_rows(P, k, which=None):
    """-> mean_dist [n] float64 of the P points `which` (default all)"""
    P = _cloud(P)
    which = None if which is None else np.ascontiguousarray(which, np.int64).reshape(-1)
    n = len(P) if which is None else len(which)
    out = np.empty(n, np.float64)
    _L().outlier_mean_rows(_p(P), len(P), _p(which), n, int(k), _p(out))
    return out


def moments(mean_dist):
    """-> (mu, sigma) of a full mean_dist array, in the contract's summation order"""
    m = np.ascontiguousarray(mean_dist, np.float64)
    out = np.empty(2, np.float64)
    _L().outlier_moments(_p(m), len(m), _p(out))
    return float(out[0]), float(out[1])


def flags(mean_dist, mu, sigma, std_ratio):
    m = np.ascontiguousarray(mean_dist, np.float64)
    out2 = np.array([mu, sigma], np.float64)
    f = np.empty(len(m), np.uint8)
    _L().outlier_flags(_p(m), len(m), _p(out2), float(std_ratio), _p(f))
    return f.astype(bool)


def statistical(P, k, std_ratio):
    """-> (keep [n_kept] int32 ascending, mean_dist [n] float64, mu, sigma)"""
    mean = mean_rows(P, k)
    mu, sigma = moments(mean)
    keep = np.nonzero(flags(mean, mu, sigma, std_ratio))[0].astype(np.int32)
    return keep, mean, mu, sigma


def radius(P, sq_radius, min_neighbors, raw=False):
    """-> (keep [n_kept] int32 ascending, counts [n] int32 capped at min_neighbors); raw=True: also the uncapped counts
    [n] int64"""
    P = _cloud(P)
    n = len(P)
    r, counts, f = np.empty(n, np.int64), np.empty(n, np.int32), np.empty(n, np.uint8)
    _L().radius_port(_p(P), n, float(sq_radius), int(min_neighbors), _p(r), _p(counts), _p(f))
    keep = np.nonzero(f)[0].astype(np.int32)
    return (keep, counts, r) if raw else (keep, counts)


def scipy_statistical(P, k, std_ratio, workers=-1):
    """-> (mask [n] bool, mean_dist [n] float64, mu, sigma): scipy cKDTree's k + 1 nearest (self dropped) on the float64
    points, numpy's mean and sample standard deviation"""
    from scipy.spatial import cKDTree
    X = np.asarray(P, np.float64).reshape(-1, 3)
    m = min(k, len(X) - 1)
    if m == 0:
        return np.ones(len(X), bool), np.zeros(len(X)), 0.0, 0.0
    d, _ = cKDTree(X).query(X, m + 1, workers=workers)
    mean = d[:, 1:].mean(1)
    mu, sigma = float(mean.mean()), float(mean.std(ddof=1)) if len(X) > 1 else 0.0
    return mean <= mu + std_ratio * sigma, mean, mu, sigma
