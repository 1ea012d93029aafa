"""TEST INFRASTRUCTURE ONLY: the oracle of s4g_euclidean_clusters (include/s4g.h).

* `clusters`        -- oracle/liboracle_clusters.so (oracle/clusters_port.cc): the contract restated -- every pair tested
                       in the device's fp32 operation order, a sequential union-find, the same ordering and CSR rules --
                       so that it equals the device bit for bit.
* `roots_from_lists`, `finish` -- the same union-find over given neighbour lists (e.g. s4g_range's, or the reference
                       kd-tree's) and the same ordering rules over a given component map, for clouds too large for the
                       brute force.
* `scipy_roots`     -- an independent check: scipy's cKDTree.query_pairs + csgraph.connected_components in float64.

The reference has no clustering; its kd-tree's range query (oracle.range.RefRange) is the reference side of the graph."""
import ctypes as C

import numpy as np

from . import _build
from ._build import _lib, _p

_f = np.float32


def _L():
    L = _lib(_build.port_lib("clusters"))
    L.clusters_root_bruteforce.argtypes = [C.c_void_p, C.c_long, C.c_float, C.c_void_p]
    L.clusters_root_from_lists.argtypes = [C.c_long, C.c_void_p, C.c_void_p, C.c_void_p]
    L.clusters_finish.argtypes = [C.c_long, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _max(max_size):
    return 2 ** 31 - 1 if max_size is None else int(max_size)


def roots(P, sq_radius):
    """-> root [n] int32: the smallest index of each point's component of d^2 < sq_radius, every pair tested"""
    P = np.ascontiguousarray(P, _f).reshape(-1, 3)
    root = np.empty(len(P), np.int32)
    _L().clusters_root_bruteforce(_p(P), len(P), float(sq_radius), _p(root))
    return root


def roots_from_lists(n, offsets, indices):
    """-> root [n] int32 of the graph with the edges (j, indices[offsets[j]:offsets[j + 1]])"""
    offsets = np.ascontiguousarray(offsets, np.int64)
    indices = np.ascontiguousarray(indices, np.int32)
    root = np.empty(int(n), np.int32)
    _L().clusters_root_from_lists(int(n), _p(offsets), _p(indices), _p(root))
    return root


def finish(root, min_size=1, max_size=None):
    """-> (labels [n] int32, offsets [n_clusters + 1] int64, members [offsets[-1]] int32) of a component map"""
    root = np.ascontiguousarray(root, np.int32)
    n = len(root)
    labels, offsets, members = np.empty(n, np.int32), np.zeros(n + 1, np.int64), np.empty(n, np.int32)
    nc = C.c_int64(0)
    _L().clusters_finish(n, _p(root), int(min_size), _max(max_size), _p(labels), C.byref(nc), _p(offsets), _p(members))
    nc = nc.value
    return labels, offsets[:nc + 1].copy(), members[:offsets[nc]].copy()


def clusters(P, sq_radius, min_size=1, max_size=None):
    """-> (labels, root, offsets, members): the contract of s4g_euclidean_clusters (Context.euclidean_clusters' form)"""
    root = roots(P, sq_radius)
    labels, offsets, members = finish(root, min_size, max_size)
    return labels, root, offsets, members


def canonical_roots(component_labels):
    """any component labelling [n] -> the smallest index of each point's component"""
    lab = np.asarray(component_labels).reshape(-1)
    first = np.full(lab.max() + 1 if len(lab) else 0, len(lab), np.int64)
    np.minimum.at(first, lab, np.arange(len(lab)))
    return first[lab].astype(np.int32)


def scipy_roots(P, radius, workers=-1):
    """-> root [n] int32 of the graph |p_i - p_j| < radius (the ball's interior) in float64: cKDTree.query_pairs (which
    takes pairs at distance <= r, so r is stepped down to the next double below) + connected_components"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    from scipy.spatial import cKDTree
    X = np.asarray(P, np.float64).reshape(-1, 3)
    n = len(X)
    pairs = cKDTree(X).query_pairs(float(np.nextafter(radius, 0.0)), output_type="ndarray")
    g = coo_matrix((np.ones(len(pairs), np.int8), (pairs[:, 0], pairs[:, 1])), shape=(n, n))
    _, lab = connected_components(g, directed=False)
    return canonical_roots(lab)
