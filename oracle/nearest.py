"""TEST INFRASTRUCTURE ONLY: the oracles of s4g_verify_nearest (include/s4g.h), the nearest P point within delta of every
transformed Q point.

* `bruteforce`  -- oracle/liboracle_nearest.so (oracle/nearest_port.cc): all P points, the contract of s4g.h;
* `RefNearest`  -- oracle/_ref/liboracle_ref_nearest.so (oracle/nearest_ref.cc): the UNMODIFIED reference's own kd-tree
                   query, linked against oracle/_ref/liboracle_ref.so; built where the reference is present and
                   travelling with oracle/_ref otherwise."""
import ctypes as C
import os
import subprocess

import numpy as np

from . import _build

HERE = _build.HERE
PORT_SRC = os.path.join(HERE, "nearest_port.cc")
PORT_SO = os.path.join(HERE, "liboracle_nearest.so")
REF_SRC = os.path.join(HERE, "nearest_ref.cc")
REF_SO = os.path.join(HERE, "_ref", "liboracle_ref_nearest.so")
_f = np.float32
_libs = {}


def _env():
    env = dict(os.environ)
    env.pop("CXX", None)
    env.pop("CC", None)
    return env


def build_port(force=False):
    if force or _build._stale(PORT_SO, [PORT_SRC]):
        subprocess.check_call(["g++", "-std=c++11", "-O2", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared", PORT_SRC,
                               "-o", PORT_SO], env=_env())
    return PORT_SO


def build_ref(force=False):
    """the path of the reference-side library, or None when it can be neither built (no reference sources) nor found"""
    ref = _build.REFERENCE_ROOT
    base = _build.build_ref()
    if base is not None and os.path.isdir(os.path.join(ref, "src", "super4pcs")) and \
            (force or _build._stale(REF_SO, [REF_SRC, base])):
        # the flags of oracle/Makefile's reference build (the reference's Release configuration)
        subprocess.check_call(["g++", "-std=c++11", "-O3", "-DNDEBUG", "-fopenmp", "-DSUPER4PCS_USE_OPENMP",
                               "-DEIGEN_DONT_PARALLELIZE", "-I", os.path.join(ref, "src"),
                               "-I", os.path.join(ref, "3rdparty", "Eigen"), "-fPIC", "-w", "-shared", REF_SRC,
                               "-o", REF_SO, "-L", os.path.dirname(base), "-loracle_ref", "-Wl,-rpath,$ORIGIN"],
                              env=_env())
    return REF_SO if os.path.exists(REF_SO) else None


def build():
    build_port()
    build_ref()


def _lib(path):
    if path not in _libs:
        _libs[path] = C.CDLL(path)
    return _libs[path]


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def bruteforce(P, Q, delta, T16):
    """-> (index [K, nQ] int32, sq_dist [K, nQ] float32, counts [K] uint32) over the centred clouds P, Q"""
    L = _lib(build_port())
    L.nearest_bruteforce.argtypes = [C.c_void_p, C.c_long, C.c_void_p, C.c_long, C.c_float, C.c_void_p, C.c_long,
                                     C.c_void_p, C.c_void_p, C.c_void_p]
    P, Q = np.ascontiguousarray(P, _f).reshape(-1, 3), np.ascontiguousarray(Q, _f).reshape(-1, 3)
    T16 = np.ascontiguousarray(T16, _f).reshape(-1, 16)
    K = len(T16)
    index, sq, counts = np.empty((K, len(Q)), np.int32), np.empty((K, len(Q)), _f), np.empty(K, np.uint32)
    L.nearest_bruteforce(_p(P), len(P), _p(Q), len(Q), float(delta), _p(T16), K, _p(index), _p(sq), _p(counts))
    return index, sq, counts


def ref_available():
    return build_ref() is not None


class RefNearest:
    """The reference's matcher after init(P, Q) with every point kept; `sampled()` = its centred clouds, `query(T16)` =
    (index [K, nQ] int32, sq_dist [K, nQ] float32) of its kd-tree for the query Verify builds (-1 / +inf: none)"""

    def __init__(self, P, Q, delta):
        path = build_ref()
        if path is None:
            raise RuntimeError("reference oracle not available (no reference sources and no prebuilt %s)" % REF_SO)
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
