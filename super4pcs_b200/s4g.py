"""ctypes binding of libs4g.so (include/s4g.h).  One `Context` = one GPU + the resident clouds."""
import ctypes as C
import os
import re
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_f = np.float32


class S4GError(RuntimeError):
    pass


def lib_path():
    return os.path.join(_HERE, "lib", "libs4g.so")


def header_path():
    return os.path.join(_ROOT, "include", "s4g.h")


class TcsResult(C.Structure):
    _fields_ = [("key", C.c_uint64), ("best_count", C.c_uint32), ("best_index", C.c_int32),
                ("n_gate_pass", C.c_uint32), ("n_q", C.c_uint32), ("best_T", C.c_float * 16),
                ("best_rms", C.c_float), ("centroid1", C.c_float * 3), ("centroid2", C.c_float * 3),
                ("best_quad", C.c_int32 * 4)]


class BaseDesc(C.Structure):
    _fields_ = [("pair_distance", C.c_float * 2), ("pair_normals_angle", C.c_float * 2), ("base_p", (C.c_float * 9) * 4),
                ("base_xyz_p", C.c_float * 12), ("invariant1", C.c_float), ("invariant2", C.c_float)]


class BaseResult(C.Structure):
    _fields_ = [("n_pairs", C.c_int64 * 2), ("n_quads", C.c_int64), ("tcs", TcsResult)]


class PairFilters(C.Structure):
    _fields_ = [("max_normal_difference", C.c_float), ("max_translation_distance", C.c_float),
                ("max_angle", C.c_float), ("max_color_distance", C.c_float)]


class Plane(C.Structure):
    _fields_ = [("coefficients", C.c_float * 4), ("hypothesis", C.c_float * 4), ("hypothesis_index", C.c_int32),
                ("sample", C.c_int32 * 3), ("hypothesis_inliers", C.c_int64), ("n_inliers", C.c_int64)]


# s4g_plane as a numpy record: Context.segment_planes returns an array of these, one field per struct member
PLANE_DTYPE = np.dtype([("coefficients", np.float32, 4), ("hypothesis", np.float32, 4), ("hypothesis_index", np.int32),
                        ("sample", np.int32, 3), ("hypothesis_inliers", np.int64), ("n_inliers", np.int64)])
assert PLANE_DTYPE.itemsize == C.sizeof(Plane) == 64

_lib = None


def declared_symbols():
    """names of every function include/s4g.h declares"""
    txt = open(header_path()).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(s4g_[a-z0-9_]+)\s*\(", txt)))


def exported_symbols(names=None):
    """subset of `names` (default: all declared) that the built library exports"""
    L = C.CDLL(lib_path())
    out = []
    for n in (names or declared_symbols()):
        try:
            getattr(L, n)
            out.append(n)
        except AttributeError:
            pass
    return out


def load_library():
    """Loads libs4g.so; raises (never falls back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    p = lib_path()
    if not os.path.exists(p):
        raise S4GError("CUDA extension %s is missing: run `python -c 'import __graft_entry__ as g; "
                       "g.build()'` (there is no CPU fallback)" % p)
    L = C.CDLL(p)
    vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float
    sig = {
        "s4g_abi_version": ([], i32),
        "s4g_create": ([i32, C.POINTER(vp)], i32),
        "s4g_destroy": ([vp], None),
        "s4g_error_string": ([vp], C.c_char_p),
        "s4g_set_stream": ([vp, vp], i32),
        "s4g_synchronize": ([vp], i32),
        "s4g_device_count": ([vp], i32),
        "s4g_set_cloud_p": ([vp, vp, i32, f32], i32),
        "s4g_set_cloud_q": ([vp, vp, vp, vp, i32], i32),
        "s4g_get_q_normalization": ([vp, vp], i32),
        "s4g_get_grid_stats": ([vp, vp], i32),
        "s4g_verify": ([vp, vp, i32, vp], i32),
        "s4g_verify_dev": ([vp, vp, i32, vp], i32),
        "s4g_verify_probe_stats": ([vp, vp, i32, vp], i32),
        "s4g_verify_nearest": ([vp, vp, i32, vp, vp, vp], i32),
        "s4g_verify_nearest_dev": ([vp, vp, i32, vp, vp, vp], i32),
        "s4g_nearest": ([vp, vp, i32, vp, f32, vp, vp, vp], i32),
        "s4g_nearest_dev": ([vp, vp, i32, vp, f32, vp, vp, vp], i32),
        "s4g_nearest_probe_stats": ([vp, vp, i32, vp, f32, vp, vp, vp, vp], i32),
        "s4g_knn": ([vp, vp, i32, vp, i32, f32, vp, vp, vp], i32),
        "s4g_knn_dev": ([vp, vp, i32, vp, i32, f32, vp, vp, vp], i32),
        "s4g_knn_probe_stats": ([vp, vp, i32, vp, i32, f32, vp, vp, vp, vp], i32),
        "s4g_normals": ([vp, i32, f32, vp, vp, vp], i32),
        "s4g_normals_dev": ([vp, i32, f32, vp, vp, vp], i32),
        "s4g_orient_normals": ([vp, vp, i32, f32, vp, vp, vp, vp, vp], i32),
        "s4g_orient_normals_dev": ([vp, vp, i32, f32, vp, vp, vp, vp, vp], i32),
        "s4g_fpfh": ([vp, vp, i32, f32, vp], i32),
        "s4g_fpfh_dev": ([vp, vp, i32, f32, vp], i32),
        "s4g_fpfh_match": ([vp, vp, C.c_int64, vp, C.c_int64, i32, vp, vp], i32),
        "s4g_fpfh_match_dev": ([vp, vp, C.c_int64, vp, C.c_int64, i32, vp, vp], i32),
        "s4g_statistical_outliers": ([vp, i32, C.c_double, vp, vp, vp, vp], i32),
        "s4g_statistical_outliers_dev": ([vp, i32, C.c_double, vp, vp, vp, vp], i32),
        "s4g_radius_outliers": ([vp, f32, i32, vp, vp, vp], i32),
        "s4g_radius_outliers_dev": ([vp, f32, i32, vp, vp, vp], i32),
        "s4g_euclidean_clusters": ([vp, f32, i32, i32, vp, vp, vp, vp, vp], i32),
        "s4g_euclidean_clusters_dev": ([vp, f32, i32, i32, vp, vp, vp, vp, vp], i32),
        "s4g_segment_planes": ([vp, f32, i32, C.c_uint64, i32, i32, i64, vp, C.POINTER(Plane), vp, vp, vp, vp], i32),
        "s4g_segment_planes_dev": ([vp, f32, i32, C.c_uint64, i32, i32, i64, vp, vp, vp, vp, vp, vp], i32),
        "s4g_range": ([vp, vp, i32, vp, f32, vp, vp], i32),
        "s4g_get_range": ([vp, vp, vp], i32),
        "s4g_range_count_dev": ([vp, vp, i32, vp, f32, vp], i32),
        "s4g_range_fill_dev": ([vp, vp, i32, vp, f32, vp, i64, vp, vp], i32),
        "s4g_verify_best_dev": ([vp, vp, i32, vp, vp, vp], i32),
        "s4g_verify_best": ([vp, vp, i32, vp, vp, vp], i32),
        "s4g_comm_unique_id": ([vp], i32),
        "s4g_comm_init_rank": ([vp, vp, i32, i32], i32),
        "s4g_comm_init_all": ([vp, i32], i32),
        "s4g_comm_destroy": ([vp], i32),
        "s4g_comm_info": ([vp, vp], i32),
        "s4g_comm_set_timeout": ([vp, i32], i32),
        "s4g_rigid_batch": ([vp, vp, vp, i64, f32, vp, vp, vp], i32),
        "s4g_try_congruent_set": ([vp, vp, vp, i64, f32, f32, i32, i32, C.POINTER(TcsResult)], i32),
        "s4g_try_congruent_set_dev": ([vp, vp, vp, i64, f32, f32, i32, i32, C.POINTER(TcsResult)], i32),
        "s4g_try_congruent_set_resident": ([vp, vp, f32, f32, i32, i32, C.POINTER(TcsResult)], i32),
        "s4g_extract_pairs": ([vp, f32, f32, f32, vp, vp, C.POINTER(PairFilters), i32, C.POINTER(i64)], i32),
        "s4g_get_pairs": ([vp, i32, vp], i32),
        "s4g_set_pairs": ([vp, i32, vp, i64], i32),
        "s4g_count_pairs": ([vp, f32, f32, C.POINTER(i64)], i32),
        "s4g_count_pairs_rows": ([vp, f32, f32, vp, C.POINTER(i64)], i32),
        "s4g_find_quads": ([vp, f32, f32, f32, vp, C.POINTER(i64)], i32),
        "s4g_try_bases": ([vp, vp, i32, f32, C.POINTER(PairFilters), f32, f32, f32, vp], i32),
        "s4g_get_quads": ([vp, vp], i32),
        "s4g_get_timings": ([vp, vp], i32),
        "s4g_voxel_sample": ([vp, vp, i64, f32, vp, C.POINTER(i64)], i32),
        "s4g_voxel_grid": ([vp, vp, vp, vp, i64, f32, i32, vp, vp, vp, vp, vp, vp, C.POINTER(i64)], i32),
        "s4g_voxel_grid_dev": ([vp, vp, vp, vp, i64, f32, i32, vp, vp, vp, vp, vp, vp, vp], i32),
    }
    for name, (args, res) in sig.items():
        try:
            fn = getattr(L, name)
        except AttributeError:
            continue  # reported by the symbol-export test, not here
        fn.argtypes = args
        fn.restype = res
    _lib = L
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _c(a, dt=_f):
    return None if a is None else np.ascontiguousarray(a, dtype=dt)


def _max_size(max_size):
    """the max_size argument of s4g_euclidean_clusters: None -> INT_MAX (no limit)"""
    return 2 ** 31 - 1 if max_size is None else int(max_size)


COMM_ID_BYTES = 128


def comm_unique_id():
    """ncclGetUniqueId through libs4g (rank 0 calls it and ships the bytes to its peers)"""
    buf = np.zeros(COMM_ID_BYTES, np.uint8)
    rc = load_library().s4g_comm_unique_id(_p(buf))
    if rc != 0:
        raise S4GError("s4g_comm_unique_id failed (rc %d): NCCL is not loadable in this process" % rc)
    return buf.tobytes()


def comm_init_all(contexts):
    """one process, several devices: ncclCommInitAll over the contexts (rank = position in the list)"""
    arr = (C.c_void_p * len(contexts))(*[c.h for c in contexts])
    rc = load_library().s4g_comm_init_all(arr, len(contexts))
    if rc != 0:
        raise S4GError("s4g_comm_init_all failed (rc %d): %s" % (rc, contexts[0]._err()))


def device_count():
    """CUDA devices visible to libs4g.so (s4g_device_count); 0 when there is none"""
    n = C.c_int(0)
    load_library().s4g_device_count(C.byref(n))
    return int(n.value)


class Context:
    """RAII wrapper of s4g_ctx.  Clouds are the CENTRED sampled clouds."""

    def __init__(self, device=0):
        self._L = load_library()
        h = C.c_void_p()
        rc = self._L.s4g_create(int(device), C.byref(h))
        if rc != 0:
            raise S4GError("s4g_create(device=%d) failed with code %d: no usable CUDA device "
                           "(libs4g has no CPU fallback)" % (device, rc))
        self.h = h
        self.device = device
        self.nP = self.nQ = 0
        self.delta = None

    def close(self):
        if getattr(self, "h", None):
            self._L.s4g_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _err(self):
        return self._L.s4g_error_string(self.h).decode()

    def _chk(self, rc):
        if rc != 0:
            raise S4GError("libs4g error %d: %s" % (rc, self._L.s4g_error_string(self.h).decode()))

    # ---- plumbing
    def set_stream(self, cuda_stream_ptr):
        self._chk(self._L.s4g_set_stream(self.h, C.c_void_p(cuda_stream_ptr)))

    def synchronize(self):
        self._chk(self._L.s4g_synchronize(self.h))

    def timings(self):
        o = np.zeros(5, np.float64)
        self._chk(self._L.s4g_get_timings(self.h, _p(o)))
        return dict(verify_ms=o[0], rigid_ms=o[1], pairs_ms=o[2], quads_ms=o[3], launches=int(o[4]))

    # ---- clouds
    def set_cloud_p(self, P, delta):
        P = _c(P).reshape(-1, 3)
        self._chk(self._L.s4g_set_cloud_p(self.h, _p(P), len(P), float(delta)))
        self.nP, self.delta = len(P), float(delta)

    def set_cloud_q(self, Q, normals=None, rgb=None):
        Q, normals, rgb = _c(Q).reshape(-1, 3), _c(normals), _c(rgb)
        self._chk(self._L.s4g_set_cloud_q(self.h, _p(Q), _p(normals), _p(rgb), len(Q)))
        self.nQ = len(Q)

    def q_normalization(self):
        o = np.zeros(5, _f)
        self._chk(self._L.s4g_get_q_normalization(self.h, _p(o)))
        return o[:3].copy(), float(o[3])

    def grid_stats(self):
        o = np.zeros(6, np.float64)
        self._chk(self._L.s4g_get_grid_stats(self.h, _p(o)))
        return dict(cell_edge=o[0], bricks=int(o[1]), brick_edge=int(o[2]), cells=int(o[3]),
                    points_per_occupied_cell=o[4], resident_bytes=o[5])

    # ---- a8
    def verify(self, T_colmajor):
        T = _c(T_colmajor).reshape(-1, 16)
        counts = np.zeros(len(T), np.uint32)
        self._chk(self._L.s4g_verify(self.h, _p(T), len(T), _p(counts)))
        return counts

    def verify_dev(self, d_T_ptr, K, d_counts_ptr):
        self._chk(self._L.s4g_verify_dev(self.h, C.c_void_p(d_T_ptr), int(K), C.c_void_p(d_counts_ptr)))

    def verify_nearest(self, T_colmajor):
        """-> (index [K, n_Q] int32, sq_dist [K, n_Q] float32, counts [K] uint32): for every sampled-Q point the sampled-P
        point nearest to T q within delta (-1 / +inf: none; equal distances -> the smallest P index), see s4g.h"""
        T = _c(T_colmajor).reshape(-1, 16)
        K = len(T)
        index, sq = np.empty((K, self.nQ), np.int32), np.empty((K, self.nQ), _f)
        counts = np.zeros(K, np.uint32)
        self._chk(self._L.s4g_verify_nearest(self.h, _p(T), K, _p(index), _p(sq), _p(counts)))
        return index, sq, counts

    def verify_nearest_dev(self, d_T_ptr, K, d_index_ptr, d_sq_dist_ptr=None, d_counts_ptr=None):
        """device pointers (K x n_Q int32 / float32, K uint32; the last two may be None), stream-ordered, nothing synchronised"""
        self._chk(self._L.s4g_verify_nearest_dev(self.h, C.c_void_p(d_T_ptr), int(K), C.c_void_p(d_index_ptr),
                                                 C.c_void_p(d_sq_dist_ptr) if d_sq_dist_ptr else None,
                                                 C.c_void_p(d_counts_ptr) if d_counts_ptr else None))

    def nearest(self, xyz, sq_radius=np.inf, T=None, exclude=None, stats=False):
        """-> (index [n] int32, sq_dist [n] float32): for every query point x the resident P point nearest to T x (x when T
        is None) with d^2 <= sq_radius and index != exclude (-1 / +inf: none; equal distances -> the smallest P index),
        see s4g.h.  stats=True: also {P points tested, coarse blocks scanned} summed over the queries."""
        xyz = _c(xyz).reshape(-1, 3)
        n = len(xyz)
        T = None if T is None else _c(T).reshape(16)
        exclude = None if exclude is None else _c(exclude, np.int32).reshape(n)
        index, sq = np.empty(n, np.int32), np.empty(n, _f)
        if not stats:
            self._chk(self._L.s4g_nearest(self.h, _p(xyz), n, _p(T), float(sq_radius), _p(exclude), _p(index), _p(sq)))
            return index, sq
        out = np.zeros(2, np.uint64)
        self._chk(self._L.s4g_nearest_probe_stats(self.h, _p(xyz), n, _p(T), float(sq_radius), _p(exclude), _p(index),
                                                  _p(sq), _p(out)))
        return index, sq, dict(tested=int(out[0]), blocks=int(out[1]))

    def nearest_dev(self, d_xyz_ptr, n, d_index_ptr, d_sq_dist_ptr=None, sq_radius=np.inf, d_T_ptr=None, d_exclude_ptr=None):
        """device pointers (n x 3 float32 queries, n int32 / float32 results, 16 float32 T, n int32 exclude; the last three
        may be None), stream-ordered, nothing synchronised"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_nearest_dev(self.h, v(d_xyz_ptr), int(n), v(d_T_ptr), float(sq_radius), v(d_exclude_ptr),
                                          v(d_index_ptr), v(d_sq_dist_ptr)))

    def knn(self, xyz, k, sq_radius=np.inf, T=None, exclude=None, stats=False):
        """-> (index [n, k] int32, sq_dist [n, k] float32): for every query point x the k resident P points nearest to T x
        (x when T is None) with d^2 <= sq_radius and index != exclude, in ascending (d^2, index); a row with fewer is padded
        with -1 / +inf.  1 <= k <= 64; see s4g.h.  stats=True: also {P points tested, coarse blocks scanned} summed over
        the queries."""
        xyz = _c(xyz).reshape(-1, 3)
        n, k = len(xyz), int(k)
        T = None if T is None else _c(T).reshape(16)
        exclude = None if exclude is None else _c(exclude, np.int32).reshape(n)
        index, sq = np.empty((n, max(k, 0)), np.int32), np.empty((n, max(k, 0)), _f)
        if not stats:
            self._chk(self._L.s4g_knn(self.h, _p(xyz), n, _p(T), k, float(sq_radius), _p(exclude), _p(index), _p(sq)))
            return index, sq
        out = np.zeros(2, np.uint64)
        self._chk(self._L.s4g_knn_probe_stats(self.h, _p(xyz), n, _p(T), k, float(sq_radius), _p(exclude), _p(index),
                                              _p(sq), _p(out)))
        return index, sq, dict(tested=int(out[0]), blocks=int(out[1]))

    def knn_dev(self, d_xyz_ptr, n, k, d_index_ptr, d_sq_dist_ptr=None, sq_radius=np.inf, d_T_ptr=None, d_exclude_ptr=None):
        """device pointers (n x 3 float32 queries, n x k int32 / float32 results, 16 float32 T, n int32 exclude; the last
        three may be None), stream-ordered, nothing synchronised"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_knn_dev(self.h, v(d_xyz_ptr), int(n), v(d_T_ptr), int(k), float(sq_radius), v(d_exclude_ptr),
                                      v(d_index_ptr), v(d_sq_dist_ptr)))

    def normals(self, k, sq_radius=np.inf, viewpoint=None):
        """-> (normals [nP, 3] float32, eigenvalues [nP, 3] float32): for every resident P point, in the order of
        set_cloud_p, the PCA normal of its k-nearest row (s4g_knn of the point itself within sq_radius) and the
        covariance's eigenvalues, ascending.  Unoriented normals have their largest component positive; with a viewpoint
        (3 floats) they face it.  (0, 0, 0) where the row holds fewer than 3 points or they coincide.  3 <= k <= 64; see
        s4g.h."""
        n = self.nP
        vp = None if viewpoint is None else _c(viewpoint).reshape(3)
        normals, eig = np.empty((n, 3), _f), np.empty((n, 3), _f)
        self._chk(self._L.s4g_normals(self.h, int(k), float(sq_radius), _p(vp), _p(normals), _p(eig)))
        return normals, eig

    def normals_dev(self, k, d_normals_ptr, d_eigenvalues_ptr=None, sq_radius=np.inf, viewpoint=None):
        """device pointers (nP x 3 float32 normals; nP x 3 float32 eigenvalues or None), stream-ordered, nothing
        synchronised; viewpoint: 3 floats or None, as in normals"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        vp = None if viewpoint is None else _c(viewpoint).reshape(3)
        self._chk(self._L.s4g_normals_dev(self.h, int(k), float(sq_radius), _p(vp), v(d_normals_ptr),
                                          v(d_eigenvalues_ptr)))

    def orient_normals(self, normals, k, sq_radius=np.inf, viewpoint=None):
        """-> (oriented [nP, 3] float32, root [nP] int32, n_components, tree_edges [n_tree, 2] int32): the normals of the
        resident P (one row per point, in the order of set_cloud_p; (0, 0, 0) = no normal) with their signs made
        consistent along the minimum spanning forest of the k-nearest graph weighted by |n_i . n_j|; root[j] = the
        smallest position in j's component (-1: no normal); each component's anchor (its root, or with a viewpoint the
        member nearest to it, turned to face it) keeps its sign.  The forest is returned in ascending (lo, hi).
        1 <= k <= 64; see s4g.h (s4g_orient_normals)."""
        n = self.nP
        N = _c(normals).reshape(-1, 3)
        if len(N) != n:
            raise ValueError("orient_normals needs one normal per resident P point")
        vp = None if viewpoint is None else _c(viewpoint).reshape(3)
        out, root = np.empty((n, 3), _f), np.empty(n, np.int32)
        tree, out2 = np.empty((max(n - 1, 0), 2), np.int32), np.zeros(2, np.int64)
        self._chk(self._L.s4g_orient_normals(self.h, _p(N), int(k), float(sq_radius), _p(vp), _p(out), _p(root),
                                             _p(out2), _p(tree)))
        return out, root, int(out2[0]), tree[:int(out2[1])].copy()

    def orient_normals_dev(self, d_normals_ptr, k, d_normals_out_ptr, d_out2_ptr, d_root_ptr=None, d_tree_edges_ptr=None,
                           sq_radius=np.inf, viewpoint=None):
        """device pointers (nP x 3 float32 normals in and out, which may be the same buffer; 2 int64 out2 = {n_components
        or -1 for a non-finite normal, n_tree_edges}; nP int32 root and 2 (nP - 1) int32 tree_edges or None),
        stream-ordered, nothing synchronised; viewpoint: 3 floats or None, as in orient_normals"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        vp = None if viewpoint is None else _c(viewpoint).reshape(3)
        self._chk(self._L.s4g_orient_normals_dev(self.h, v(d_normals_ptr), int(k), float(sq_radius), _p(vp),
                                                 v(d_normals_out_ptr), v(d_root_ptr), v(d_out2_ptr), v(d_tree_edges_ptr)))

    def fpfh(self, normals, k, sq_radius=np.inf):
        """-> [nP, 33] float32: the FPFH descriptor of every resident P point (in the order of set_cloud_p) from its k
        nearest other points within sq_radius and the normals (one row per point; (0, 0, 0) or non-finite = no normal,
        which gives an all-zero descriptor).  Bins 0-10 f1, 11-21 f2, 22-32 f3.  Orient the normals consistently first:
        their signs mirror f1 and f3.  1 <= k <= 64; see s4g.h (s4g_fpfh)."""
        N = _c(normals).reshape(-1, 3)
        if len(N) != self.nP:
            raise ValueError("fpfh needs one normal per resident P point")
        out = np.empty((self.nP, 33), _f)
        self._chk(self._L.s4g_fpfh(self.h, _p(N), int(k), float(sq_radius), _p(out)))
        return out

    def fpfh_dev(self, d_normals_ptr, k, d_fpfh_ptr, sq_radius=np.inf):
        """device pointers (nP x 3 float32 normals, nP x 33 float32 descriptors), stream-ordered, nothing synchronised"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_fpfh_dev(self.h, v(d_normals_ptr), int(k), float(sq_radius), v(d_fpfh_ptr)))

    def fpfh_match(self, a, b, mutual=False):
        """-> (index [n_a] int32, sq_dist [n_a] float32): for every row of a (n_a x 33) the row of b (n_b x 33) with the
        smallest (d^2, index), d^2 summed in fp32 over the 33 bins in order; -1 / +inf when no d^2 is finite.  mutual:
        index[i] = -1 unless a[i] is also the nearest row of a to b[index[i]].  See s4g.h (s4g_fpfh_match)."""
        A, B = _c(a).reshape(-1, 33), _c(b).reshape(-1, 33)
        index, sq = np.empty(len(A), np.int32), np.empty(len(A), _f)
        self._chk(self._L.s4g_fpfh_match(self.h, _p(A), len(A), _p(B), len(B), int(bool(mutual)), _p(index), _p(sq)))
        return index, sq

    def fpfh_match_dev(self, d_a_ptr, n_a, d_b_ptr, n_b, d_index_ptr, d_sq_dist_ptr=None, mutual=False):
        """device pointers (n_a x 33 and n_b x 33 float32 descriptors, n_a int32 index, n_a float32 sq_dist or None),
        stream-ordered, nothing synchronised"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_fpfh_match_dev(self.h, v(d_a_ptr), int(n_a), v(d_b_ptr), int(n_b), int(bool(mutual)),
                                             v(d_index_ptr), v(d_sq_dist_ptr)))

    def statistical_outliers(self, k, std_ratio):
        """-> (keep [n_kept] int32, mean_dist [nP] float64, mu, sigma): the resident P points (positions in the array of
        set_cloud_p, ascending) whose mean distance to their k nearest other points is at most mu + std_ratio * sigma, mu
        and sigma the mean and sample standard deviation of those means over P.  1 <= k <= 64; see s4g.h."""
        n = self.nP
        keep, mean, out2 = np.empty(n, np.int32), np.empty(n, np.float64), np.zeros(2, np.float64)
        nk = C.c_int64(0)
        self._chk(self._L.s4g_statistical_outliers(self.h, int(k), float(std_ratio), _p(keep), C.byref(nk), _p(mean),
                                                   _p(out2)))
        return keep[:nk.value].copy(), mean, float(out2[0]), float(out2[1])

    def statistical_outliers_dev(self, k, std_ratio, d_keep_ptr, d_n_kept_ptr, d_mean_dist_ptr=None, d_out2_ptr=None):
        """device pointers (nP int32 keep, 1 int64 n_kept, nP float64 mean_dist or None, 2 float64 {mu, sigma} or None),
        stream-ordered, nothing synchronised"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_statistical_outliers_dev(self.h, int(k), float(std_ratio), v(d_keep_ptr), v(d_n_kept_ptr),
                                                       v(d_mean_dist_ptr), v(d_out2_ptr)))

    def radius_outliers(self, sq_radius, min_neighbors):
        """-> (keep [n_kept] int32, counts [nP] int32): the resident P points (ascending positions) with at least
        min_neighbors other P points at d^2 < sq_radius; counts[j] = that number, capped at min_neighbors.  See s4g.h."""
        n = self.nP
        keep, counts = np.empty(n, np.int32), np.empty(n, np.int32)
        nk = C.c_int64(0)
        self._chk(self._L.s4g_radius_outliers(self.h, float(sq_radius), int(min_neighbors), _p(keep), C.byref(nk),
                                              _p(counts)))
        return keep[:nk.value].copy(), counts

    def radius_outliers_dev(self, sq_radius, min_neighbors, d_keep_ptr, d_n_kept_ptr, d_counts_ptr=None):
        """device pointers (nP int32 keep, 1 int64 n_kept, nP int32 counts or None), stream-ordered, nothing
        synchronised"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_radius_outliers_dev(self.h, float(sq_radius), int(min_neighbors), v(d_keep_ptr),
                                                  v(d_n_kept_ptr), v(d_counts_ptr)))

    def euclidean_clusters(self, sq_radius, min_size=1, max_size=None):
        """-> (labels [nP] int32, root [nP] int32, offsets [n_clusters + 1] int64, members [offsets[-1]] int32): the
        connected components of the resident P under d^2 < sq_radius (root[j] = the smallest position in j's component),
        the clusters among them (min_size <= size <= max_size; None: no upper limit) ordered by size descending, ties by
        root; labels[j] = the rank of j's cluster or -1; cluster c is members[offsets[c]:offsets[c + 1]], ascending.
        See s4g.h."""
        n = self.nP
        labels, root = np.empty(n, np.int32), np.empty(n, np.int32)
        offsets, members = np.empty(n + 1, np.int64), np.empty(n, np.int32)
        nc = C.c_int64(0)
        self._chk(self._L.s4g_euclidean_clusters(self.h, float(sq_radius), int(min_size), _max_size(max_size), _p(labels),
                                                 _p(root), C.byref(nc), _p(offsets), _p(members)))
        nc = nc.value
        return labels, root, offsets[:nc + 1].copy(), members[:offsets[nc]].copy()

    def euclidean_clusters_dev(self, sq_radius, d_labels_ptr, d_n_clusters_ptr, d_root_ptr=None, d_offsets_ptr=None,
                               d_members_ptr=None, min_size=1, max_size=None):
        """device pointers (nP int32 labels, 1 int64 n_clusters, nP int32 root or None, nP + 1 int64 offsets or None, nP
        int32 members or None), stream-ordered, nothing synchronised"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_euclidean_clusters_dev(self.h, float(sq_radius), int(min_size), _max_size(max_size),
                                                     v(d_labels_ptr), v(d_root_ptr), v(d_n_clusters_ptr),
                                                     v(d_offsets_ptr), v(d_members_ptr)))

    def segment_planes(self, threshold, n_hypotheses=1000, max_planes=1, min_inliers=1, seed=0, refine=True,
                       hyp_counts=False):
        """-> (labels [nP] int32, planes [n_planes] PLANE_DTYPE, offsets [n_planes + 1] int64, members [offsets[-1]]
        int32), and counts [max_planes, n_hypotheses] uint32 when hyp_counts: RANSAC planes of the resident P, every
        hypothesis counted (inlier iff |a x + b y + c z + d| < threshold in fp32), the winner refitted by least squares
        (refine), up to max_planes planes of at least min_inliers points each, one after the other on the points no
        earlier plane claimed.  labels[j] = the plane of position j or -1; plane r is members[offsets[r]:offsets[r + 1]],
        ascending.  A pure function of its arguments; see s4g.h (s4g_segment_planes)."""
        n, H, R = self.nP, int(n_hypotheses), int(max_planes)
        labels, members = np.empty(n, np.int32), np.empty(n, np.int32)
        planes, offsets = np.zeros(max(R, 0), PLANE_DTYPE), np.zeros(max(R, 0) + 1, np.int64)
        counts = np.empty((max(R, 0), max(H, 0)), np.uint32) if hyp_counts else None
        np_ = C.c_int(0)
        self._chk(self._L.s4g_segment_planes(self.h, float(threshold), H, C.c_uint64(int(seed) % 2 ** 64),
                                             1 if refine else 0, R, int(min_inliers), _p(labels),
                                             planes.ctypes.data_as(C.POINTER(Plane)), C.byref(np_), _p(offsets),
                                             _p(members), _p(counts)))
        k = np_.value
        out = (labels, planes[:k].copy(), offsets[:k + 1].copy(), members[:offsets[k]].copy())
        return out + (counts,) if hyp_counts else out

    def segment_planes_dev(self, threshold, d_labels_ptr, d_planes_ptr, d_n_planes_ptr, d_offsets_ptr=None,
                           d_members_ptr=None, d_hyp_counts_ptr=None, n_hypotheses=1000, max_planes=1, min_inliers=1,
                           seed=0, refine=True):
        """device pointers (nP int32 labels, max_planes 64-byte s4g_plane records, 1 int32 n_planes, max_planes + 1
        int64 offsets or None, nP int32 members or None, max_planes x n_hypotheses uint32 counts or None),
        stream-ordered, nothing synchronised"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_segment_planes_dev(self.h, float(threshold), int(n_hypotheses),
                                                 C.c_uint64(int(seed) % 2 ** 64), 1 if refine else 0, int(max_planes),
                                                 int(min_inliers), v(d_labels_ptr), v(d_planes_ptr), v(d_n_planes_ptr),
                                                 v(d_offsets_ptr), v(d_members_ptr), v(d_hyp_counts_ptr)))

    def range_query(self, xyz, sq_radius, T=None):
        """-> (offsets [n + 1] int64, indices [total] int32, sq_dist [total] float32): for every query point x, every
        resident P point j with d^2 = |T x - p_j|^2 < sq_radius (x when T is None), in ascending j; list i is
        indices[offsets[i]:offsets[i + 1]].  See s4g.h (s4g_range)."""
        xyz = _c(xyz).reshape(-1, 3)
        n = len(xyz)
        T = None if T is None else _c(T).reshape(16)
        offsets = np.zeros(n + 1, np.int64)
        total = C.c_int64(0)
        self._chk(self._L.s4g_range(self.h, _p(xyz), n, _p(T), float(sq_radius), _p(offsets), C.byref(total)))
        indices, sq = np.empty(total.value, np.int32), np.empty(total.value, _f)
        self._chk(self._L.s4g_get_range(self.h, _p(indices), _p(sq)))
        return offsets, indices, sq

    def range_count_dev(self, d_xyz_ptr, n, d_offsets_ptr, sq_radius, d_T_ptr=None):
        """device pointers (n x 3 float32 queries, n + 1 int64 offsets, 16 float32 T or None): the CSR offsets of the
        range query, stream-ordered, nothing synchronised; the total is d_offsets[n]"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_range_count_dev(self.h, v(d_xyz_ptr), int(n), v(d_T_ptr), float(sq_radius),
                                              v(d_offsets_ptr)))

    def range_fill_dev(self, d_xyz_ptr, n, d_offsets_ptr, total, d_indices_ptr, d_sq_dist_ptr, sq_radius, d_T_ptr=None):
        """device pointers (the queries and offsets given to range_count_dev, total = d_offsets[n]; total int32 indices,
        total float32 d^2 or None): the sorted lists, stream-ordered, nothing synchronised"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_range_fill_dev(self.h, v(d_xyz_ptr), int(n), v(d_T_ptr), float(sq_radius), v(d_offsets_ptr),
                                             int(total), v(d_indices_ptr), v(d_sq_dist_ptr)))

    def verify_best_dev(self, d_T_ptr, K, d_index_ptr, d_counts_ptr, d_key_ptr):
        """Verify + first-maximum key (+ the maximum over the communicator's ranks), stream-ordered, nothing synchronised"""
        self._chk(self._L.s4g_verify_best_dev(self.h, C.c_void_p(d_T_ptr), int(K),
                                              C.c_void_p(d_index_ptr) if d_index_ptr else None,
                                              C.c_void_p(d_counts_ptr), C.c_void_p(d_key_ptr)))

    def verify_best(self, T_colmajor, index=None):
        """host buffers -> (counts, key); key = max (count << 32 | 0xFFFFFFFF - index) over this and the peers' lists"""
        T = _c(T_colmajor).reshape(-1, 16)
        idx = None if index is None else _c(index, np.uint32).reshape(-1)
        counts, key = np.zeros(len(T), np.uint32), np.zeros(1, np.uint64)
        self._chk(self._L.s4g_verify_best(self.h, _p(T), len(T), _p(idx), _p(counts), _p(key)))
        return counts, int(key[0])

    # ---- row e: the reduction of a sharded candidate set inside the library (NCCL, loaded on first use)
    def comm_init_rank(self, unique_id, n_ranks, rank):
        buf = np.frombuffer(bytes(unique_id), np.uint8).copy()
        assert buf.size == COMM_ID_BYTES
        self._chk(self._L.s4g_comm_init_rank(self.h, _p(buf), int(n_ranks), int(rank)))

    def comm_destroy(self):
        self._chk(self._L.s4g_comm_destroy(self.h))

    def comm_info(self):
        o = np.zeros(4, np.int32)
        self._chk(self._L.s4g_comm_info(self.h, _p(o)))
        return dict(ranks=int(o[0]), rank=int(o[1]), nccl_version=int(o[2]), collectives=int(o[3]))

    def comm_set_timeout(self, seconds):
        self._chk(self._L.s4g_comm_set_timeout(self.h, int(seconds)))

    def verify_probe_stats(self, T_colmajor):
        T = _c(T_colmajor).reshape(-1, 16)
        o = np.zeros(5, np.uint64)
        self._chk(self._L.s4g_verify_probe_stats(self.h, _p(T), len(T), _p(o)))
        return dict(points_tested=int(o[0]), ranges_read=int(o[1]), brick_entries_read=int(o[2]),
                    bitmap_words_read=int(o[3]), tile_pairs_culled=int(o[4]))

    # ---- a6 / a7
    def rigid_batch(self, base_xyz, quads, max_angle_deg=-1.0):
        b, q = _c(base_xyz).reshape(12), _c(quads, np.int32).reshape(-1, 4)
        K = len(q)
        T, rms, ok = np.zeros((K, 16), _f), np.zeros(K, _f), np.zeros(K, np.int32)
        self._chk(self._L.s4g_rigid_batch(self.h, _p(b), _p(q), K, float(max_angle_deg), _p(T), _p(rms), _p(ok)))
        return T, rms, ok.astype(bool)

    @staticmethod
    def _tcs_dict(r):
        return dict(key=int(r.key), best_count=int(r.best_count), best_index=int(r.best_index),
                    n_gate_pass=int(r.n_gate_pass), n_q=int(r.n_q), T=np.array(r.best_T, _f),
                    rms=float(r.best_rms), centroid1=np.array(r.centroid1, _f),
                    centroid2=np.array(r.centroid2, _f), quad=np.array(r.best_quad, np.int32))

    def try_congruent_set(self, base_xyz, quads, rms_threshold, max_angle_deg=-1.0, shard_rank=0, shard_world=1):
        b, q = _c(base_xyz).reshape(12), _c(quads, np.int32).reshape(-1, 4)
        r = TcsResult()
        self._chk(self._L.s4g_try_congruent_set(self.h, _p(b), _p(q), len(q), float(max_angle_deg),
                                                float(rms_threshold), int(shard_rank), int(shard_world), C.byref(r)))
        return self._tcs_dict(r)

    def try_congruent_set_dev(self, base_xyz, d_quads_ptr, K, rms_threshold, max_angle_deg=-1.0, shard_rank=0,
                              shard_world=1):
        b = _c(base_xyz).reshape(12)
        r = TcsResult()
        self._chk(self._L.s4g_try_congruent_set_dev(self.h, _p(b), C.c_void_p(d_quads_ptr), int(K),
                                                    float(max_angle_deg), float(rms_threshold), int(shard_rank),
                                                    int(shard_world), C.byref(r)))
        return self._tcs_dict(r)

    def try_congruent_set_resident(self, base_xyz, rms_threshold, max_angle_deg=-1.0, shard_rank=0, shard_world=1):
        b = _c(base_xyz).reshape(12)
        r = TcsResult()
        self._chk(self._L.s4g_try_congruent_set_resident(self.h, _p(b), float(max_angle_deg), float(rms_threshold),
                                                         int(shard_rank), int(shard_world), C.byref(r)))
        return self._tcs_dict(r)

    # ---- f1: several bases per launch chain
    def try_bases(self, bases, eps, thr2, rms_threshold, filters=None, max_angle_deg=-1.0):
        """bases: list of dicts(d1, d2, na1, na2, b9 (4 x 9), bxp (4 x 3), inv1, inv2) -> list of dicts(n_pairs, n_quads, tcs)"""
        B = len(bases)
        arr = (BaseDesc * B)()
        for k, b in enumerate(bases):
            arr[k].pair_distance[0], arr[k].pair_distance[1] = float(b["d1"]), float(b["d2"])
            arr[k].pair_normals_angle[0], arr[k].pair_normals_angle[1] = float(b.get("na1", 0.0)), float(b.get("na2", 0.0))
            b9 = _c(b["b9"]).reshape(4, 9)
            for i in range(4):
                for j in range(9):
                    arr[k].base_p[i][j] = float(b9[i, j])
            bxp = _c(b["bxp"]).reshape(12)
            for j in range(12):
                arr[k].base_xyz_p[j] = float(bxp[j])
            arr[k].invariant1, arr[k].invariant2 = float(b["inv1"]), float(b["inv2"])
        res = (BaseResult * B)()
        f = filters if filters is not None else PairFilters(-1, -1, -1, -1)
        self._chk(self._L.s4g_try_bases(self.h, C.byref(arr), B, float(eps), C.byref(f), float(thr2), float(max_angle_deg),
                                        float(rms_threshold), C.byref(res)))
        return [dict(n_pairs=[int(r.n_pairs[0]), int(r.n_pairs[1])], n_quads=int(r.n_quads), tcs=self._tcs_dict(r.tcs)) for r in res]

    # ---- a2 / a3
    def extract_pairs(self, pair_distance, pair_normals_angle, eps, base_p1=None, base_p2=None, filters=None,
                      slot=0, fetch=True):
        """base_p1/base_p2: 9 floats (pos, normal, rgb) of base_3D_[base_point1/2]."""
        d9 = np.array([0, 0, 0, 0, 0, 0, -1, -1, -1], _f)
        b1 = d9 if base_p1 is None else _c(base_p1).reshape(9)
        b2 = d9 if base_p2 is None else _c(base_p2).reshape(9)
        f = filters if filters is not None else PairFilters(-1, -1, -1, -1)
        n = C.c_int64(0)
        self._chk(self._L.s4g_extract_pairs(self.h, float(pair_distance), float(pair_normals_angle), float(eps),
                                            _p(b1), _p(b2), C.byref(f), int(slot), C.byref(n)))
        if not fetch:
            return int(n.value)
        return self.get_pairs(slot, int(n.value))

    def get_pairs(self, slot, n):
        out = np.zeros((n, 2), np.int32)
        if n:
            self._chk(self._L.s4g_get_pairs(self.h, int(slot), _p(out)))
        return out

    def set_pairs(self, slot, pairs):
        p = _c(pairs, np.int32).reshape(-1, 2)
        self._chk(self._L.s4g_set_pairs(self.h, int(slot), _p(p), len(p)))

    def count_pairs(self, pair_distance, eps):
        n = C.c_int64(0)
        self._chk(self._L.s4g_count_pairs(self.h, float(pair_distance), float(eps), C.byref(n)))
        return int(n.value)

    def count_pairs_rows(self, pair_distance, eps):
        """(total, rows) with rows[a] = number of ordered pairs (a, .) of the shell query"""
        n = C.c_int64(0)
        rows = np.zeros(self.nQ, np.uint32)
        self._chk(self._L.s4g_count_pairs_rows(self.h, float(pair_distance), float(eps), _p(rows), C.byref(n)))
        return int(n.value), rows

    # ---- f2
    def voxel_sample(self, xyz, voxel):
        """indices (ascending) of the first point of every voxel of edge `voxel`"""
        X = _c(xyz).reshape(-1, 3)
        out = np.zeros(len(X), np.int32)
        n = C.c_int64(0)
        self._chk(self._L.s4g_voxel_sample(self.h, _p(X), len(X), float(voxel), _p(out), C.byref(n)))
        return out[:n.value].copy()

    def voxel_grid(self, xyz, leaf, normals=None, rgb=None, min_points=1):
        """-> (centroids [m, 3] float32, normals [m, 3] float32 or None, rgb [m, 3] float32 or None, counts [m] int32,
        first [m] int32, voxel_of [n] int32): the voxel grid of edge `leaf` downsampled to one centroid per voxel with at
        least min_points points, the normal and colour averaged over the same points, in the order of each voxel's first
        point; voxel_of[i] = the output row of point i's voxel or -1.  Fixed-order double sums; see s4g.h
        (s4g_voxel_grid)."""
        X = _c(xyz).reshape(-1, 3)
        N = None if normals is None else _c(normals).reshape(-1, 3)
        R = None if rgb is None else _c(rgb).reshape(-1, 3)
        n = len(X)
        for a in (N, R):
            if a is not None and len(a) != n:
                raise ValueError("normals and rgb need one row per point")
        out = np.empty((n, 3), np.float32)
        nout = None if N is None else np.empty((n, 3), np.float32)
        rout = None if R is None else np.empty((n, 3), np.float32)
        counts, first, voxel_of = np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n, np.int32)
        m = C.c_int64(0)
        self._chk(self._L.s4g_voxel_grid(self.h, _p(X), _p(N), _p(R), n, float(leaf), int(min_points), _p(out),
                                         _p(nout), _p(rout), _p(counts), _p(first), _p(voxel_of), C.byref(m)))
        k = m.value
        cut = lambda a: None if a is None else a[:k].copy()  # noqa: E731
        return out[:k].copy(), cut(nout), cut(rout), counts[:k].copy(), first[:k].copy(), voxel_of

    def voxel_grid_dev(self, d_xyz_ptr, n, leaf, d_xyz_out_ptr, d_n_out_ptr, d_normals_ptr=None, d_rgb_ptr=None,
                       d_normals_out_ptr=None, d_rgb_out_ptr=None, d_counts_ptr=None, d_first_ptr=None,
                       d_voxel_of_ptr=None, min_points=1):
        """device pointers (n x 3 float32 inputs; outputs of capacity n; 1 int64 n_out, -1 for an invalid coordinate or
        span), stream-ordered, nothing synchronised"""
        v = lambda p: C.c_void_p(p) if p else None  # noqa: E731
        self._chk(self._L.s4g_voxel_grid_dev(self.h, v(d_xyz_ptr), v(d_normals_ptr), v(d_rgb_ptr), int(n), float(leaf),
                                             int(min_points), v(d_xyz_out_ptr), v(d_normals_out_ptr),
                                             v(d_rgb_out_ptr), v(d_counts_ptr), v(d_first_ptr), v(d_voxel_of_ptr),
                                             v(d_n_out_ptr)))

    # ---- a4 / a5
    def find_quads(self, inv1, inv2, thr2, base_xyz, fetch=True):
        b = _c(base_xyz).reshape(12)
        n = C.c_int64(0)
        self._chk(self._L.s4g_find_quads(self.h, float(inv1), float(inv2), float(thr2), _p(b), C.byref(n)))
        if not fetch:
            return int(n.value)
        out = np.zeros((int(n.value), 4), np.int32)
        if n.value:
            self._chk(self._L.s4g_get_quads(self.h, _p(out)))
        return out
