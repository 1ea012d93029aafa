"""Euclidean clusters on the GPU: s4g_euclidean_clusters over the resident P.

labels, root, n_clusters, offsets and members are bit-equal to the port's restatement (oracle/clusters_port.cc: every
pair tested, a sequential union-find, the same ordering and CSR rules) over the grid regimes of the k-nearest tests at
the radii of the outlier tests, on blobs whose clusters are known, and on union-find stress shapes: a 1M-point chain
(deep trees; one component, or pieces of known sizes when cut), a lattice at a spacing just under and just over the
radius, and 10^4 coincident points (a complete graph).  On a 1M-point cfg2 sample at 2 delta, the components equal the
union-find of the GPU's own range lists, whose sampled rows equal the brute force.  Two calls give the same bits, the
_dev and host forms agree, the error codes hold, and Utils::ExtractEuclideanClusters equals Context."""
import ctypes as C

import numpy as np
import pytest

from oracle import clusters as oc, range as orange
from tests import clusters as tcl, common, edges as E
from tests.test_decision_edges_gpu import cloud
from tests.test_knn_gpu import make_ctx  # noqa: F401  (fixture)
from tests.test_outliers_gpu import radii

pytestmark = pytest.mark.gpu

S4G_OK, S4G_ERR_ARG, S4G_ERR_STATE = 0, 2, 3   # include/s4g.h
INT_MAX = 2 ** 31 - 1


def same(got, want):
    for g, w, name in zip(got, want, ("labels", "root", "offsets", "members")):
        assert g.dtype == w.dtype and np.array_equal(g, w), (name, np.argwhere(g != w)[:5] if g.shape == w.shape else
                                                             (g.shape, w.shape))


def check(ctx, P, sq_radius, limits=((1, None),)):
    """every (min_size, max_size) against the port; returns the number of components"""
    root = oc.roots(P, sq_radius)
    for lo, hi in limits:
        got = ctx.euclidean_clusters(sq_radius, lo, hi)
        same(got, (oc.finish(root, lo, hi)[0], root) + oc.finish(root, lo, hi)[1:])
    return len(np.unique(root))


@pytest.mark.parametrize("name,cshift_min", [("centred", None), ("centred", 3), ("brick8", None), ("widened", None),
                                             ("offcentre1e3", None), ("offcentre1e4", None)])
def test_bit_equal_to_port_over_grid_regimes(make_ctx, name, cshift_min):  # noqa: F811
    delta = E.REGIMES[name][0]
    P, _, _ = cloud(name, cshift_min=cshift_min or 1)
    ctx = make_ctx(cshift_min)
    ctx.set_cloud_p(P, delta)
    counts = [check(ctx, P, r, ((1, None), (2, None), (3, 40))) for r in radii(delta)]
    assert counts[0] == counts[1] == len(P) and counts[-1] == 1     # sq_radius -1 and 0: singletons; +inf: one


def test_blobs_with_known_labels(make_ctx):  # noqa: F811
    """many small blobs and a few large ones: each blob is one component at radius 0.05 (tests/clusters.py blobs)"""
    rng = np.random.RandomState(1)
    sizes = list(rng.randint(1, 12, 300)) + [4000, 2500, 2500, 900]
    P, blob = tcl.blobs(sizes, seed=2)
    ctx = make_ctx()
    ctx.set_cloud_p(P, 0.025)
    for lo, hi in ((1, None), (5, None), (2, 10), (2500, 2500)):
        labels, root, offsets, members = ctx.euclidean_clusters(0.05 ** 2, lo, hi)
        assert np.array_equal(root, oc.canonical_roots(blob))
        same((labels, root, offsets, members), (oc.finish(root, lo, hi)[0], root) + oc.finish(root, lo, hi)[1:])
        want = sorted(s for s in sizes if s >= lo and (hi is None or s <= hi))[::-1]
        assert list(np.diff(offsets)) == want
    check(ctx, P, 0.05 ** 2)


def chain(n):
    """n points of the integer lattice, consecutive ones at distance 1 and any two others at d^2 >= 2: rows of 100
    along x, 3 apart in y and in z, joined at their ends by two turn points"""
    pts, x, y, z, dx, dy = [], 0, 0, 0, 1, 3
    while len(pts) < n:
        for _ in range(100):
            pts.append((x, y, z))
            x += dx
        x -= dx
        dx = -dx
        if 0 <= y + dy <= 297:
            for s in (1, 2):
                pts.append((x, y + s * dy // 3, z))
            y += dy
        else:
            for s in (1, 2):
                pts.append((x, y, z + s))
            z += 3
            dy = -dy
    return np.asarray(pts[:n], np.float32)


def test_chain(make_ctx):  # noqa: F811
    """1M points joined only to their neighbours along the chain: one component (root 0 everywhere, the answer in closed
    form), in chain order and with the indices shuffled; cut at known points, pieces of known sizes"""
    n = 1_000_000
    P = chain(n)
    d2 = ((P[1:] - P[:-1]) ** 2).sum(1)
    assert (d2 == 1).all()
    ctx = make_ctx()
    for perm in (np.arange(n), np.random.RandomState(3).permutation(n)):
        ctx.set_cloud_p(P[perm], 0.6)
        labels, root, offsets, members = ctx.euclidean_clusters(1.5)
        assert (root == 0).all() and (labels == 0).all()
        assert list(offsets) == [0, n] and np.array_equal(members, np.arange(n))
    cuts = np.array([17, 100_000, 100_001, 523_456, 999_000])
    Pc = np.delete(P, cuts, 0)
    ctx.set_cloud_p(Pc, 0.6)
    labels, root, offsets, members = ctx.euclidean_clusters(1.5)
    starts = np.concatenate([[0], cuts - np.arange(len(cuts))])
    ends = np.concatenate([starts[1:], [len(Pc)]])
    pieces = [(e - s, s) for s, e in zip(starts, ends) if e > s]
    assert np.array_equal(root, np.repeat([s for _, s in pieces], [m for m, _ in pieces]))
    want = sorted(pieces, key=lambda p: (-p[0], p[1]))
    assert list(np.diff(offsets)) == [m for m, _ in want]
    for c, (m, s) in enumerate(want):
        assert np.array_equal(members[offsets[c]:offsets[c + 1]], np.arange(s, s + m))
        assert (labels[s:s + m] == c).all()


def test_lattice_and_coincident_points(make_ctx):  # noqa: F811
    """a 20^3 lattice of spacing 1 at sq_radius one ulp under 1 (no edge: singletons) and one ulp over (the 6-neighbour
    graph: one component), a spacing-0.1 lattice against the port, and 10^4 coincident points (a complete graph)"""
    g = np.arange(20, dtype=np.float32)
    L = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)
    L = L[np.random.RandomState(4).permutation(len(L))]
    ctx = make_ctx()
    ctx.set_cloud_p(L, 0.5)
    labels, root, offsets, members = ctx.euclidean_clusters(float(np.nextafter(np.float32(1), np.float32(0))))
    assert np.array_equal(root, np.arange(len(L))) and np.array_equal(labels, np.arange(len(L)))
    labels, root, offsets, members = ctx.euclidean_clusters(float(np.nextafter(np.float32(1), np.float32(2))))
    assert (root == 0).all() and list(offsets) == [0, len(L)]
    for r in (float(np.nextafter(np.float32(1), np.float32(0))), float(np.nextafter(np.float32(1), np.float32(2)))):
        check(ctx, L, r)
    L1 = (L * np.float32(0.1)).astype(np.float32)
    ctx.set_cloud_p(L1, 0.05)
    for r in (0.0099, 0.01, 0.0101, 0.02, 0.0201):
        check(ctx, L1, r)
    same_pts = np.tile(np.float32([[0.3, -0.1, 0.2]]), (10_000, 1))
    ctx.set_cloud_p(same_pts, 0.01)
    labels, root, offsets, members = ctx.euclidean_clusters(1e-6)
    assert (root == 0).all() and (labels == 0).all() and list(offsets) == [0, 10_000]
    labels, root, offsets, members = ctx.euclidean_clusters(0.0)
    assert np.array_equal(root, np.arange(10_000)) and len(offsets) == 10_001
    single = np.float32([[0.1, 0.2, 0.3]])
    ctx.set_cloud_p(single, 0.01)
    same(ctx.euclidean_clusters(1.0), (np.int32([0]), np.int32([0]), np.int64([0, 1]), np.int32([0])))
    assert len(ctx.euclidean_clusters(1.0, 2)[2]) == 1


def test_full_size_sample(make_ctx):  # noqa: F811
    """1M points (cfg2, delta = 0.003) at 2 delta: the components equal the union-find of the GPU's own s4g_range
    lists, 300 sampled rows of which equal the brute force; labels, offsets and members follow from the root"""
    n, delta = 1_000_000, 0.003
    P = common.scenario(n, 0.3, delta, seed=42)["P"]
    sq = (2 * delta) ** 2
    ctx = make_ctx()
    ctx.set_cloud_p(P, delta)
    got = ctx.euclidean_clusters(sq, 1, None)
    off, idx, _ = ctx.range_query(P, sq)
    root = oc.roots_from_lists(n, off, idx)
    same(got, (oc.finish(root)[0], root) + oc.finish(root)[1:])
    for lo, hi in ((10, None), (2, 50)):
        same(ctx.euclidean_clusters(sq, lo, hi), (oc.finish(root, lo, hi)[0], root) + oc.finish(root, lo, hi)[1:])
    sub = np.sort(np.random.RandomState(0).choice(n, 300, replace=False))
    boff, bidx, _ = orange.bruteforce(P, P[sub], sq)
    for k, j in enumerate(sub):
        assert np.array_equal(idx[off[j]:off[j + 1]], bidx[boff[k]:boff[k + 1]]), j
    assert 1 < len(got[2]) - 1 < n


def test_repeatable_and_dev_form_equals_host_form(make_ctx):  # noqa: F811
    import torch
    P = tcl.blobs(list(np.random.RandomState(5).randint(1, 40, 400)) + [3000], seed=6)[0]
    P = np.concatenate([P, common.scenario(20000, 0.4, 0.01, seed=5)["P"] * np.float32(0.2)])
    ctx = make_ctx()
    ctx.set_cloud_p(P, 0.01)
    n = len(P)
    for r, lo, hi in ((0.02 ** 2, 1, None), (0.05 ** 2, 3, 100), (0.0, 1, None), (np.inf, 1, None)):
        want = ctx.euclidean_clusters(r, lo, hi)
        same(ctx.euclidean_clusters(r, lo, hi), want)
        labels, root = (torch.full((n,), 7, dtype=torch.int32, device="cuda") for _ in range(2))
        offsets, nc = torch.full((n + 1,), 7, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int64,
                                                                                              device="cuda")
        members = torch.full((n,), 7, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.euclidean_clusters_dev(r, labels.data_ptr(), nc.data_ptr(), root.data_ptr(), offsets.data_ptr(),
                                   members.data_ptr(), lo, hi)
        ctx.synchronize()
        k = int(nc.item())
        off = offsets[:k + 1].cpu().numpy()
        same((labels.cpu().numpy(), root.cpu().numpy(), off, members[:off[-1]].cpu().numpy()), want)
        labels.fill_(7)
        nc.zero_()
        torch.cuda.synchronize()
        ctx.euclidean_clusters_dev(r, labels.data_ptr(), nc.data_ptr(), min_size=lo, max_size=hi)   # the rest optional
        ctx.synchronize()
        assert np.array_equal(labels.cpu().numpy(), want[0]) and int(nc.item()) == k


def test_error_codes(s4g_lib):
    from super4pcs_b200 import Context
    with Context(0) as ctx:
        L, h = ctx._L, ctx.h
        lab, root, mem, off = np.empty(100, np.int32), np.empty(100, np.int32), np.empty(100, np.int32), np.empty(101,
                                                                                                             np.int64)
        nc = C.c_int64(0)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        args = lambda r, lo, hi: (h, r, lo, hi, p(lab), p(root), C.byref(nc), p(off), p(mem))  # noqa: E731
        assert L.s4g_euclidean_clusters(*args(1.0, 1, INT_MAX)) == S4G_ERR_STATE
        assert "s4g_set_cloud_p" in L.s4g_error_string(h).decode()
        assert L.s4g_euclidean_clusters_dev(*args(1.0, 1, INT_MAX)) == S4G_ERR_STATE
        ctx.set_cloud_p(np.random.RandomState(0).rand(100, 3).astype(np.float32), 0.05)
        for r, lo, hi in ((float("nan"), 1, 10), (1.0, 0, 10), (1.0, -1, 10), (1.0, 5, 4), (1.0, 1, 0)):
            assert L.s4g_euclidean_clusters(*args(r, lo, hi)) == S4G_ERR_ARG, (r, lo, hi)
            assert "min_size" in L.s4g_error_string(h).decode()
            assert L.s4g_euclidean_clusters_dev(*args(r, lo, hi)) == S4G_ERR_ARG
        assert L.s4g_euclidean_clusters(h, 1.0, 1, 10, None, p(root), C.byref(nc), p(off), p(mem)) == S4G_ERR_ARG
        assert L.s4g_euclidean_clusters(h, 1.0, 1, 10, p(lab), p(root), None, p(off), p(mem)) == S4G_ERR_ARG
        assert L.s4g_euclidean_clusters(None, 1.0, 1, 10, p(lab), p(root), C.byref(nc), p(off), p(mem)) == S4G_ERR_ARG
        assert L.s4g_euclidean_clusters(h, 0.0, 1, 1, p(lab), None, C.byref(nc), None, None) == S4G_OK
        assert nc.value == 100 and np.array_equal(lab, np.arange(100))
        assert L.s4g_euclidean_clusters(h, float("inf"), 5, 5, p(lab), p(root), C.byref(nc), p(off), p(mem)) == S4G_OK
        assert nc.value == 0 and (lab == -1).all() and (root == 0).all() and off[0] == 0
        with pytest.raises(Exception):
            ctx.euclidean_clusters(1.0, 0)


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = tcl.build(tmp_path_factory.mktemp("clusters"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


@pytest.mark.parametrize("tol,lo,hi", [(0.02, 1, INT_MAX), (0.05, 10, 3000), (0.0, 1, INT_MAX), (float("inf"), 1, INT_MAX)])
def test_cpp_function_equals_context(program, make_ctx, tmp_path, tol, lo, hi):  # noqa: F811
    """Utils::ExtractEuclideanClusters on the real library: the Context clusters at fl(tolerance^2) on the same cloud
    at the function's grid delta"""
    P = tcl.blobs(list(np.random.RandomState(7).randint(1, 30, 200)) + [2000, 500], seed=8)[0]
    P = np.concatenate([P, np.random.RandomState(9).uniform(-0.4, 0.4, (3000, 3)).astype(np.float32)])
    got = tcl.run(program, tmp_path, P, tol, lo, hi)
    assert got is not None
    ctx = make_ctx()
    ctx.set_cloud_p(P, tcl.tolerance_delta(P, tol))
    _, _, off, mem = ctx.euclidean_clusters(float(np.float32(tol) * np.float32(tol)), lo, hi)
    want = tcl.as_lists(off, mem)
    assert len(got) == len(want) and all(np.array_equal(a, b) for a, b in zip(got, want))
