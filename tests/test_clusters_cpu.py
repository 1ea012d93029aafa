"""Euclidean clusters (s4g_euclidean_clusters) without a GPU: the port's components against those built from the compiled
reference's own kd-tree range lists and against scipy (cKDTree.query_pairs + connected_components, float64), the
ordering, size-limit and degenerate-cloud rules of the contract, and the C++ layer's Utils::ExtractEuclideanClusters on
the oracle stand-in.

Contract (include/s4g.h): edge (i, j) iff d^2 < sq_radius (fp32, s4g_range's d^2); root[j] = the smallest index of j's
component; clusters are the components with min_size <= size <= max_size, ordered by size descending, ties by root
ascending; labels[j] = the rank of j's cluster or -1; members in CSR form, ascending j within a cluster."""
import numpy as np
import pytest

from oracle import clusters as oc, range as orange
from tests import build_shim, clusters as tcl, edges as E
from tests.test_outliers_cpu import boundary_cloud

needs_ref = pytest.mark.skipif(not orange.ref_available(), reason="oracle/_ref (compiled reference) not present")
INT_MAX = 2 ** 31 - 1


def check_csr(labels, root, offsets, members, min_size=1, max_size=INT_MAX):
    """the port's output is consistent with its own root: every rule of the contract that follows from root"""
    n = len(root)
    assert (root <= np.arange(n)).all() and (root[root] == root).all()
    size = np.bincount(root, minlength=n)
    ok = (root == np.arange(n)) & (size >= min_size) & (size <= max_size)
    order = sorted(np.nonzero(ok)[0], key=lambda r: (-size[r], r))
    assert len(offsets) == len(order) + 1 and offsets[0] == 0
    for c, r in enumerate(order):
        mem = members[offsets[c]:offsets[c + 1]]
        assert np.array_equal(mem, np.nonzero(root == r)[0])
        assert (labels[mem] == c).all()
    assert (labels[~np.isin(root, order)] == -1).all()


@needs_ref
def test_components_equal_reference_range_lists():
    """the port's components equal those of the graph of the reference kd-tree's range lists, at generic radii and at
    radii equal to (and one ulp either side of) fl(d^2) of point pairs placed ulps around delta"""
    delta = 0.02
    Praw, Qraw, anchors, first = boundary_cloud(delta=delta)
    m = orange.RefRange(Praw, Qraw, delta)
    P, _ = m.sampled()
    assert len(P) == len(Praw)
    d2 = np.unique(E.fp32_d2(P[first:], P[anchors]).ravel())
    d2 = d2[np.abs(d2 - np.float32(delta) ** 2) <= 1e-3 * delta ** 2][:8]
    assert len(d2) >= 4
    rs = [-1.0, 0.0, (0.1 * delta) ** 2, delta * delta, 4 * delta * delta, np.inf]
    for x in d2:
        rs += [float(x), float(np.nextafter(x, np.float32(np.inf))), float(np.nextafter(x, np.float32(-np.inf)))]
    seen = set()
    for r in rs:
        off, idx, _ = m.query(P, r)
        want = oc.roots_from_lists(len(P), off, idx)
        root = oc.roots(P, r)
        assert np.array_equal(root, want), (r, np.argwhere(root != want)[:5])
        labels, root2, offsets, members = oc.clusters(P, r, 2)
        assert np.array_equal(root2, root)
        check_csr(labels, root, offsets, members, 2)
        seen.add(len(np.unique(root)))
    assert len(seen) >= 4                                # the radii move the partition


@pytest.mark.parametrize("kind", ["uniform", "clustered", "offcentre1e3"])
def test_components_equal_scipy(kind):
    """clouds with no pair distance within 1e-5 relative of the radius: the fp32 and float64 tests agree on every pair,
    so the components equal scipy's query_pairs + connected_components"""
    rng = np.random.RandomState(7)
    if kind == "uniform":
        P = rng.uniform(-1, 1, (3000, 3))
    elif kind == "clustered":
        P = tcl.blobs([400, 300, 300, 200, 100, 50, 20, 5, 1], spread=0.03, gap=0.12, seed=3)[0].astype(np.float64)
    else:
        P = rng.uniform(-0.1, 0.1, (2000, 3)) + 1e3
    P = P.astype(np.float32)
    from scipy.spatial.distance import pdist
    d = np.sort(pdist(P.astype(np.float64)))
    tested = 0
    for q in (1e-5, 1e-4, 5e-4, 2e-3, 1e-2):
        k = int(q * len(d))
        gaps = np.nonzero(d[k + 1:k + 2001] - d[k:k + 2000] > 3e-5 * d[k:k + 2000])[0]
        if len(gaps) == 0:
            continue
        r = float(np.float32(0.5 * (d[k + gaps[0]] + d[k + gaps[0] + 1])))    # the middle of a gap between distances
        if np.abs(d - r).min() <= 1e-5 * r:
            continue
        sq = float(np.float32(r) * np.float32(r))
        want = oc.scipy_roots(P, float(np.sqrt(sq)))
        assert np.array_equal(oc.roots(P, sq), want), r
        tested += 1
    assert tested >= 3


def test_rules():
    """ties by root; min_size / max_size at, above and below a size; sq_radius <= 0; +inf; nP = 1; coincident points;
    duplicates"""
    P, blob = tcl.blobs([5, 3, 5, 1, 3, 5], seed=1)
    labels, root, offsets, members = oc.clusters(P, 0.05 ** 2)
    assert np.array_equal(root, oc.canonical_roots(blob))
    assert np.array_equal(np.diff(offsets), [5, 5, 5, 3, 3, 1])
    firsts = [members[offsets[c]] for c in range(6)]
    assert firsts[0] < firsts[1] < firsts[2] and firsts[3] < firsts[4]     # equal sizes: ascending root
    check_csr(labels, root, offsets, members)
    for lo, hi, want in ((3, 3, [3, 3]), (4, 5, [5, 5, 5]), (6, INT_MAX, []), (1, 1, [1]), (2, 4, [3, 3]),
                         (5, 5, [5, 5, 5]), (1, INT_MAX, [5, 5, 5, 3, 3, 1])):
        lab, _, off, mem = oc.clusters(P, 0.05 ** 2, lo, hi)
        assert list(np.diff(off)) == want, (lo, hi)
        check_csr(lab, root, off, mem, lo, hi)
    for r in (0.0, -1.0, -np.inf):
        lab, rt, off, mem = oc.clusters(P, r)
        assert np.array_equal(rt, np.arange(len(P))) and np.array_equal(lab, np.arange(len(P)))
        assert np.array_equal(mem, np.arange(len(P)))
    lab, rt, off, mem = oc.clusters(P, np.inf)
    assert (rt == 0).all() and (lab == 0).all() and list(off) == [0, len(P)]
    assert oc.clusters(P, np.inf, 1, len(P) - 1)[2].tolist() == [0]        # one component, too big: no cluster
    one = oc.clusters(np.float32([[0.5, -0.25, 2.0]]), 1.0)
    assert [x.tolist() for x in one] == [[0], [0], [0, 1], [0]]
    same = np.tile(np.float32([[0.1, 0.2, 0.3]]), (50, 1))
    for r in (1e-30, 1.0):
        lab, rt, off, mem = oc.clusters(same, r)
        assert (rt == 0).all() and list(off) == [0, 50]
    assert np.array_equal(oc.clusters(same, 0.0)[1], np.arange(50))      # d^2 = 0 is not < 0
    rng = np.random.RandomState(2)
    P0 = rng.uniform(-1, 1, (300, 3)).astype(np.float32)
    Pd = np.concatenate([P0, P0[::7]])
    lab, rt, off, mem = oc.clusters(Pd, 1e-12)                             # only the duplicates join
    assert np.array_equal(rt[300:], np.arange(0, 300, 7)) and np.array_equal(rt[:300], np.arange(300))
    assert list(np.diff(off)) == [2] * len(P0[::7]) + [1] * (300 - len(P0[::7]))
    check_csr(lab, rt, off, mem)


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    d = tmp_path_factory.mktemp("clusters")
    exe = tcl.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


@pytest.mark.parametrize("tol,lo,hi", [(0.05, 1, INT_MAX), (0.05, 4, 5), (0.0, 1, INT_MAX), (float("inf"), 1, INT_MAX),
                                       (0.03, 2, 40)])
def test_cpp_function_on_oracle_shim(program, tmp_path, tol, lo, hi):
    """ExtractEuclideanClusters through the stand-in equals the port at fl(tolerance^2): the same clusters in the same
    order, each in ascending index order"""
    exe, shim = program
    P = tcl.blobs([60, 5, 40, 5, 1, 4, 4, 30], seed=4)[0]
    P = np.concatenate([P, np.random.RandomState(5).uniform(-0.3, 0.3, (200, 3)).astype(np.float32)])
    got = tcl.run(exe, tmp_path, P, tol, lo, hi, preload=shim)
    assert got is not None
    _, _, off, mem = oc.clusters(P, float(np.float32(tol) * np.float32(tol)), lo, hi)
    want = tcl.as_lists(off, mem)
    assert len(got) == len(want) and all(np.array_equal(a, b) for a, b in zip(got, want))
    if tol == 0.05 and lo == 1:
        assert len(got) > 8


def test_cpp_function_throws_on_bad_arguments(program, tmp_path):
    exe, shim = program
    P = np.random.RandomState(1).rand(100, 3).astype(np.float32)
    for tol, lo, hi in ((-1.0, 1, 10), (float("nan"), 1, 10), (0.1, 0, 10), (0.1, -2, 10), (0.1, 5, 4)):
        assert tcl.run(exe, tmp_path, P, tol, lo, hi, preload=shim) is None, (tol, lo, hi)
    assert tcl.run(exe, tmp_path, P[:0], 0.1, 1, 10, preload=shim) == []
