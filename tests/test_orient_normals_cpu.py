"""Consistent normal orientation (s4g_orient_normals) without a GPU: the port (oracle/orient_normals_port.cc) against
restatements that share no code with it -- scipy's minimum_spanning_tree and breadth_first_order on clouds whose |dot| are
all distinct, a plain-Python Kruskal keyed on (-|dot|, lo, hi) where the tie rule alone decides -- the edge cases, the
quality on shapes with analytic normals, and Utils::OrientNormals on the oracle stand-in.

Contract (include/s4g.h): rows = s4g_knn with exclude = j; edges of the symmetrised rows between non-zero normals;
dot = (xi xj + yi yj) + zi zj and flip dot < 0 in fp32; the forest of the order (|dot| descending, lo, hi); root = the
smallest member; the anchor (the root, or the member nearest the viewpoint facing it) keeps its sign; each normal is
negated iff the xor of the flips on its forest path from the anchor, and the anchor's negation, say so."""
import numpy as np
import pytest

from oracle import knn as oknn, normals as onormals, orient_normals as oon
from tests import build_shim, common, normals as tnormals, orient_normals as ton

_f = np.float32


def same(got, want):
    assert got[2] == want[2], (got[2], want[2])
    assert np.array_equal(common.bits(got[0]), common.bits(want[0])), np.argwhere(got[0] != want[0])[:5]
    assert np.array_equal(got[1], want[1])
    assert np.array_equal(got[3], want[3])


def rows(P, k, sq_radius=np.inf):
    return oknn.bruteforce(P, P, k, sq_radius, exclude=np.arange(len(P), dtype=np.int32))[0]


def signs_only(got, N):
    """every output is + or - its input, bit for bit"""
    N = np.asarray(N, _f)
    b, nb, g = common.bits(N), common.bits(-N), common.bits(got)
    assert ((g == b).all(1) | (g == nb).all(1)).all()


@pytest.mark.parametrize("n,k,r,vp,seed", [(400, 8, np.inf, None, 0), (600, 6, np.inf, (0, 0, 5), 1),
                                           (1500, 4, 0.004, None, 2), (300, 1, np.inf, (1, 2, 3), 3),
                                           (500, 3, 0.01, (0.5, 0.5, -2), 4)])
def test_port_equals_scipy_on_distinct_weights(n, k, r, vp, seed):
    rng = np.random.RandomState(seed)
    P = rng.rand(n, 3).astype(_f)
    N = rng.normal(size=(n, 3)).astype(_f)
    N[::17] = 0                                            # points without a normal
    R = rows(P, k, r)
    assert ton.distinct_weights(N, R)                      # scipy's tree is the unique one only then
    got = oon.port(P, N, k, r, vp)
    same(got, ton.scipy_orient(P, N, R, vp))
    same(got, ton.kruskal_orient(P, N, R, vp))
    signs_only(got[0], N)
    assert len(got[3]) == int((N != 0).any(1).sum()) - got[2]


def test_three_normals_at_120_degrees_tie():
    """an odd cycle of flips whose three edges tie on |dot|: only (lo, hi) picks the two tree edges, and the third
    normal's sign depends on which"""
    c, s = _f(-0.5), _f(np.sqrt(_f(3)) / 2)
    N = np.array([[1, 0, 0], [c, s, 0], [c, -s, 0]], _f)
    P = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], _f)
    d = ton.dots(N, np.array([0, 0, 1]), np.array([1, 2, 2]))
    assert (d < 0).all() and len(set(np.abs(d).tolist())) == 1, d
    got = oon.port(P, N, 2)
    same(got, ton.kruskal_orient(P, N, rows(P, 2)))
    assert got[3].tolist() == [[0, 1], [0, 2]]
    assert np.array_equal(got[0], np.array([N[0], -N[1], -N[2]]))
    # the same normals renumbered: the tree follows the indices
    for perm in ([1, 2, 0], [2, 0, 1], [0, 2, 1]):
        got = oon.port(P[perm], N[perm], 2)
        same(got, ton.kruskal_orient(P[perm], N[perm], rows(P[perm], 2)))


@pytest.mark.parametrize("m", [9, 15, 21])
def test_ring_of_tied_edges(m):
    """a ring of m points, each joined to its two neighbours, normals cycling through three directions 120 degrees
    apart: every edge ties on |dot| and flips"""
    a = 2 * np.pi * np.arange(m) / m
    P = np.stack([np.cos(a), np.sin(a), np.zeros(m)], 1).astype(_f)
    c, s = _f(-0.5), _f(np.sqrt(_f(3)) / 2)
    dirs = np.array([[1, 0, 0], [c, s, 0], [c, -s, 0]], _f)
    N = dirs[np.arange(m) % 3]
    R = rows(P, 2)
    E = ton.edges_from_rows(N, R)
    assert len(E) == m and len(set(np.abs(ton.dots(N, E[:, 0], E[:, 1])).tolist())) == 1
    for vp in (None, (0, 0, 3), (2, 0, 0)):
        same(oon.port(P, N, 2, viewpoint=vp), ton.kruskal_orient(P, N, R, vp))


def test_zero_normals_and_isolated_points():
    rng = np.random.RandomState(5)
    P = rng.rand(200, 3).astype(_f)
    N = rng.normal(size=(200, 3)).astype(_f)
    N[[3, 50, 51, 199]] = 0
    P[7] = [40, 40, 40]                                    # far from all: isolated under a finite radius
    got = oon.port(P, N, 6, 0.05)
    assert (got[1][[3, 50, 51, 199]] == -1).all() and (got[0][[3, 50, 51, 199]] == 0).all()
    assert got[1][7] == 7 and np.array_equal(got[0][7], N[7])          # its own component, its own sign
    assert not (got[3] == 7).any()
    same(got, ton.kruskal_orient(P, N, rows(P, 6, 0.05)))
    # a zero normal joins nothing: a chain through it breaks
    P = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0]], _f)
    N = np.array([[0, 0, 1], [0, 0, 0], [0, 0, -1]], _f)
    got = oon.port(P, N, 1, 1.5)
    assert got[2] == 2 and got[1].tolist() == [0, -1, 2] and len(got[3]) == 0


def test_n_one_and_two_and_k_one():
    P = np.array([[0.1, 0.2, 0.3]], _f)
    got = oon.port(P, np.array([[0, -1, 0]], _f), 5)
    assert got[2] == 1 and got[1].tolist() == [0] and len(got[3]) == 0 and got[0].tolist() == [[0, -1, 0]]
    got = oon.port(P, np.array([[0, -1, 0]], _f), 5, viewpoint=(0, 5, 0))
    assert got[0].tolist() == [[0, 1, 0]]                  # faces the viewpoint
    P = np.array([[0, 0, 0], [1, 0, 0]], _f)
    N = np.array([[0, 0, 1], [0, 0.1, -1]], _f)
    got = oon.port(P, N, 1)
    assert got[2] == 1 and got[3].tolist() == [[0, 1]] and np.array_equal(got[0], np.array([N[0], -N[1]]))
    got = oon.port(P, N, 1, 0.5)                           # the radius splits them
    assert got[2] == 2 and got[1].tolist() == [0, 1] and np.array_equal(got[0], N)
    # k = 1 on a larger cloud: the rows are nearest neighbours, the graph their symmetrisation
    rng = np.random.RandomState(9)
    P = rng.rand(700, 3).astype(_f)
    N = rng.normal(size=(700, 3)).astype(_f)
    same(oon.port(P, N, 1), ton.kruskal_orient(P, N, rows(P, 1)))


def test_finite_radius_splits_the_graph():
    rng = np.random.RandomState(6)
    A = rng.rand(300, 3).astype(_f) * 0.3
    B = A + _f(5)
    P = np.concatenate([A, B])
    N = rng.normal(size=(600, 3)).astype(_f)
    got = oon.port(P, N, 8, 0.5)
    assert got[2] == 2 and set(got[1].tolist()) == {0, 300}
    same(got, ton.kruskal_orient(P, N, rows(P, 8, 0.5)))
    got_vp = oon.port(P, N, 8, 0.5, viewpoint=(10, 10, 10))
    same(got_vp, ton.kruskal_orient(P, N, rows(P, 8, 0.5), (10, 10, 10)))
    # each component keeps its own anchor's rule: the halves are oriented independently
    assert got[2] == got_vp[2]


@pytest.mark.parametrize("swap", [False, True])
def test_viewpoint_tie_goes_to_the_smaller_index(swap):
    """two points equidistant from the viewpoint: the anchor is the smaller j, and the choice shows: the other one's
    normal would be the one negated to face the viewpoint"""
    P = np.array([[-1, 0, 0], [1, 0, 0]], _f)
    N = np.array([[1, 0, 0], [1, 0.1, 0]], _f)          # n0 faces the viewpoint at the origin, n1 does not
    if swap:
        P, N = P[::-1].copy(), N[::-1].copy()
    got = oon.port(P, N, 1, viewpoint=(0, 0, 0))
    same(got, ton.kruskal_orient(P, N, rows(P, 1), (0, 0, 0)))
    if swap:
        assert np.array_equal(got[0], -N)               # anchor 0 = the one facing away: both turned
    else:
        assert np.array_equal(got[0], N)


def test_dot_exactly_zero_is_no_flip():
    P = np.array([[0, 0, 0], [1, 0, 0]], _f)
    for N in (np.array([[1, 1, 0], [-0.0, -0.0, -1]], _f),   # every product -0: dot = -0
              np.array([[1, 0, 0], [0, 1, 0]], _f)):         # dot = +0
        d = ton.dots(N, np.array([0]), np.array([1]))[0]
        assert d == 0
        got = oon.port(P, N, 1)
        assert np.array_equal(common.bits(got[0]), common.bits(N)) and got[3].tolist() == [[0, 1]]
    N = np.array([[1, 1, 0], [-1e-30, 0, -1]], _f)            # just below zero: a flip
    assert np.array_equal(oon.port(P, N, 1)[0], np.array([N[0], -N[1]]))


def test_non_unit_normals():
    """lengths change |dot| and so the tree, never the rule: the outputs are the inputs' signs, as the restatement"""
    rng = np.random.RandomState(8)
    P = rng.rand(500, 3).astype(_f)
    N = (rng.normal(size=(500, 3)) * np.exp(rng.uniform(-6, 6, (500, 1)))).astype(_f)
    R = rows(P, 6)
    assert ton.distinct_weights(N, R)
    got = oon.port(P, N, 6, viewpoint=(0, 0, 4))
    same(got, ton.scipy_orient(P, N, R, (0, 0, 4)))
    signs_only(got[0], N)


def test_in_place():
    rng = np.random.RandomState(10)
    P = rng.rand(800, 3).astype(_f)
    N = rng.normal(size=(800, 3)).astype(_f)
    want = oon.port(P, N, 8, viewpoint=(0, 0, 3))
    M = N.copy()
    got = oon.port(P, M, 8, viewpoint=(0, 0, 3), out=M)
    assert got[0] is M
    same(got, want)


def test_errors():
    P = np.random.RandomState(0).rand(50, 3).astype(_f)
    N = np.random.RandomState(1).normal(size=(50, 3)).astype(_f)
    for k in (0, 65):
        with pytest.raises(oon.OrientError):
            oon.port(P, N, k)
    for r in (np.nan, -1.0):
        with pytest.raises(oon.OrientError):
            oon.port(P, N, 8, r)
    for bad in (np.nan, np.inf, -np.inf):
        M = N.copy()
        M[4, 1] = bad
        with pytest.raises(oon.OrientError):
            oon.port(P, M, 8)
        with pytest.raises(oon.OrientError):
            oon.port(P, N, 8, viewpoint=(0, bad, 0))
    oon.port(P, N, 64)                                     # 64 with 49 others: padded rows


def test_sphere_comes_out_outward():
    """a dense sphere: sign-scrambled true normals and PCA normals of the port both come out outward with a viewpoint
    outside, in one component"""
    X, T = ton.sphere(20000, 1)
    for N in (ton.scramble(T, 3), onormals.port(X, 16)[0]):
        for vp in ((0, 0, 5), (4, -3, 1)):
            o = oon.port(X, N, 16, viewpoint=vp)
            assert o[2] == 1
            assert ((o[0] * T).sum(1) > 0).all()
    # without a viewpoint the root's sign decides: all outward or all inward
    o = oon.port(X, ton.scramble(T, 4), 16)
    s = (o[0] * T).sum(1) > 0
    assert s.all() or (~s).all()


def test_torus_needs_more_than_the_per_point_viewpoint_rule():
    """on a torus no viewpoint is faced by every point: s4g_normals' per-point rule turns the far side and the inner
    ring inward; orientation along the forest from the anchor nearest the viewpoint turns every normal outward"""
    X, T = ton.torus(20000, 1)
    for k in (8, 16):
        Np, _ = onormals.port(X, k)
        for vp in ((0, 0, 5), (3, 0, 1)):
            per_point, _ = onormals.port(X, k, viewpoint=vp)
            inward = ((per_point * T).sum(1) < 0).mean()
            assert inward > 0.3, inward
            o = oon.port(X, Np, k, viewpoint=vp)
            assert o[2] == 1 and ((o[0] * T).sum(1) > 0).all()
        o = oon.port(X, ton.scramble(T, k), k, viewpoint=(0, 0, 5))
        assert ((o[0] * T).sum(1) > 0).all()


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    d = tmp_path_factory.mktemp("orient_normals")
    exe = ton.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


@pytest.mark.parametrize("vp", [None, (0.0, 0.0, 5.0)])
@pytest.mark.parametrize("max_distance", [np.inf, 0.08])
def test_cpp_function_on_oracle_shim(program, tmp_path, vp, max_distance):
    """the port's signs on the normals the points hold (set_normal of the input); a flipped normal through
    set_normal(-normal()), whose float32 arithmetic tests/normals.py restates; the returned component count"""
    exe, shim = program
    X, T = ton.torus(3000, 2)
    N = ton.scramble(T, 2) * _f(3)                          # not unit: set_normal renormalises on the way in
    held = tnormals.set_normal(N)
    threw, count, got = ton.run(exe, tmp_path, X, N, 12, max_distance, vp, preload=shim)
    assert not threw
    want = oon.port(X, held, 12, np.float32(max_distance) * np.float32(max_distance), vp)
    assert count == want[2]
    assert np.array_equal(common.bits(got), common.bits(ton.expected_held(held, want[0])))


def test_cpp_function_throws_and_keeps_the_cloud(program, tmp_path):
    exe, shim = program
    X, T = ton.torus(500, 3)
    N = ton.scramble(T, 3)
    held = tnormals.set_normal(N)
    for k, md in ((0, np.inf), (65, np.inf), (8, -1.0), (8, np.nan)):
        threw, count, got = ton.run(exe, tmp_path, X, N, k, md, preload=shim)
        assert threw and count == 0, (k, md)
        assert np.array_equal(common.bits(got), common.bits(held))
    threw, count, got = ton.run(exe, tmp_path, X[:0], N[:0], 8, preload=shim)
    assert not threw and count == 0 and len(got) == 0
