"""s4g_fpfh and s4g_fpfh_match on the CPU: the port (oracle/fpfh_port.cc) against Open3D's formulas restated in numpy
float64 (atan2, acos, S_h interleaved) on smooth random surfaces, and against the contract restated in plain Python
doubles where decisions flip; the boundary table; the permutation and normal-negation properties; the match against a
numpy float32 restatement; the errors; and Utils::ComputeFPFH / Utils::MatchFPFH on the oracle stand-in."""
import math

import numpy as np
import pytest

from oracle import fpfh as ofpfh, knn as oknn, normals as onormals
from tests import build_shim, common, fpfh as tf, normals as tnormals

_f = np.float32


def rows_of(P, k, r=np.inf):
    n = len(P)
    return oknn.bruteforce(P, P, k, r, exclude=np.arange(n, dtype=np.int32))


def clean(P, N, k, r):
    """the port and Open3D's restatement on the same rows -> (port fpfh, port spfh, o3d fpfh, o3d spfh, margin, rows)"""
    R, S = rows_of(P, k, r)
    got, sp = ofpfh.port(P, N, k, r, spfh=True)
    want, wsp, margin = tf.open3d_fpfh(P, N, R, S)
    return got, sp, want, wsp, margin, R


@pytest.mark.parametrize("k", [1, 8, 32, 64])
@pytest.mark.parametrize("r", [np.inf, 0.02])
def test_port_against_open3d_formulas(k, r):
    """bins equal for every pair more than 1e-9 from a face; descriptors within rtol 1e-5 where every pair that feeds
    them is that far"""
    P = tf.surface(1500, seed=k)
    N = onormals.port(P, 16)[0]
    got, sp, want, wsp, margin, R = clean(P, N, k, r)
    far = margin > 1e-9                                    # row entries far from every face (and padding)
    ok_pt = far.all(1)
    assert ok_pt.mean() > 0.9 and (R >= 0).sum() > 500, "the inputs must hold pairs away from the faces"
    assert (margin[np.isfinite(margin)] < 1e-3).any(), "and some near them"
    cnt_port = np.rint(sp * (R >= 0).sum(1)[:, None] / 100.0)
    cnt_o3d = np.rint(wsp * (R >= 0).sum(1)[:, None] / 100.0)
    assert np.array_equal(cnt_port[ok_pt], cnt_o3d[ok_pt])
    feeds = ok_pt & np.array([ok_pt[R[j][R[j] >= 0]].all() for j in range(len(P))])
    assert feeds.mean() > 0.8
    np.testing.assert_allclose(got[feeds], want[feeds], rtol=1e-5, atol=1e-5)


def test_boundary_table():
    try:
        import mpmath
        mpmath.mp.prec = 200
        for i in range(1, 6):
            b = -mpmath.pi + 2 * mpmath.pi * i / 11
            c, s = tf.face(i)
            assert c == float(mpmath.cos(b)) and s == float(mpmath.sin(b)), i
    except ImportError:
        for i in range(1, 6):
            b = -math.pi + 2 * math.pi * i / 11
            c, s = tf.face(i)
            assert abs(c - math.cos(b)) <= math.ulp(c) and abs(s - math.sin(b)) <= math.ulp(s), i
    for i in range(1, 6):
        assert tf.face(11 - i) == (tf.face(i)[0], -tf.face(i)[1])


def test_f1_rule_against_atan2():
    rng = np.random.RandomState(0)
    for x, y in rng.normal(size=(20000, 2)):
        t = 11 * (math.atan2(y, x) + math.pi) / (2 * math.pi)
        if abs(t - round(t)) > 1e-9:
            assert tf.contract_f1_bin(x, y) == min(max(int(math.floor(t)), 0), 10)
    for i in range(1, 11):                                  # on a face: the upper bin
        c, s = tf.face(i)
        assert tf.contract_f1_bin(c, s) == i, i
    assert tf.contract_f1_bin(-1.0, 0.0) == 10 and tf.contract_f1_bin(-1.0, -0.0) == 10
    assert tf.contract_f1_bin(0.0, 0.0) == 5 and tf.contract_f1_bin(1.0, 0.0) == 5 and tf.contract_f1_bin(1.0, -0.0) == 5


def port_vs_contract(P, N, k, r=np.inf):
    R, S = rows_of(P, k, r)
    got = ofpfh.port(P, N, k, r)
    want = tf.contract_fpfh(P, N, R, S)
    assert np.array_equal(common.bits(got), common.bits(want))
    return got


def pair_cloud(p2, n1, n2):
    return np.array([[0, 0, 0], p2], _f), np.array([n1, n2], _f)


def spfh_bins(P, N):
    """the port's SPFH bins of point 0 of a two-point cloud"""
    _, sp = ofpfh.port(P, N, 1, spfh=True)
    return tuple(np.nonzero(sp[0])[0])


@pytest.mark.parametrize("case, want", [
    ("coincident", (5, 16, 27)),
    ("dp_parallel_n1", (5, 16, 27)),
])
def test_degenerate_pairs(case, want):
    if case == "coincident":
        P, N = pair_cloud([0, 0, 0], [0, 0, 1], [1, 0, 0])
    else:
        P, N = pair_cloud([0, 0, 2], [0, 0, 1], [0, 0, 1])          # a1 = a2 = 1, v = dp x n1 = 0
    assert spfh_bins(P, N) == want
    port_vs_contract(P, N, 1)


def test_equal_angles_do_not_swap():
    """|a1| = |a2| = 2 / sqrt(29) exactly (the lengths are sqrt(29) from exact integer sums): no swap gives f3 = a1 in bin
    29, where a swap (|a1| <= |a2|) would give f3 = -a2 in bin 25; f1 = atan2(2, 24) and f2 = -3 / sqrt(29)"""
    P, N = pair_cloud([1, 0, 0], [2, 0, 5], [2, 3, 4])
    assert spfh_bins(P, N)[:3] == (5, 13, 29)
    assert tf.contract_pair(P[0], tf.contract_normal(N[0]), P[1], tf.contract_normal(N[1])) == (5, 13, 29)
    port_vs_contract(P, N, 1)


@pytest.mark.parametrize("x, y, want", [(-1.0, 0.0, 10), (-1.0, -0.0, 10), (0.0, 0.0, 5), (1.0, 0.0, 5), (1.0, -0.0, 5),
                                        (0.0, 1.0, 8), (0.0, -1.0, 2)])
def test_f1_zero_y(x, y, want):
    assert tf.contract_f1_bin(x, y) == want


@pytest.mark.parametrize("n2, want", [((0, 0, -1), (10, 16, 27)), ((0, 0, 1), (5, 16, 27))])
def test_f1_y_zero_in_the_port(n2, want):
    """n1 = (0, 0, 1), dp = (1, 0, 0): no swap (a1 = a2 = 0), v = (0, -1, 0), w = (1, 0, 0), so y = w . n2 = 0 exactly and
    x = n2_z: bin 10 for x < 0, 5 for x > 0; f2 = f3 = 0 land in bins 16 and 27"""
    P, N = pair_cloud([1, 0, 0], [0, 0, 1], n2)
    assert tf.contract_pair(P[0], (0.0, 0.0, 1.0), P[1], tf.contract_normal(N[1])) == want
    _, sp = ofpfh.port(P, N, 1, spfh=True)
    assert tuple(np.nonzero(sp[0])[0]) == want
    port_vs_contract(P, N, 1)


def test_pairs_on_faces():
    """tests/fpfh.py's face_pairs: rows whose f1 face test lies within about 1e-14 of zero, and rows whose f2, f3 or swap
    decision lies exactly on its face, so that only the contract's rounding decides.  The vectorised and the scalar
    restatements agree on every bin, the port equals the contract bit for bit, and each wrong form a kernel could take
    (f1 by atan2, reassociated dot products, a swap on |a1| <= |a2|) changes some bin"""
    P, N, kind = tf.face_pairs()
    m = len(kind)
    bins, margin = tf.contract_pairs_np(P[:m], N[:m], P[m:], N[m:])
    assert (margin["f1"][kind == 1] < 1e-14).sum() >= 200 and (margin["f1"][kind == 1] < 1e-15).sum() >= 40
    for k, name in ((2, "f2"), (3, "f3"), (4, "swap")):
        assert (kind == k).sum() >= 20 and (margin[name][kind == k] < 1e-15).all(), name
    scalar = np.array([tf.contract_pair(P[j], tf.contract_normal(N[j]), P[m + j], tf.contract_normal(N[m + j]))
                       for j in range(m)])
    assert np.array_equal(scalar, bins)
    for flag in ("f1_atan2", "dot_right", "swap_le"):
        wrong, _ = tf.contract_pairs_np(P[:m], N[:m], P[m:], N[m:], **{flag: True})
        assert (wrong != bins).any(), flag
    port_vs_contract(P, N, 1)
    port_vs_contract(P, -N, 1)


def test_normals_zero_non_unit_non_finite():
    P = tf.surface(200, seed=3)
    N = onormals.port(P, 16)[0].copy()
    N[::7] *= 3.5                                              # not unit: divided by their length
    N[1] = 0
    N[2] = [np.nan, 0, 1]
    N[3] = [np.inf, 0, 0]
    got = port_vs_contract(P, N, 12)
    assert not got[1].any() and not got[2].any() and not got[3].any()
    base = ofpfh.port(P, onormals.port(P, 16)[0], 12)
    assert not np.array_equal(base, got)


def test_tiny_clouds():
    P = np.array([[0, 0, 0]], _f)
    assert not ofpfh.port(P, [[0, 0, 1]], 8).any()            # nP = 1: an empty row
    P = np.array([[0, 0, 0], [1, 0, 0.5]], _f)
    got = port_vs_contract(P, np.array([[0, 0, 1], [0.3, 0, 1]], _f), 8)
    assert np.isclose(got[0].sum(), 300.0 * 2, rtol=1e-6)    # each block: spfh 100 + the neighbour's, scaled to 100


def test_radius_that_empties_rows():
    P = tf.surface(300, seed=5)
    N = onormals.port(P, 16)[0]
    got = port_vs_contract(P, N, 16, 1e-12)
    assert not got.any()                                      # every row empty: m = 0 and S_h = 0 everywhere


def test_m_zero_row_with_described_neighbours():
    """point 0 has a normal but its only neighbour has none: m_0 = 0 and spfh_0 = 0; its acc is empty too.  Point 2,
    whose neighbours have descriptors, gets them"""
    P = np.array([[0, 0, 0], [0.1, 0, 0], [5, 0, 0], [5.1, 0.1, 0], [5.1, -0.1, 0.05]], _f)
    N = np.array([[0, 0, 1], [0, 0, 0], [0, 0.1, 1], [0.1, 0, 1], [0, 0, 1]], _f)
    got = port_vs_contract(P, N, 1)
    assert not got[0].any() and not got[1].any() and got[2].any()
    got = port_vs_contract(P, N, 2)
    assert not got[1].any()


def test_permutation():
    """on a cloud whose rows have distinct d^2, including the first one beyond the row (so no tie decides which index is
    in a row or where), permuting the input permutes the descriptors bit for bit"""
    P = tf.surface(800, seed=9)
    N = onormals.port(P, 16)[0]
    _, S = rows_of(P, 17)
    assert np.isfinite(S).all() and (np.diff(S, axis=1) > 0).all()
    perm = np.random.RandomState(1).permutation(len(P))
    a = ofpfh.port(P, N, 16)
    b = ofpfh.port(P[perm], N[perm], 16)
    assert np.array_equal(common.bits(a[perm]), common.bits(b))


def test_negated_normals_mirror_f1_and_f3():
    P = tf.surface(1000, seed=11)
    N = onormals.port(P, 16)[0]
    R, S = rows_of(P, 16)
    _, _, margin = tf.open3d_pairs(P, N, R)
    # the inputs hold no pair within rounding of a face, so the mirrored bins are exactly the mirrored rule's
    assert (margin > 1e-9).all()
    a = ofpfh.port(P, N, 16)
    b = ofpfh.port(P, -N, 16)
    want = a.copy()
    want[:, 0:11] = a[:, 10::-1]
    want[:, 22:33] = a[:, 32:21:-1]
    assert np.array_equal(common.bits(b), common.bits(want))


@pytest.mark.parametrize("na, nb", [(0, 5), (5, 0), (1, 1), (1, 40), (40, 1), (300, 200)])
@pytest.mark.parametrize("mutual", [False, True])
def test_match_against_numpy(na, nb, mutual):
    rng = np.random.RandomState(na * 7 + nb)
    A = rng.uniform(0, 50, (na, 33)).astype(_f)
    B = rng.uniform(0, 50, (nb, 33)).astype(_f)
    if nb > 3:
        B[3] = B[1]                                            # duplicate rows: the smaller index wins
        B[2] = np.nan                                          # a NaN row never wins
    if na > 2:
        A[1] = np.nan                                          # no finite d^2: -1, +inf
        A[2] = B[min(1, nb - 1)] if nb else A[2]
    got = ofpfh.match_port(A, B, mutual)
    want = tf.match_numpy(A, B, mutual)
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(common.bits(got[1]), common.bits(want[1]))
    if na > 2 and nb > 3:
        assert got[0][1] == -1 and got[1][1] == np.inf and got[0][2] in (1, -1)


def test_errors():
    P = tf.surface(50, seed=1)
    N = onormals.port(P, 16)[0]
    for k, r in ((0, np.inf), (65, np.inf), (8, -1.0), (8, np.nan)):
        with pytest.raises(ofpfh.FPFHError):
            ofpfh.port(P, N, k, r)


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    d = tmp_path_factory.mktemp("fpfh")
    exe = tf.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


@pytest.mark.parametrize("max_distance", [np.inf, 0.15])
def test_cpp_compute_on_oracle_shim(program, tmp_path, max_distance):
    exe, shim = program
    P = tf.surface(1200, seed=4)
    N = onormals.port(P, 16)[0] * _f(2)
    held = tnormals.set_normal(N)
    got = tf.run_compute(exe, tmp_path, P, N, 24, max_distance, preload=shim)
    want = ofpfh.port(P, held, 24, np.float32(max_distance) * np.float32(max_distance))
    assert np.array_equal(common.bits(got), common.bits(want))


def test_cpp_match_on_oracle_shim(program, tmp_path):
    exe, shim = program
    rng = np.random.RandomState(2)
    A, B = rng.uniform(0, 9, (150, 33)).astype(_f), rng.uniform(0, 9, (170, 33)).astype(_f)
    B[:100] = A[:100] + rng.normal(0, 0.01, (100, 33)).astype(_f)
    for mutual in (False, True):
        got = tf.run_match(exe, tmp_path, A, B, mutual, preload=shim)
        assert np.array_equal(got, ofpfh.match_port(A, B, mutual)[0])
    assert len(tf.run_match(exe, tmp_path, A[:0], B, True, preload=shim)) == 0
    assert (tf.run_match(exe, tmp_path, A, B[:0], True, preload=shim) == -1).all()


def test_cpp_errors(program, tmp_path):
    exe, shim = program
    P = tf.surface(100, seed=4)
    N = onormals.port(P, 16)[0]
    for k, md in ((0, np.inf), (65, np.inf), (8, -1.0), (8, np.nan)):
        assert tf.run_compute(exe, tmp_path, P, N, k, md, preload=shim) is None, (k, md)
    assert len(tf.run_compute(exe, tmp_path, P[:0], N[:0], 8, preload=shim)) == 0
