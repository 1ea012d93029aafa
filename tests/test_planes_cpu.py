"""Plane segmentation (s4g_segment_planes) without a GPU: the port's draws, hypothesis planes and every hypothesis count
against the numpy restatement of tests/planes.py, its refit against float64 eigh, its strict test at exact residuals,
the degenerate-cloud and stop rules of the contract, the planes of a labelled room, and the C++ layer's
Utils::SegmentPlanes on the oracle stand-in.

Contract (include/s4g.h): round r draws H hypotheses from A_r (the points no earlier plane claimed) with SplitMix64 of
seed + r, counts each exactly (fp32 |((a x + b y) + c z) + d| < threshold), takes the largest count (ties: smallest h),
refits it over its inliers in double, keeps the final inliers if there are at least min_inliers, else stops."""
import numpy as np
import pytest

from oracle import clusters as oc, planes as op
from tests import build_shim, planes as tp

U64 = 2 ** 64


def active_before(labels, r):
    """the ascending positions that no plane before round r claimed"""
    return np.nonzero((labels < 0) | (labels >= r))[0].astype(np.int32)


@pytest.mark.parametrize("kind", ["room", "outliers", "offcentre", "tiny"])
def test_draws_and_counts_equal_numpy(kind):
    """every round's draws, planes (bits, NaN where invalid) and hyp_counts row equal the numpy restatement"""
    if kind == "room":
        P = tp.room(6000, seed=1)[0]
    elif kind == "outliers":
        P = tp.room(6000, outliers=0.2, seed=2)[0]
    elif kind == "offcentre":
        P = tp.room(4000, seed=3, offset=(1e3, -2e3, 5e2))[0]
    else:
        P = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 0], [1, 0, 0]])   # repeated points: invalid draws
    for H, seed in ((1, 0), (33, 7), (500, U64 - 1), (257, 12345678901234567)):
        labels, planes, offsets, members, counts = op.planes(P, 0.01, H, max_planes=3, min_inliers=2, seed=seed,
                                                              hyp_counts=True)
        for r in range(3):
            act = active_before(labels, r)
            if r > len(planes) or len(act) < 3:                    # an earlier round stopped, or too few points
                assert (counts[r] == 0).all()
                continue
            s_np, pl_np, v_np = tp.hypotheses(P, act, H, (seed + r) % U64)
            s_po, pl_po, v_po = op.hypotheses(P, act, H, (seed + r) % U64)
            assert np.array_equal(s_np, s_po) and np.array_equal(v_np, v_po)
            assert np.array_equal(pl_np.view(np.uint32), pl_po.view(np.uint32))
            want = tp.counts(P, act, pl_np, 0.01)
            assert np.array_equal(want, op.counts(P, act, pl_po, 0.01))
            assert np.array_equal(counts[r], want), (kind, H, r)
            if r < len(planes):
                h = int(planes[r]["hypothesis_index"])
                key = np.where(v_np, want.astype(np.int64) * 2 ** 32 + (2 ** 32 - 1 - np.arange(H)), 0)
                assert h == int(np.argmax(key)) and planes[r]["hypothesis_inliers"] == want[h]
                assert np.array_equal(planes[r]["sample"], s_np[h])
                assert np.array_equal(planes[r]["hypothesis"].view(np.uint32), pl_np[h].view(np.uint32))
    if kind == "tiny":
        assert not tp.hypotheses(P, np.arange(5), 50, 0)[2].all()     # some draws repeat a point


def test_refit_agrees_with_eigh():
    """the refitted plane equals float64 eigh of its hypothesis' inliers within 2e-7 per coefficient (rounding to float)"""
    P, _, _ = tp.room(20000, noise=0.004, seed=4)
    for thr in (0.01, 0.02):
        labels, planes, offsets, members = op.planes(P, thr, 300, max_planes=3, seed=5)
        assert len(planes) == 3
        for r in range(3):
            act = active_before(labels, r)
            hp = planes[r]["hypothesis"]
            X = P[act].astype(np.float32)
            res = ((hp[0] * X[:, 0] + hp[1] * X[:, 1]) + hp[2] * X[:, 2]) + hp[3]
            I = X[np.abs(res) < np.float32(thr)].astype(np.float64)
            assert len(I) == planes[r]["hypothesis_inliers"]
            c = I.mean(0)
            w, V = np.linalg.eigh((I - c).T @ (I - c) / len(I))
            n = V[:, 0] * np.sign(V[np.argmax(np.abs(V[:, 0])), 0])
            want = np.concatenate([n, [-n @ c]])
            assert np.abs(planes[r]["coefficients"] - want).max() <= 2e-7, (r, planes[r]["coefficients"], want)


def test_threshold_at_exact_residual_flips_the_point():
    """one hypothesis (H = 1), no refit: a threshold of exactly |r| of a point leaves it out (strict), one ulp above takes
    it in, one ulp below leaves it out; the counts move by that point alone"""
    P, _, _ = tp.room(3000, noise=0.01, seed=6)
    _, planes, _, _ = op.planes(P, 0.05, 1, refine=False)
    pl = planes[0]["coefficients"]
    r = np.abs(((pl[0] * P[:, 0] + pl[1] * P[:, 1]) + pl[2] * P[:, 2]) + pl[3])
    order = np.argsort(r)
    tried = 0
    for q in order[[100, 500, 1000]]:
        if np.sum(r == r[q]) != 1:
            continue
        thr = r[q]
        got = {}
        for name, t in (("at", thr), ("up", np.nextafter(thr, np.float32(np.inf))), ("down", np.nextafter(thr, np.float32(0)))):
            labels, pls, _, _, cnt = op.planes(P, float(t), 1, refine=False, hyp_counts=True)
            assert pls[0]["n_inliers"] == cnt[0, 0] == tp.counts(P, np.arange(len(P)), pl[None], float(t))[0]
            got[name] = (labels[q], int(cnt[0, 0]))
        assert got["at"][0] == -1 and got["down"][0] == -1 and got["up"][0] == 0
        assert got["up"][1] == got["at"][1] + 1 and got["down"][1] <= got["at"][1]
        tried += 1
    assert tried >= 2


def test_degenerate_clouds():
    """nP < 3, all points coincident, all collinear: no plane and zero counts; all exactly coplanar: one plane holding
    every point at any threshold > 0 and none at 0; +inf takes every active point"""
    for n in (1, 2):
        labels, planes, offsets, members, cnt = op.planes(np.float32(np.random.rand(n, 3)), 0.1, 10, max_planes=2,
                                                          hyp_counts=True)
        assert len(planes) == 0 and (labels == -1).all() and list(offsets) == [0] and (cnt == 0).all()
    same = np.tile(np.float32([[0.3, -0.2, 0.1]]), (500, 1))
    labels, planes, offsets, members, cnt = op.planes(same, 1.0, 100, hyp_counts=True)
    assert len(planes) == 0 and (labels == -1).all() and (cnt == 0).all()
    t = np.linspace(-1, 1, 400, dtype=np.float32)[:, None]
    line = (np.float32([0.1, 0.2, 0.3]) + t * np.float32([1, 0, 0])).astype(np.float32)   # exactly collinear in fp32
    labels, planes, offsets, members = op.planes(line, 1.0, 100)
    assert len(planes) == 0
    g = np.arange(30, dtype=np.float32) / 10
    flat = np.stack(list(np.meshgrid(g, g, indexing="ij")) + [np.zeros((30, 30), np.float32)], -1).reshape(-1, 3)
    for thr, refine in ((1e-30, True), (0.5, False), (0.5, True)):
        labels, planes, offsets, members = op.planes(flat, thr, 20, max_planes=2, refine=refine)
        assert len(planes) == 1 and (labels == 0).all() and np.array_equal(members, np.arange(900))
        assert planes[0]["coefficients"].tolist() == [0, 0, 1, 0]
    assert len(op.planes(flat, 0.0, 20)[1]) == 0                   # |r| = 0 is not < 0
    P = tp.room(2000, seed=7)[0]
    labels, planes, offsets, members = op.planes(P, np.inf, 5, max_planes=3)
    assert len(planes) == 1 and (labels == 0).all() and planes[0]["n_inliers"] == len(P)


def test_min_inliers_and_max_planes_stop():
    P, lab, _ = tp.room(10000, seed=8)
    full = op.planes(P, 0.01, 200, max_planes=6, min_inliers=500)
    assert len(full[1]) == 3                                          # the leftovers hold no 500-point plane
    for R in (1, 2, 3):
        part = op.planes(P, 0.01, 200, max_planes=R, min_inliers=500)
        assert len(part[1]) == R
        assert part[1].tobytes() == full[1][:R].tobytes() and np.array_equal(part[2], full[2][:R + 1])
        assert np.array_equal(part[0], np.where(full[0] < R, full[0], -1))
    biggest = int(full[1][0]["n_inliers"])
    assert len(op.planes(P, 0.01, 200, max_planes=3, min_inliers=biggest + 1)[1]) == 0
    two = op.planes(P, 0.01, 200, max_planes=3, min_inliers=int(full[1][2]["n_inliers"]) + 1)
    assert len(two[1]) == 2 and (two[0] < 2).all()


@pytest.mark.parametrize("outliers", [0.0, 0.2])
def test_room_gives_its_three_planes(outliers):
    """a labelled room: three planes, each within 0.5 degrees of its true plane and within 2e-3 in d, each holding at
    least 97 % of its true points, and at most 2 % of its members from another plane"""
    P, lab, truth = tp.room(30000, noise=0.002, outliers=outliers, seed=9)
    labels, planes, offsets, members = op.planes(P, 0.01, 500, max_planes=4, min_inliers=2000)
    assert len(planes) == 3
    for r, k in enumerate((0, 1, 2)):                                # the largest first: floor, then wall 1, wall 2
        c = planes[r]["coefficients"].astype(np.float64)
        assert tp.angle_deg(c, truth[k]) < 0.5
        s = np.sign(np.dot(c[:3], truth[k][:3]))
        assert abs(s * c[3] - truth[k][3]) < 2e-3
        mem = members[offsets[r]:offsets[r + 1]]
        assert np.mean((lab[mem] == k) | (lab[mem] == -1)) >= 0.98     # the rest: other planes' points near a corner
        assert np.mean(labels[lab == k] == r) >= 0.97


def test_table_scene_clusters_after_plane_removal():
    """the motivation: on a table scene the table top joins every object into one radius-0.02 component; with the top's
    plane removed the components are the objects (scipy's components, float64)"""
    P, lab = tp.table(n_plane=40000, n_object=3000)
    root = oc.scipy_roots(P, 0.02)
    assert len(np.unique(root)) == 1
    labels, planes, offsets, members = op.planes(P, 0.01, 200)
    assert len(planes) == 1 and tp.angle_deg(planes[0]["coefficients"], [0, 0, 1]) < 0.1
    assert (labels[lab == 0] == 0).all()
    rest = np.nonzero(labels < 0)[0]
    root = oc.scipy_roots(P[rest], 0.02)
    comps = [rest[root == r] for r in np.unique(root)]
    big = [c for c in comps if len(c) >= 100]
    assert len(big) == 4 and sum(len(c) for c in big) >= 0.999 * len(rest)
    for c in big:
        k = lab[c[0]]
        assert k > 0 and (lab[c] == k).all() and len(c) >= 0.99 * np.sum(lab[rest] == k)


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    d = tmp_path_factory.mktemp("planes")
    exe = tp.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


@pytest.mark.parametrize("thr,R,lo,H,seed,refine", [(0.01, 3, 100, 200, 0, True), (0.02, 1, 1, 50, 9, False),
                                                     (0.01, 5, 2000, 300, 3, True)])
def test_cpp_function_on_oracle_shim(program, tmp_path, thr, R, lo, H, seed, refine):
    """SegmentPlanes through the stand-in equals the port: the same planes (coefficient bits) and inlier lists"""
    exe, shim = program
    P = tp.room(8000, outliers=0.1, seed=10)[0]
    got = tp.run(exe, tmp_path, P, thr, R, lo, H, seed, refine, preload=shim)
    assert got is not None
    _, planes, off, mem = op.planes(P, thr, H, R, lo, seed, refine)
    assert len(got) == len(planes) and len(got) >= 1
    for (coef, inl), pl, a, b in zip(got, planes, off[:-1], off[1:]):
        assert np.array_equal(coef.view(np.uint32), pl["coefficients"].view(np.uint32))
        assert np.array_equal(inl, mem[a:b])


def test_cpp_function_throws_on_bad_arguments(program, tmp_path):
    exe, shim = program
    P = np.random.RandomState(1).rand(100, 3).astype(np.float32)
    for thr, R, lo, H in ((-1.0, 1, 1, 10), (float("nan"), 1, 1, 10), (0.1, 0, 1, 10), (0.1, 1, 0, 10), (0.1, 1, 1, 0),
                          (0.1, 1, 1, 2 ** 20 + 1)):
        assert tp.run(exe, tmp_path, P, thr, R, lo, H, preload=shim) is None, (thr, R, lo, H)
    assert tp.run(exe, tmp_path, P[:0], 0.1, preload=shim) == []
