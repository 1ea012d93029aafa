"""Plane segmentation on the GPU: s4g_segment_planes over the resident P.

Every output -- labels, the plane records (float bits), offsets, members and hyp_counts -- is bit-equal to the port's
restatement (oracle/planes_port.cc) on 10, 10^4 and 10^6 points (a room, a cfg2 sample, a cfg3-style sample with 20 %
outliers), at hypothesis counts around the warp and k_plane_count's hypothesis tile (512) and cloud sizes around its
point tile (1024), at thresholds equal to a point's exact residual and one ulp either side, off-centre, on 10^4
coincident points, and over several rounds.  Two calls give the same bits, the _dev and host forms agree, the error
codes hold, Utils::SegmentPlanes equals Context, and on a table scene the plane's removal is what lets the Euclidean
clusters find the objects."""
import ctypes as C

import numpy as np
import pytest

from oracle import planes as op
from super4pcs_b200 import s4g
from tests import common, planes as tp
from tests.test_knn_gpu import make_ctx  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

S4G_OK, S4G_ERR_ARG, S4G_ERR_STATE = 0, 2, 3   # include/s4g.h


def same(got, want):
    for g, w, name in zip(got, want, ("labels", "planes", "offsets", "members", "hyp_counts")):
        assert g.dtype == w.dtype and g.shape == w.shape, (name, g.shape, w.shape)
        assert g.tobytes() == w.tobytes(), (name, g, w) if g.size < 20 else name


def check(ctx, P, threshold, H, max_planes=1, min_inliers=1, seed=0, refine=True):
    """the Context call against the port; returns the number of planes"""
    got = ctx.segment_planes(threshold, H, max_planes, min_inliers, seed, refine, hyp_counts=True)
    same(got, op.planes(P, threshold, H, max_planes, min_inliers, seed, refine, hyp_counts=True))
    return len(got[1])


def test_small_clouds(make_ctx):  # noqa: F811
    """10 points, and clouds of 3, 1023, 1024, 1025 and 2049 points around the point tile"""
    ctx = make_ctx()
    rng = np.random.RandomState(0)
    P = rng.uniform(-1, 1, (10, 3)).astype(np.float32)
    ctx.set_cloud_p(P, 0.1)
    for thr, H, R in ((0.5, 1, 1), (0.5, 31, 3), (1.0, 1000, 4), (0.05, 33, 2), (np.inf, 5, 2)):
        check(ctx, P, thr, H, R)
    for n in (3, 1023, 1024, 1025, 2049):
        Pn = tp.room(n, outliers=0.3, seed=n)[0]
        ctx.set_cloud_p(Pn, 0.05)
        for H, R in ((1, 2), (32, 3), (511, 2), (512, 2), (513, 3)):
            check(ctx, Pn, 0.02, H, R, min_inliers=2, seed=n + H)


@pytest.mark.parametrize("H", [1, 31, 32, 33, 511, 512, 513, 1000, 1025, 4096])
def test_room_10k(make_ctx, H):  # noqa: F811
    P = tp.room(10_000, outliers=0.1, seed=1)[0]
    ctx = make_ctx()
    ctx.set_cloud_p(P, 0.02)
    for refine, R, lo, seed in ((True, 4, 200, 0), (False, 2, 1, 5), (True, 1, 1, 2 ** 64 - 1)):
        check(ctx, P, 0.01, H, R, lo, seed, refine)


def test_full_size_samples(make_ctx):  # noqa: F811
    """1M points: a cfg2 P sample and a cfg3-style sample with 20 % uniform outliers (no dominant plane: the winner is
    whatever the counts say) and a 1M-point room (three rounds)"""
    ctx = make_ctx()
    for outliers in (0.0, 0.2):
        P = common.scenario(1_000_000, 0.3, 0.003, seed=42, outliers=outliers)["P"]
        ctx.set_cloud_p(P, 0.003)
        assert check(ctx, P, 0.003, 1000, max_planes=2) == 2
    P = tp.room(1_000_000, noise=0.002, seed=3)[0]
    ctx.set_cloud_p(P, 0.003)
    assert check(ctx, P, 0.01, 4096, max_planes=3) == 3
    assert check(ctx, P, 0.01, 256, max_planes=4, min_inliers=10_000, refine=False) == 3


def test_exact_residual_thresholds(make_ctx):  # noqa: F811
    """one hypothesis, no refit: thresholds at |r| of chosen points and one ulp either side; then the same thresholds
    with the refit and many hypotheses"""
    P = tp.room(10_000, noise=0.01, seed=6)[0]
    ctx = make_ctx()
    ctx.set_cloud_p(P, 0.02)
    pl = op.planes(P, 0.05, 1, refine=False)[1][0]["coefficients"]
    r = np.abs(((pl[0] * P[:, 0] + pl[1] * P[:, 1]) + pl[2] * P[:, 2]) + pl[3])
    for q in np.argsort(r)[[10, 1000, 3000]]:
        for t in (r[q], np.nextafter(r[q], np.float32(np.inf)), np.nextafter(r[q], np.float32(0))):
            check(ctx, P, float(t), 1, refine=False)
            check(ctx, P, float(t), 300, max_planes=2)


def test_off_centre_and_coincident(make_ctx):  # noqa: F811
    ctx = make_ctx()
    P = tp.room(20_000, seed=7, offset=(1e3, -2e3, 5e2))[0]
    ctx.set_cloud_p(P, 0.05)
    assert check(ctx, P, 0.01, 500, max_planes=3, min_inliers=100) >= 1
    same_pts = np.tile(np.float32([[0.3, -0.1, 0.2]]), (10_000, 1))
    ctx.set_cloud_p(same_pts, 0.01)
    assert check(ctx, same_pts, 1.0, 1000, max_planes=2) == 0
    mixed = np.concatenate([same_pts, tp.room(3000, seed=8)[0]])
    ctx.set_cloud_p(mixed, 0.02)
    check(ctx, mixed, 0.01, 1000, max_planes=3, min_inliers=50)
    check(ctx, mixed, 0.0, 100, max_planes=2)
    check(ctx, mixed, np.inf, 100, max_planes=2)


def test_repeatable_and_dev_form_equals_host_form(make_ctx):  # noqa: F811
    import torch
    P = tp.room(50_000, outliers=0.2, seed=9)[0]
    ctx = make_ctx()
    ctx.set_cloud_p(P, 0.02)
    n = len(P)
    for thr, H, R, lo, refine in ((0.01, 1000, 4, 1000, True), (0.02, 64, 2, 1, False), (0.0, 10, 2, 1, True)):
        want = ctx.segment_planes(thr, H, R, lo, 11, refine, hyp_counts=True)
        same(ctx.segment_planes(thr, H, R, lo, 11, refine, hyp_counts=True), want)
        dev = lambda k, dt: torch.full((k,), 7, dtype=dt, device="cuda")  # noqa: E731
        labels, members, offsets = dev(n, torch.int32), dev(n, torch.int32), dev(R + 1, torch.int64)
        planes, n_planes = torch.zeros(R * 64, dtype=torch.uint8, device="cuda"), dev(1, torch.int32)
        counts = torch.full((R, H), 7, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        ctx.segment_planes_dev(thr, labels.data_ptr(), planes.data_ptr(), n_planes.data_ptr(), offsets.data_ptr(),
                               members.data_ptr(), counts.data_ptr(), H, R, lo, 11, refine)
        ctx.synchronize()
        k = int(n_planes.item())
        off = offsets[:k + 1].cpu().numpy()
        got = (labels.cpu().numpy(), planes.cpu().numpy()[:64 * k].view(s4g.PLANE_DTYPE), off,
               members[:off[-1]].cpu().numpy(), counts.cpu().numpy().view(np.uint32))
        same(got, want)
        labels.fill_(7)
        torch.cuda.synchronize()
        ctx.segment_planes_dev(thr, labels.data_ptr(), planes.data_ptr(), n_planes.data_ptr(), n_hypotheses=H,
                               max_planes=R, min_inliers=lo, seed=11, refine=refine)   # the rest optional
        ctx.synchronize()
        assert np.array_equal(labels.cpu().numpy(), want[0]) and int(n_planes.item()) == k


def test_error_codes(s4g_lib):
    from super4pcs_b200 import Context
    with Context(0) as ctx:
        L, h = ctx._L, ctx.h
        lab, mem, off = np.empty(100, np.int32), np.empty(100, np.int32), np.empty(4, np.int64)
        pls, cnt = np.zeros(3, s4g.PLANE_DTYPE), np.empty(3 * 10, np.uint32)
        npl = C.c_int(0)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        pp = pls.ctypes.data_as(C.POINTER(s4g.Plane))

        def args(thr=0.1, H=10, R=3, lo=1, labels=True, planes=True, n_planes=True):
            return (h, thr, H, C.c_uint64(0), 1, R, lo, p(lab) if labels else None, pp if planes else None,
                    C.byref(npl) if n_planes else None, p(off), p(mem), p(cnt))
        assert L.s4g_segment_planes(*args()) == S4G_ERR_STATE
        assert "s4g_set_cloud_p" in L.s4g_error_string(h).decode()
        assert L.s4g_segment_planes_dev(*args()) == S4G_ERR_STATE
        ctx.set_cloud_p(np.random.RandomState(0).rand(100, 3).astype(np.float32), 0.05)
        bad = [dict(thr=float("nan")), dict(thr=-1e-30), dict(thr=-np.inf), dict(H=0), dict(H=2 ** 20 + 1), dict(H=-5),
               dict(R=0), dict(R=-1), dict(lo=0), dict(lo=-3), dict(labels=False), dict(planes=False),
               dict(n_planes=False)]
        for b in bad:
            assert L.s4g_segment_planes(*args(**b)) == S4G_ERR_ARG, b
            assert "n_hypotheses" in L.s4g_error_string(h).decode()
            assert L.s4g_segment_planes_dev(*args(**b)) == S4G_ERR_ARG, b
        assert L.s4g_segment_planes(None, 0.1, 10, C.c_uint64(0), 1, 3, 1, p(lab), pp, C.byref(npl), None, None,
                                    None) == S4G_ERR_ARG
        assert L.s4g_segment_planes(h, 0.1, 10, C.c_uint64(0), 1, 3, 1, p(lab), pp, C.byref(npl), None, None,
                                    None) == S4G_OK
        big = np.empty(2 ** 20, np.uint32)                                   # the largest count is allowed
        assert L.s4g_segment_planes(h, 0.1, 2 ** 20, C.c_uint64(0), 1, 1, 1, p(lab), pp, C.byref(npl), p(off), p(mem),
                                    p(big)) == S4G_OK
        assert npl.value == 1 and big.sum() > 0
        assert L.s4g_segment_planes(*args(thr=np.inf, R=3)) == S4G_OK
        assert npl.value == 1 and (lab == 0).all() and list(off[:2]) == [0, 100]
        with pytest.raises(Exception):
            ctx.segment_planes(0.1, 0)


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = tp.build(tmp_path_factory.mktemp("planes"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


@pytest.mark.parametrize("thr,R,lo,H,seed,refine", [(0.01, 3, 100, 1000, 0, True), (0.02, 1, 1, 50, 9, False),
                                                     (0.01, 5, 2000, 300, 3, True)])
def test_cpp_function_equals_context(program, make_ctx, tmp_path, thr, R, lo, H, seed, refine):  # noqa: F811
    P = tp.room(30_000, outliers=0.1, seed=10)[0]
    got = tp.run(program, tmp_path, P, thr, R, lo, H, seed, refine)
    assert got is not None and len(got) >= 1
    ctx = make_ctx()
    ctx.set_cloud_p(P, 0.02)
    _, planes, off, mem = ctx.segment_planes(thr, H, R, lo, seed, refine)
    assert len(got) == len(planes)
    for (coef, inl), pl, a, b in zip(got, planes, off[:-1], off[1:]):
        assert np.array_equal(coef.view(np.uint32), pl["coefficients"].view(np.uint32))
        assert np.array_equal(inl, mem[a:b])


def test_table_scene_end_to_end(make_ctx):  # noqa: F811
    """the motivation: the table top joins every object into one Euclidean cluster; with its plane segmented away the
    clusters are the objects"""
    P, lab = tp.table()
    ctx = make_ctx()
    ctx.set_cloud_p(P, 0.01)
    _, _, off, _ = ctx.euclidean_clusters(0.02 ** 2, 100)
    assert len(off) == 2 and off[1] == len(P)                           # one cluster: the whole scene
    labels, planes, offsets, members = ctx.segment_planes(0.01, 1000)
    same((labels, planes, offsets, members), op.planes(P, 0.01, 1000))
    assert len(planes) == 1 and (labels[lab == 0] == 0).all()
    rest = np.nonzero(labels < 0)[0]
    ctx.set_cloud_p(P[rest], 0.01)
    _, _, off, mem = ctx.euclidean_clusters(0.02 ** 2, 100)
    assert len(off) == 5                                                  # the four objects
    for c in range(4):
        idx = rest[mem[off[c]:off[c + 1]]]
        k = lab[idx[0]]
        assert k > 0 and (lab[idx] == k).all() and len(idx) >= 0.99 * np.sum(lab[rest] == k)
