"""s4g_normals on the GPU: PCA normals of k-nearest neighbourhoods of the resident P.

normals and eigenvalues are bit-equal to the port's restatement (oracle/normals_port.cc on the brute-force rows of
oracle/knn_port.cc) over the grid regimes of the k-nearest tests, degenerate clouds, every k_knn capacity instance, with
and without a viewpoint, and on 20 000 sampled points of a 1M-point cloud.  The _dev and host forms agree, the error codes
hold, Utils::EstimateNormals of the C++ layer equals Context.normals, and a registration with GPU-estimated normals is the
compiled reference's, bit for bit."""
import ctypes as C
import os

import numpy as np
import pytest

from oracle import _build, normals as onormals
from tests import common, edges as E, normals as tnormals
from tests.test_decision_edges_gpu import cloud
from tests.test_knn_gpu import make_ctx  # noqa: F401  (fixture)
from tests.test_normals_cpu import register_both, registration_inputs, same_registration

pytestmark = pytest.mark.gpu

S4G_OK, S4G_ERR_ARG, S4G_ERR_STATE = 0, 2, 3   # include/s4g.h
KS = [3, 8, 9, 16, 17, 32, 33, 64]             # both sides of every k_knn capacity (8, 16, 32, 64 slots)
VIEW = np.float32([0.3, -2.0, 1.5])


def same(a, b, what=""):
    assert np.array_equal(common.bits(a[0]), common.bits(b[0])), (what, np.argwhere(a[0] != b[0])[:5])
    assert np.array_equal(common.bits(a[1]), common.bits(b[1])), what


def check(ctx, P, delta, ks=KS, radii=None):
    radii = [delta * delta, 9 * delta * delta, np.inf] if radii is None else radii
    live = 0
    for k in ks:
        for r in radii:
            for vp in (None, VIEW):
                got = ctx.normals(k, r, vp)
                same(got, onormals.port(P, k, r, vp), (k, r, vp is None))
                live += int((np.abs(got[0]).sum(1) > 0).sum())
    return live


@pytest.mark.parametrize("name,cshift_min", [("centred", None), ("centred", 3), ("brick8", None), ("widened", None),
                                             ("offcentre1e3", None), ("offcentre1e4", None)])
def test_bit_equal_to_port_over_grid_regimes(make_ctx, name, cshift_min):  # noqa: F811
    delta = E.REGIMES[name][0]
    P, _, _ = cloud(name, cshift_min=cshift_min or 1)
    ctx = make_ctx(cshift_min)
    ctx.set_cloud_p(P, delta)
    assert check(ctx, P, delta) > 0


@pytest.mark.parametrize("kind", ["identical", "planar", "line", "duplicates", "single", "fewer_than_k"])
def test_bit_equal_to_port_on_degenerate_clouds(make_ctx, kind):  # noqa: F811
    rng = np.random.RandomState(11)
    delta = 0.01
    if kind == "identical":
        P = np.tile([[0.1, -0.2, 0.3]], (300, 1))
    elif kind == "planar":
        P = np.concatenate([rng.uniform(-0.3, 0.3, (4000, 2)), np.zeros((4000, 1))], 1)
    elif kind == "line":
        P = np.concatenate([rng.uniform(-0.5, 0.5, (3000, 1)), np.zeros((3000, 2))], 1)
    elif kind == "duplicates":
        P0 = rng.uniform(-0.2, 0.2, (2000, 3))
        P = np.concatenate([P0, P0[::3], P0[::2], np.tile(P0[:1], (70, 1))])
    elif kind == "single":
        P = np.array([[0.1, -0.2, 0.3]])
    else:
        P = rng.uniform(-0.05, 0.05, (20, 3))
    P = P.astype(np.float32)
    ctx = make_ctx()
    ctx.set_cloud_p(P, delta)
    check(ctx, P, delta)
    n, _ = ctx.normals(64)
    if kind in ("identical", "single"):
        assert (n == 0).all()
    if kind == "planar":
        assert (n[np.abs(n).sum(1) > 0] == np.float32([0, 0, 1])).all()


def test_full_size_sample(make_ctx):  # noqa: F811
    """1M points (cfg2, delta = 0.003), unbounded, k = 16: 20 000 sampled points against the port"""
    n, delta = 1_000_000, 0.003
    sc = common.scenario(n, 0.3, delta, seed=42)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], delta)
    sub = np.random.RandomState(0).choice(n, 20000, replace=False)
    for vp, rows in ((None, sub), (VIEW, sub[:2000])):
        got = ctx.normals(16, np.inf, vp)
        want = onormals.port(sc["P"], 16, np.inf, vp, which=rows)
        same((got[0][rows], got[1][rows]), want)
        assert (np.abs(got[0]).sum(1) > 0).mean() > 0.99


def test_dev_form_equals_host_form(make_ctx):  # noqa: F811
    import torch
    sc = common.scenario(20000, 0.4, 0.01, seed=5)
    ctx = make_ctx()
    ctx.set_cloud_p(sc["P"], 0.01)
    n = len(sc["P"])
    for k in (3, 16, 64):
        for r in (0.01 ** 2, np.inf):
            for vp in (None, VIEW):
                want = ctx.normals(k, r, vp)
                dn = torch.full((n, 3), 7, dtype=torch.float32, device="cuda")
                de = torch.full((n, 3), 7, dtype=torch.float32, device="cuda")
                torch.cuda.synchronize()
                ctx.normals_dev(k, dn.data_ptr(), de.data_ptr(), r, vp)
                ctx.synchronize()
                same((dn.cpu().numpy(), de.cpu().numpy()), want)
    dn = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
    ctx.normals_dev(8, dn.data_ptr(), None)                     # eigenvalues are optional
    ctx.synchronize()
    assert np.array_equal(dn.cpu().numpy(), ctx.normals(8)[0])


def test_error_codes(s4g_lib):
    from super4pcs_b200 import Context
    with Context(0) as ctx:
        L, h = ctx._L, ctx.h
        out = np.empty((100, 3), np.float32)
        p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
        assert L.s4g_normals(h, 8, float("inf"), None, p(out), None) == S4G_ERR_STATE     # before s4g_set_cloud_p
        assert "s4g_set_cloud_p" in L.s4g_error_string(h).decode()
        assert L.s4g_normals_dev(h, 8, float("inf"), None, p(out), None) == S4G_ERR_STATE
        ctx.set_cloud_p(np.random.RandomState(0).rand(100, 3).astype(np.float32), 0.05)
        for k in (2, 65, 0, -1):
            assert L.s4g_normals(h, k, 1.0, None, p(out), None) == S4G_ERR_ARG
            assert "k" in L.s4g_error_string(h).decode()
            assert L.s4g_normals_dev(h, k, 1.0, None, p(out), None) == S4G_ERR_ARG
        for r in (float("nan"), -1.0, -float("inf")):
            assert L.s4g_normals(h, 8, r, None, p(out), None) == S4G_ERR_ARG
        assert L.s4g_normals(h, 8, 1.0, None, None, p(out)) == S4G_ERR_ARG
        assert L.s4g_normals_dev(h, 8, 1.0, None, None, None) == S4G_ERR_ARG
        assert L.s4g_normals(None, 8, 1.0, None, p(out), None) == S4G_ERR_ARG
        assert L.s4g_normals(h, 3, 0.0, None, p(out), None) == S4G_OK                 # radius 0: every point alone
        assert (out == 0).all()
        with pytest.raises(Exception):
            ctx.normals(1)


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    exe = tnormals.build(tmp_path_factory.mktemp("normals"))
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe


@pytest.mark.parametrize("which", ["hippo", "synthetic"])
def test_cpp_estimate_normals_equals_context_normals(program, make_ctx, tmp_path, which):  # noqa: F811
    """Utils::EstimateNormals on the real library: Context.normals on the same cloud at the rule's delta, through
    Point3D::set_normal"""
    if which == "hippo":
        P, k, dist, vp = np.load(os.path.join(tnormals.ROOT, "tests", "golden", "hippo.npz"))["P"], 8, np.inf, None
    else:
        from super4pcs_b200 import synth
        P, k, dist, vp = synth.make_pair(30000, 0.6, seed=2)["P"], 33, 0.05, VIEW
    got = tnormals.run(program, tmp_path, P, k, dist, vp)
    assert got is not None
    ctx = make_ctx()
    ctx.set_cloud_p(P, tnormals.grid_delta(P, k))
    want, _ = ctx.normals(k, np.float32(dist) * np.float32(dist), vp)
    assert np.array_equal(common.bits(got[1]), common.bits(tnormals.set_normal(want)))
    assert got[0] == int((np.abs(want).sum(1) > 0).sum()) > 0


def test_registration_with_gpu_estimated_normals_equals_reference(s4g_lib, tmp_path):
    """the synthetic registration of the CPU tests with normals from the GPU: the C++ layer on the real library against
    the compiled reference, both given the same normals"""
    from super4pcs_b200 import Context, build_cpp
    if not _build.build_ref() or build_cpp.build_all()["lib"] is None or _build.build_dropin_harness() is None:
        pytest.skip("oracle/_ref or the C++ layer not present")

    def estimate(X):
        with Context(0) as ctx:
            ctx.set_cloud_p(X, tnormals.grid_delta(X, 16))
            return ctx.normals(16)[0]
    P, Q, Pn, Qn = registration_inputs(estimate)
    same_registration(*register_both(P, Q, Pn, Qn, tmp_path))
