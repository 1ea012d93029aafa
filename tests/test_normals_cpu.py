"""Normal estimation (s4g_normals) without a GPU: the port's restatement against numpy's float64 eigh of the same rows, its
sign and no-normal rules, its agreement with the hippo files' own normals, Utils::EstimateNormals of the C++ layer on the
oracle stand-in, and a registration that uses the estimated normals against the compiled reference.

Contract (include/s4g.h): the neighbourhood of P point j is its s4g_knn row (no T, no exclusion); centroid, covariance
and cyclic Jacobi in double; the normal is the eigenvector of the smallest eigenvalue, (0, 0, 0) when the row holds fewer
than 3 points or the covariance is exactly zero."""
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import _build, knn as oknn, normals as onormals, ref as oref
from tests import build_shim, common, edges as E, normals as tnormals

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = [3, 8, 16, 33, 64]
ASSETS = os.path.join(_build.REFERENCE_ROOT, "assets")


def rotated_plane(rng, n=2500):
    R = E.rotations(1, rng)[0]
    P = np.concatenate([rng.uniform(-0.5, 0.5, (n, 2)), np.zeros((n, 1))], 1) @ R.T + 0.1
    return P.astype(np.float32), R[:, 2]


def sphere(rng, n=2500, centre=(0.2, -0.1, 0.3), radius=0.7):
    d = rng.normal(0, 1, (n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return (np.float64(centre) + radius * d).astype(np.float32), d


def synthetic(seed=3, n=3000):
    from super4pcs_b200 import synth
    d = synth.make_pair(n, 0.6, seed=seed, with_normals=True)
    return d["P"].astype(np.float32), d["Pn"].astype(np.float64)


def line(rng, n=1500):
    u = rng.normal(0, 1, 3)
    u /= np.linalg.norm(u)
    return (rng.uniform(-0.5, 0.5, (n, 1)) * u + 0.05).astype(np.float32), u


def spacing(P):
    """a typical neighbour distance: the median distance to the nearest other point"""
    _, sq = oknn.bruteforce(P, P[:400], 2)
    return float(np.sqrt(np.median(sq[:, 1])))


def sin_angle(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.linalg.norm(np.cross(a / np.linalg.norm(a, axis=1, keepdims=True), b / np.linalg.norm(b, axis=1, keepdims=True)),
                          axis=1)


def check_against_eigh(P, k, r):
    """every row: eigenvalues within 1e-6 lambda2 of eigh's; where the relative gap (lambda1 - lambda0) / lambda2 is at
    least 1e-4, sin(angle to eigh's eigenvector) <= 1e-6; rows of fewer than 3 points get (0, 0, 0).  Returns (normals,
    the rows' m, the mask of gapped rows)"""
    n, ev, rows = onormals.port(P, k, r, rows=True)
    val, vec, m = onormals.eigh(P, rows)
    lam2 = np.maximum(val[:, 2], 0)
    assert (np.abs(ev.astype(np.float64) - val) <= 1e-6 * lam2[:, None] + 1e-30).all()
    assert (ev[:, 0] <= ev[:, 1]).all() and (ev[:, 1] <= ev[:, 2]).all()
    assert (n[m < 3] == 0).all()
    real = (m >= 3) & (lam2 > 0)
    assert (np.abs(np.linalg.norm(n[real].astype(np.float64), axis=1) - 1) < 1e-6).all()
    gap = real & ((val[:, 1] - val[:, 0]) >= 1e-4 * lam2)
    assert (sin_angle(n[gap], vec[gap][:, :, 0]) <= 1e-6).all()
    return n, m, gap


@pytest.mark.parametrize("kind", ["plane", "sphere", "synthetic", "offcentre1e3", "offcentre1.2e4"])
def test_port_equals_numpy_eigh(kind):
    rng = np.random.RandomState(7)
    truth = None
    if kind == "plane":
        P, normal = rotated_plane(rng)
        truth = np.tile(normal, (len(P), 1))
    elif kind == "sphere":
        P, truth = sphere(rng)
    elif kind == "synthetic":
        P, truth = synthetic()
    else:
        off = 1e3 if kind == "offcentre1e3" else 1.2e4
        P = (synthetic(seed=5)[0].astype(np.float64) * 0.3 + off).astype(np.float32)
    delta = spacing(P)
    gapped = 0
    for k in KS:
        for r in (delta * delta, 9 * delta * delta, np.inf):
            n, m, gap = check_against_eigh(P, k, r)
            gapped += int(gap.sum())
            if truth is not None and k >= 8 and r == np.inf:
                s = sin_angle(n, truth)
                if kind == "plane":
                    assert s.max() <= 1e-5                   # the float rounding of the points is the only noise
                else:
                    assert np.median(s) <= np.sin(np.radians(5 if kind == "sphere" else 10))
    assert gapped > 10000


def test_collinear_rows_are_perpendicular_to_the_line():
    rng = np.random.RandomState(3)
    P, u = line(rng)
    for k in (3, 16, 64):
        n, _, rows = onormals.port(P, k, rows=True)
        live = np.linalg.norm(n, axis=1) > 0
        assert live.mean() > 0.9
        line_dir = onormals.eigh(P, rows)[1][:, :, 2]              # each row's own line (the float points are not exactly on u)
        assert np.abs((n[live].astype(np.float64) * line_dir[live]).sum(1)).max() <= 1e-6
        assert np.abs(n[live].astype(np.float64) @ u).max() <= 1e-3


def test_sign_rules():
    """with a viewpoint the normal faces it; without, its largest component is positive, ties to the lowest axis"""
    rng = np.random.RandomState(4)
    P, truth = sphere(rng, 2000, centre=(0, 0, 0))
    n0, _ = onormals.port(P, 16)
    a = np.argmax(np.abs(n0), axis=1)
    assert (n0[np.arange(len(P)), a] > 0).all()
    inside, _ = onormals.port(P, 16, viewpoint=[0, 0, 0])          # the centre: every normal points inwards
    assert ((inside.astype(np.float64) * truth).sum(1) < 0).all()
    outside, _ = onormals.port(P, 16, viewpoint=[0, 0, 100])
    assert (((np.float64([0, 0, 100]) - P) * outside).sum(1) >= 0).all()
    assert np.array_equal(np.abs(n0), np.abs(inside)) and np.array_equal(np.abs(n0), np.abs(outside))
    # ties of the canonical rule: the planes x = y and y = z, whose normals are (1, -1, 0) / sqrt 2 and (0, 1, -1) / sqrt 2
    # up to sign
    for first in (0, 1):
        s, t = rng.uniform(-1, 1, (2, 600)).astype(np.float32)
        P = np.stack([s, s, t] if first == 0 else [t, s, s], 1)
        n, _ = onormals.port(P, 16)
        live = np.linalg.norm(n, axis=1) > 0
        tied = live & (np.abs(n[:, first]) == np.abs(n[:, first + 1])) & (np.abs(n[:, first]) >= np.abs(n[:, 2 - first * 2]))
        assert tied.sum() > 0
        assert (n[tied, first] > 0).all() and (n[tied, first + 1] < 0).all()


def test_no_normal_rules():
    rng = np.random.RandomState(5)
    P = rng.uniform(-1, 1, (400, 3)).astype(np.float32)
    P = np.concatenate([P, [[5, 5, 5]], [[-5, 5, 5], [-5, 5, 5.001]]]).astype(np.float32)   # one isolated point, one pair
    n, ev, rows = onormals.port(P, 8, 0.01, rows=True)
    m = (rows >= 0).sum(1)
    assert (m[-3:] == [1, 2, 2]).all() and (n[-3:] == 0).all()
    assert (n[m < 3] == 0).all() and (np.linalg.norm(n[m >= 3], axis=1) > 0).all()
    # a radius of 0 leaves every point alone: no normal anywhere, eigenvalues 0
    n, ev = onormals.port(P, 8, 0.0)
    assert (n == 0).all() and (ev == 0).all()
    # coincident points: more than k duplicates of one point, and exactly 3
    D = np.concatenate([np.tile([[0.3, 0.2, 0.1]], (80, 1)), np.tile([[2, 2, 2]], (3, 1)), rng.uniform(4, 5, (50, 3))])
    n, ev = onormals.port(D.astype(np.float32), 16, 0.5)
    assert (n[:83] == 0).all() and (ev[:83] == 0).all() and (np.linalg.norm(n[83:], axis=1) > 0).all()


def read_obj_normals(path):
    v, vn = [], []
    for ln in open(path):
        if ln.startswith("v "):
            v.append(ln.split()[1:4])
        elif ln.startswith("vn "):
            vn.append(ln.split()[1:4])
    return np.array(v, np.float32), np.array(vn, np.float64)


@pytest.mark.skipif(not os.path.exists(os.path.join(ASSETS, "hippo1.obj")), reason="the reference's assets are not present")
@pytest.mark.parametrize("name,key,floor", [("hippo1", "P", 0.876), ("hippo2", "Q", 0.840)])
def test_hippo_normals_agree_with_the_files(name, key, floor):
    """the share of points whose k = 8 normal lies within 10 degrees of the file's normal (up to sign; a zero file
    normal disagrees): 0.8770 (hippo1) and 0.8409 (hippo2) for the port, as for scipy's kd-tree + float64 PCA"""
    P, N = read_obj_normals(os.path.join(ASSETS, name + ".obj"))
    assert np.array_equal(P, np.load(os.path.join(ROOT, "tests", "golden", "hippo.npz"))[key])
    n, _ = onormals.port(P, 8)
    nn = np.linalg.norm(N, axis=1)
    cos = np.abs((n.astype(np.float64) * N).sum(1)) / np.where(nn > 0, nn, 1)
    share = float(((cos >= np.cos(np.radians(10))) & (nn > 0)).mean())
    assert floor <= share < floor + 0.01


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    d = tmp_path_factory.mktemp("normals")
    exe = tnormals.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


@pytest.mark.parametrize("kind", ["synthetic", "plane_viewpoint", "radius", "duplicates"])
def test_estimate_normals_on_oracle_shim(program, tmp_path, kind):
    """Utils::EstimateNormals on the stand-in: the port's normals through Point3D::set_normal, bit for bit, and the count
    of non-zero ones"""
    exe, shim = program
    rng = np.random.RandomState(8)
    k, dist, vp = 16, np.inf, None
    if kind == "synthetic":
        P = synthetic(seed=6, n=6000)[0]
    elif kind == "plane_viewpoint":
        P, vp = rotated_plane(rng, 3000)[0], np.float32([0.3, 2.0, -1.0])
    elif kind == "radius":
        P, k = synthetic(seed=7, n=4000)[0], 33
        dist = 2 * spacing(P)
    else:
        P, k = np.concatenate([np.tile([[0.1, 0.1, 0.1]], (70, 1)), rng.uniform(-1, 1, (500, 3))]).astype(np.float32), 64
    got = tnormals.run(exe, tmp_path, P, k, dist, vp, preload=shim)
    assert got is not None
    want, _ = onormals.port(P, k, np.float32(dist) * np.float32(dist), vp)
    assert np.array_equal(common.bits(got[1]), common.bits(tnormals.set_normal(want)))
    assert got[0] == int((np.abs(want).sum(1) > 0).sum()) > 0
    if kind == "duplicates":
        assert (got[1][:70] == 0).all()


def test_estimate_normals_throws_on_bad_arguments(program, tmp_path):
    exe, shim = program
    P = np.random.RandomState(1).rand(100, 3).astype(np.float32)
    for k, dist in ((2, np.inf), (65, np.inf), (8, -1.0), (8, np.nan)):
        assert tnormals.run(exe, tmp_path, P, k, dist, preload=shim) is None, (k, dist)


# the registration of tests/host_logic_driver.py's "synth2n" scenario, with estimated normals instead of analytic ones
REGISTRATION = dict(delta=0.02, overlap=0.6, sample_size=300, max_time_seconds=10000, random_seed=102,
                    max_normal_difference=40.0)
_DROPIN = """
import sys
import numpy as np
sys.path.insert(0, {root!r})
from oracle import _build, ref as oref
d = np.load({src!r})
score, T, Qt = oref.compute_transformation(d["P"], d["Q"], oref.make_options(**{kw!r}), Pn=d["Pn"], Qn=d["Qn"],
                                           libpath=_build.DROPIN_SO)
np.savez({dst!r}, score=np.float32(score), T=T, Qt=Qt)
"""


def registration_inputs(estimate):
    """the 30 000-point synthetic pair without normals, and normals estimate(cloud) for both clouds"""
    from super4pcs_b200 import synth
    d = synth.make_pair(30000, 0.6, seed=2, with_normals=False)
    return d["P"], d["Q"], estimate(d["P"]), estimate(d["Q"])


def register_both(P, Q, Pn, Qn, tmp_path, preload=None):
    """-> (reference, C++ layer) results (score, T, transformed Q) on the same inputs and normals"""
    opt = oref.make_options(**REGISTRATION)
    ref = oref.compute_transformation(P, Q, opt, Pn=Pn, Qn=Qn)
    src, dst = str(tmp_path / "in.npz"), str(tmp_path / "out.npz")
    np.savez(src, P=P, Q=Q, Pn=Pn, Qn=Qn)
    env = dict(os.environ)
    if preload:
        env["LD_PRELOAD"] = preload
    r = subprocess.run([sys.executable, "-c", _DROPIN.format(root=ROOT, src=src, dst=dst, kw=REGISTRATION)], env=env,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stderr[-3000:]
    o = np.load(dst)
    return ref, (float(o["score"]), o["T"], o["Qt"])


def same_registration(a, b):
    assert np.float32(a[0]) == np.float32(b[0])
    assert np.array_equal(common.bits(a[1]), common.bits(b[1]))
    assert np.array_equal(common.bits(a[2]), common.bits(b[2]))
    assert a[0] > 0.2


@pytest.mark.skipif(_build.build_ref() is None, reason="oracle/_ref (compiled reference) not present")
def test_registration_with_estimated_normals_on_oracle_shim(s4g_lib, tmp_path):
    from super4pcs_b200 import build_cpp
    if build_cpp.build_all()["lib"] is None or _build.build_dropin_harness() is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    P, Q, Pn, Qn = registration_inputs(lambda X: onormals.port(X, 16)[0])
    assert (np.abs(Pn).sum(1) > 0).mean() > 0.99 and (np.abs(Qn).sum(1) > 0).mean() > 0.99
    ref, ours = register_both(P, Q, Pn, Qn, tmp_path, preload=build_shim.build())
    same_registration(ref, ours)
