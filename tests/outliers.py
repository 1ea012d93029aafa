"""Builds and runs tests/cpp/outliers_main.cc, the test program of Utils::RemoveStatisticalOutliers and
Utils::RemoveRadiusOutliers, for tests/test_outliers_cpu.py (on the oracle stand-in) and tests/test_outliers_gpu.py (on the
real library), and the stand-in's companion that answers the two filters on the CPU (tests/stubs/s4g_outliers_shim.cc).
Also the rules of the grid delta of the two functions, and a cloud of surface points and uniform outliers whose labels are
known."""
import os
import subprocess

import numpy as np

from tests import knn as tknn, normals as tnormals

ROOT = tknn.ROOT
_f = np.float32


def build(outdir):
    """compiles the program into `outdir` against the C++ layer; None when the layer or Eigen is missing"""
    from oracle import _build
    from super4pcs_b200 import build_cpp
    if build_cpp.build_all()["lib"] is None:
        return None
    eig = None
    for c in (os.environ.get("S4_EIGEN_ROOT"), os.path.join(_build.REFERENCE_ROOT, "3rdparty", "Eigen"), "/usr/include/eigen3"):
        if c and os.path.exists(os.path.join(c, "Eigen", "Core")):
            eig = c
            break
    if eig is None:
        return None
    libdir = os.path.join(ROOT, "super4pcs_b200", "lib")
    exe = os.path.join(str(outdir), "outliers_main")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-w", "-I", os.path.join(ROOT, "include"), "-I", eig,
                           os.path.join(ROOT, "tests", "cpp", "outliers_main.cc"), "-o", exe, "-L", libdir,
                           "-lsuper4pcs_b200", "-ls4g", "-Wl,-rpath," + libdir], env=tknn._env())
    return exe


def build_shim(outdir):
    """compiles tests/stubs/s4g_outliers_shim.cc (+ oracle/outliers_port.cc and oracle/knn_port.cc) into `outdir`;
    preload it ahead of the oracle stand-in of libs4g"""
    out = os.path.join(str(outdir), "libs4g_outliers_shim.so")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                           "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "stubs", "s4g_outliers_shim.cc"),
                           os.path.join(ROOT, "oracle", "outliers_port.cc"), os.path.join(ROOT, "oracle", "knn_port.cc"),
                           "-o", out, "-ldl"], env=tknn._env())
    return out


def run(exe, workdir, xyz, normals, rgb, mode, a, b, preload=None):
    """mode 'statistical' (a = k, b = std_ratio) or 'radius' (a = radius, b = min_neighbors) -> None when the call threw,
    else (returned count, points [m, 9] float32: position, normal, rgb of each point left, as Point3D holds them)"""
    xyz = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    blob = np.concatenate([xyz, np.asarray(normals, _f).reshape(-1, 3), np.asarray(rgb, _f).reshape(-1, 3)])
    src, dst = os.path.join(str(workdir), "in.bin"), os.path.join(str(workdir), "out.bin")
    with open(src, "wb") as f:
        f.write(np.int32(len(xyz)).tobytes() + np.ascontiguousarray(blob, _f).tobytes())
    env = dict(os.environ)
    if preload:
        env["LD_PRELOAD"] = preload
    r = subprocess.run([exe, src, dst, mode, repr(a), repr(b)], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    buf = open(dst, "rb").read()
    if np.frombuffer(buf, np.int32, 1)[0]:
        return None
    count, m = np.frombuffer(buf, np.int32, 2, 4)
    return int(count), np.frombuffer(buf, _f, 9 * int(m), 12).reshape(-1, 9).copy()


def held(xyz, normals, rgb):
    """[n, 9] float32: what the program's Point3D hold before any filter (the normal through set_normal)"""
    return np.concatenate([np.asarray(xyz, _f).reshape(-1, 3), tnormals.set_normal(normals), np.asarray(rgb, _f)], 1)


def grid_delta(xyz, k):
    """the delta of RemoveStatisticalOutliers' grid: EstimateNormals' rule"""
    return tnormals.grid_delta(xyz, k)


def radius_delta(xyz, radius, min_neighbors):
    """the delta of RemoveRadiusOutliers' grid: radius / 2.02 (float32), or EstimateNormals' rule with k = min_neighbors
    when that is not a positive finite number"""
    d = np.float32(radius) / np.float32(2.02)
    return float(d) if np.isfinite(d) and d > 0 else tnormals.grid_delta(xyz, min_neighbors)


def labelled_pair(n=20000, overlap=0.6, noise_sigma=0.005, outlier_frac=0.2, seed=43):
    """cfg3's recipe (synth.make_pair: Gaussian noise on Q, a share `outlier_frac` of each cloud uniform over its
    bounding box, shuffled) with the labels kept, which make_pair's shuffle loses: dict(P, Q, out_P, out_Q), out_* [n]
    bool = the point is one of the uniform outliers"""
    from super4pcs_b200 import synth
    rng = np.random.RandomState(seed)
    n_out = int(round(outlier_frac * n))
    d = synth.make_pair(n - n_out, overlap, seed=seed, noise_sigma=noise_sigma)
    out = {}
    for key in ("P", "Q"):
        X = d[key].astype(np.float64)
        lo, hi = X.min(0), X.max(0)
        X = np.concatenate([X, lo + rng.random_sample((n_out, 3)) * (hi - lo)])
        label = np.arange(n) >= n - n_out
        perm = rng.permutation(n)
        out[key], out["out_" + key] = X[perm].astype(_f), label[perm]
    return out
