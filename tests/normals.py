"""Builds and runs tests/cpp/normals_main.cc, the test program of Utils::EstimateNormals, for tests/test_normals_cpu.py
(on the oracle stand-in) and tests/test_normals_gpu.py (on the real library), and the stand-in's companion that answers
s4g_normals on the CPU (tests/stubs/s4g_normals_shim.cc).  Also the float32 arithmetic of Point3D::set_normal, which
EstimateNormals stores its normals through, and the rule of its grid's delta."""
import os
import subprocess

import numpy as np

from tests import knn as tknn

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
    exe = os.path.join(str(outdir), "normals_main")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-w", "-I", os.path.join(ROOT, "include"), "-I", eig,
                           os.path.join(ROOT, "tests", "cpp", "normals_main.cc"), "-o", exe, "-L", libdir,
                           "-lsuper4pcs_b200", "-ls4g", "-Wl,-rpath," + libdir], env=tknn._env())
    return exe


def build_shim(outdir):
    """compiles tests/stubs/s4g_normals_shim.cc (+ oracle/normals_port.cc and oracle/knn_port.cc) into `outdir`; preload
    it ahead of the oracle stand-in of libs4g"""
    out = os.path.join(str(outdir), "libs4g_normals_shim.so")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                           "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "stubs", "s4g_normals_shim.cc"),
                           os.path.join(ROOT, "oracle", "normals_port.cc"), os.path.join(ROOT, "oracle", "knn_port.cc"),
                           "-o", out, "-ldl"], env=tknn._env())
    return out


def run(exe, workdir, xyz, k, max_distance=np.inf, viewpoint=None, preload=None):
    """-> None when EstimateNormals threw, else (returned count, normals [n, 3] float32 as the points hold them)"""
    xyz = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    src, dst = os.path.join(str(workdir), "in.bin"), os.path.join(str(workdir), "out.bin")
    with open(src, "wb") as f:
        f.write(np.int32(len(xyz)).tobytes() + xyz.tobytes())
    env = dict(os.environ)
    if preload:
        env["LD_PRELOAD"] = preload
    args = [exe, src, dst, str(int(k)), repr(float(max_distance))]
    if viewpoint is not None:
        args += [repr(float(v)) for v in np.asarray(viewpoint, _f)]
    r = subprocess.run(args, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    b = open(dst, "rb").read()
    if np.frombuffer(b, np.int32, 1)[0]:
        return None
    return int(np.frombuffer(b, np.int32, 1, 4)[0]), np.frombuffer(b, _f, 3 * len(xyz), 8).reshape(-1, 3).copy()


def set_normal(n):
    """Point3D::set_normal (Eigen's normalized()) in float32: n / sqrt(x^2 + (y^2 + z^2)) when that is > 0, else n"""
    n = np.asarray(n, _f)
    sq = n[:, 0] * n[:, 0] + (n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2])
    out = n.copy()
    pos = sq > 0
    out[pos] = n[pos] / np.sqrt(sq[pos])[:, None]
    return out


def grid_delta(xyz, k):
    """the delta EstimateNormals builds its grid with: 0.5 E sqrt(k / n), E the largest edge of the bounding box; 1 when
    E is 0"""
    xyz = np.asarray(xyz, _f)
    E = float((xyz.max(0).astype(np.float64) - xyz.min(0).astype(np.float64)).max())
    d = np.float32(0.5 * E * np.sqrt(k / len(xyz)))
    return float(d) if d > 0 else 1.0
