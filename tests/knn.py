"""Builds and runs tests/cpp/knn_main.cc, the test program of Match4PCSBase::getKNearest, for tests/test_knn_cpu.py (on
the oracle stand-in) and tests/test_knn_gpu.py (on the real library), and the stand-in's companion that answers s4g_knn
on the CPU (tests/stubs/s4g_knn_shim.cc)."""
import os
import subprocess

import numpy as np

from tests import nearest_any

ROOT = nearest_any.ROOT


def _env():
    env = dict(os.environ)
    env.pop("CXX", None)
    env.pop("CC", None)
    return env


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
    exe = os.path.join(str(outdir), "knn_main")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-w", "-I", os.path.join(ROOT, "include"), "-I", eig,
                           os.path.join(ROOT, "tests", "cpp", "knn_main.cc"), "-o", exe, "-L", libdir,
                           "-lsuper4pcs_b200", "-ls4g", "-Wl,-rpath," + libdir], env=_env())
    return exe


def build_shim(outdir):
    """compiles tests/stubs/s4g_knn_shim.cc (+ the brute force of oracle/knn_port.cc) into `outdir`; preload it ahead of
    the oracle stand-in of libs4g"""
    out = os.path.join(str(outdir), "libs4g_knn_shim.so")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                           "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "stubs", "s4g_knn_shim.cc"),
                           os.path.join(ROOT, "oracle", "knn_port.cc"), "-o", out, "-ldl"], env=_env())
    return out


def run(exe, workdir, P, Q, delta, overlap, sample_size, preload=None):
    """ComputeTransformation + getKNearest for (k, max_distance) = (1, delta), (8, 3 delta), (16, +inf), (64, +inf) ->
    dict(threw_before, score, C (centred), sP, sQ, runs [K] of (k, max_distance), rows [K] of (index, sq) [nSQ, k])"""
    P, Q = np.ascontiguousarray(P, np.float32), np.ascontiguousarray(Q, np.float32)
    src, dst = os.path.join(str(workdir), "in.bin"), os.path.join(str(workdir), "out.bin")
    with open(src, "wb") as f:
        f.write(np.array([len(P), len(Q)], np.int32).tobytes() + P.tobytes() + Q.tobytes())
    env = dict(os.environ)
    if preload:
        env["LD_PRELOAD"] = preload
    r = subprocess.run([exe, src, dst, repr(float(delta)), repr(float(overlap)), str(int(sample_size))], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    b = open(dst, "rb").read()
    at = 0

    def take(dt, n):
        nonlocal at
        a = np.frombuffer(b, dt, n, at).copy()
        at += a.nbytes
        return a
    out = dict(threw_before=int(take(np.int32, 1)[0]), score=take(np.float32, 1)[0], C=take(np.float32, 16))
    out["sP"] = take(np.float32, 3 * int(take(np.int32, 1)[0])).reshape(-1, 3)
    out["sQ"] = take(np.float32, 3 * int(take(np.int32, 1)[0])).reshape(-1, 3)
    nq = len(out["sQ"])
    K = int(take(np.int32, 1)[0])
    out["runs"] = [(int(take(np.int32, 1)[0]), take(np.float32, 1)[0]) for _ in range(K)]
    out["rows"] = [(take(np.int32, nq * k).reshape(nq, k), take(np.float32, nq * k).reshape(nq, k)) for k, _ in out["runs"]]
    assert at == len(b)
    return out
