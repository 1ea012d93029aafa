"""Builds and runs tests/cpp/clusters_main.cc, the test program of Utils::ExtractEuclideanClusters, for
tests/test_clusters_cpu.py (on the oracle stand-in) and tests/test_clusters_gpu.py (on the real library), and the
stand-in's companion that answers s4g_euclidean_clusters on the CPU (tests/stubs/s4g_clusters_shim.cc).  Also the grid
delta rule of the function, and clouds whose clusters are known."""
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
    exe = os.path.join(str(outdir), "clusters_main")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-w", "-I", os.path.join(ROOT, "include"), "-I", eig,
                           os.path.join(ROOT, "tests", "cpp", "clusters_main.cc"), "-o", exe, "-L", libdir,
                           "-lsuper4pcs_b200", "-ls4g", "-Wl,-rpath," + libdir], env=tknn._env())
    return exe


def build_shim(outdir):
    """compiles tests/stubs/s4g_clusters_shim.cc (+ oracle/clusters_port.cc) into `outdir`; preload it ahead of the
    oracle stand-in of libs4g"""
    out = os.path.join(str(outdir), "libs4g_clusters_shim.so")
    subprocess.check_call(["g++", "-std=c++14", "-O2", "-ffp-contract=off", "-fopenmp", "-fPIC", "-shared",
                           "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "tests", "stubs", "s4g_clusters_shim.cc"),
                           os.path.join(ROOT, "oracle", "clusters_port.cc"), "-o", out, "-ldl"], env=tknn._env())
    return out


def run(exe, workdir, xyz, tolerance, min_size=1, max_size=2 ** 31 - 1, preload=None):
    """-> None when the call threw, else the clusters: a list of int32 index arrays, in the function's order"""
    xyz = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    src, dst = os.path.join(str(workdir), "in.bin"), os.path.join(str(workdir), "out.bin")
    with open(src, "wb") as f:
        f.write(np.int32(len(xyz)).tobytes() + xyz.tobytes())
    env = dict(os.environ)
    if preload:
        env["LD_PRELOAD"] = preload
    r = subprocess.run([exe, src, dst, repr(float(tolerance)), str(int(min_size)), str(int(max_size))], env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, (r.returncode, r.stdout[-2000:], r.stderr[-2000:])
    buf = np.frombuffer(open(dst, "rb").read(), np.int32)
    if buf[0]:
        return None
    out, at = [], 2
    for _ in range(int(buf[1])):
        s = int(buf[at])
        out.append(buf[at + 1:at + 1 + s].copy())
        at += 1 + s
    return out


def as_lists(offsets, members):
    """CSR (offsets, members) -> the list of index arrays of ExtractEuclideanClusters' form"""
    return [members[offsets[c]:offsets[c + 1]] for c in range(len(offsets) - 1)]


def tolerance_delta(xyz, tolerance):
    """the delta of ExtractEuclideanClusters' grid: tolerance / 2.02 (float32), or EstimateNormals' rule with k = 16
    when that is not a positive finite number"""
    d = np.float32(tolerance) / np.float32(2.02)
    return float(d) if np.isfinite(d) and d > 0 else tnormals.grid_delta(xyz, 16)


def blobs(sizes, spread=0.01, gap=0.2, seed=0):
    """well separated blobs of the given sizes, shuffled: (P [n, 3] float32, blob [n] int, the blob of each point).  Blob
    b is uniform in a cube of half-edge `spread` around a centre on a lattice of spacing `gap`, so any two of its points
    are closer than 2 sqrt(3) spread and points of two blobs are at least gap - 2 spread apart: at a radius between the
    two (0.05 with the defaults) each blob is exactly one component"""
    rng = np.random.RandomState(seed)
    m = int(np.ceil(len(sizes) ** (1 / 3.0) - 1e-9))
    centres = np.stack(np.meshgrid(*[np.arange(m)] * 3, indexing="ij"), -1).reshape(-1, 3)[:len(sizes)] * gap
    P = np.concatenate([c + rng.uniform(-spread, spread, (s, 3)) for c, s in zip(centres, sizes)])
    lab = np.repeat(np.arange(len(sizes)), sizes)
    perm = rng.permutation(len(P))
    return (P[perm] - P.mean(0)).astype(_f), lab[perm]
