"""Builds and runs tests/cpp/clusters_main.cc, the test program of Utils::ExtractEuclideanClusters, for
tests/test_clusters_cpu.py (on the oracle stand-in) and tests/test_clusters_gpu.py (on the real library).  Also the grid
delta rule of the function, and clouds whose clusters are known."""
import numpy as np

from tests import cpp_main, normals as tnormals

_f = np.float32


def build(outdir):
    return cpp_main.build("clusters_main", outdir)


def run(exe, workdir, xyz, tolerance, min_size=1, max_size=2 ** 31 - 1, preload=None):
    """-> None when the call threw, else the clusters: a list of int32 index arrays, in the function's order"""
    xyz = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    buf = np.frombuffer(cpp_main.run(exe, workdir, np.int32(len(xyz)).tobytes() + xyz.tobytes(),
                                     [repr(float(tolerance)), str(int(min_size)), str(int(max_size))], preload), np.int32)
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
