"""Builds and runs tests/cpp/range_main.cc, the test program of Match4PCSBase::getNeighbors, for tests/test_range_cpu.py
(on the oracle stand-in) and tests/test_range_gpu.py (on the real library)."""
import numpy as np

from tests import correspondences, cpp_main


def build(outdir):
    return cpp_main.build("range_main", outdir)


def run(exe, workdir, P, Q, delta, overlap, sample_size, preload=None):
    """ComputeTransformation + getNeighbors at max_distance = delta, 3 delta -> dict(threw_before, score, C (centred),
    sP, sQ, max_distance [K], lists [K] of (offsets, indices, sq))"""
    r = correspondences.run_pair(exe, workdir, P, Q, delta, overlap, sample_size, preload)
    take = r.take
    out = dict(threw_before=int(take(np.int32, 1)[0]), score=take(np.float32, 1)[0], C=take(np.float32, 16))
    out["sP"] = take(np.float32, 3 * int(take(np.int32, 1)[0])).reshape(-1, 3)
    out["sQ"] = take(np.float32, 3 * int(take(np.int32, 1)[0])).reshape(-1, 3)
    nq = len(out["sQ"])
    K = int(take(np.int32, 1)[0])
    out["max_distance"] = take(np.float32, K)
    out["lists"] = []
    for _ in range(K):
        off = take(np.int64, nq + 1)
        out["lists"].append((off, take(np.int32, int(off[-1])), take(np.float32, int(off[-1]))))
    assert r.done()
    return out
