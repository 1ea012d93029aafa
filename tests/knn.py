"""Builds and runs tests/cpp/knn_main.cc, the test program of Match4PCSBase::getKNearest, for tests/test_knn_cpu.py (on
the oracle stand-in) and tests/test_knn_gpu.py (on the real library)."""
import numpy as np

from tests import correspondences, cpp_main


def build(outdir):
    return cpp_main.build("knn_main", outdir)


def run(exe, workdir, P, Q, delta, overlap, sample_size, preload=None):
    """ComputeTransformation + getKNearest for (k, max_distance) = (1, delta), (8, 3 delta), (16, +inf), (64, +inf) ->
    dict(threw_before, score, C (centred), sP, sQ, runs [K] of (k, max_distance), rows [K] of (index, sq) [nSQ, k])"""
    r = correspondences.run_pair(exe, workdir, P, Q, delta, overlap, sample_size, preload)
    take = r.take
    out = dict(threw_before=int(take(np.int32, 1)[0]), score=take(np.float32, 1)[0], C=take(np.float32, 16))
    out["sP"] = take(np.float32, 3 * int(take(np.int32, 1)[0])).reshape(-1, 3)
    out["sQ"] = take(np.float32, 3 * int(take(np.int32, 1)[0])).reshape(-1, 3)
    nq = len(out["sQ"])
    K = int(take(np.int32, 1)[0])
    out["runs"] = [(int(take(np.int32, 1)[0]), take(np.float32, 1)[0]) for _ in range(K)]
    out["rows"] = [(take(np.int32, nq * k).reshape(nq, k), take(np.float32, nq * k).reshape(nq, k)) for k, _ in out["runs"]]
    assert r.done()
    return out
