"""Builds and runs tests/cpp/nearest_any_main.cc, the test program of Match4PCSBase::MeanDistance and
getCorrespondences(nearest, sq_dist, max_distance), for tests/test_nearest_any_cpu.py (on the oracle stand-in) and
tests/test_nearest_any_gpu.py (on the real library)."""
import numpy as np

from tests import correspondences, cpp_main


def build(outdir):
    return cpp_main.build("nearest_any_main", outdir)


def run(exe, workdir, P, Q, delta, overlap, sample_size, preload=None):
    """ComputeTransformation + MeanDistance + getCorrespondences at max_distance = delta, 3 delta, +inf -> dict(
    threw_before, score, T, C (centred), diameter, mean_distance, sP, sQ, max_distance [K], nearest [K, nSQ], sq [K, nSQ],
    nearest_delta, sq_delta (the two-argument form))"""
    r = correspondences.run_pair(exe, workdir, P, Q, delta, overlap, sample_size, preload)
    take = r.take
    out = dict(threw_before=int(take(np.int32, 1)[0]), score=take(np.float32, 1)[0], T=take(np.float32, 16),
               C=take(np.float32, 16), diameter=take(np.float32, 1)[0], mean_distance=take(np.float32, 1)[0])
    out["sP"] = take(np.float32, 3 * int(take(np.int32, 1)[0])).reshape(-1, 3)
    out["sQ"] = take(np.float32, 3 * int(take(np.int32, 1)[0])).reshape(-1, 3)
    nq = len(out["sQ"])
    K = int(take(np.int32, 1)[0])
    out["max_distance"] = take(np.float32, K)
    rows = [(take(np.int32, nq), take(np.float32, nq)) for _ in range(K)]
    out["nearest"], out["sq"] = np.array([a for a, _ in rows]), np.array([s for _, s in rows])
    out["nearest_delta"], out["sq_delta"] = take(np.int32, nq), take(np.float32, nq)
    assert r.done()
    return out
