"""Builds and runs tests/cpp/correspondences_main.cc, the test program of Match4PCSBase::getCorrespondences, for
tests/test_verify_nearest_cpu.py (on the oracle stand-in) and tests/test_verify_nearest_gpu.py (on the real library).
Also the input of every test program that registers a pair of clouds first (this one, nearest_any, range, knn)."""
import numpy as np

from tests import cpp_main


def build(outdir):
    return cpp_main.build("correspondences_main", outdir)


def run_pair(exe, workdir, P, Q, delta, overlap, sample_size, preload):
    """runs a program that calls ComputeTransformation(P, Q) at (delta, overlap, sample_size) first -> a Reader of its
    output"""
    P, Q = np.ascontiguousarray(P, np.float32), np.ascontiguousarray(Q, np.float32)
    payload = np.array([len(P), len(Q)], np.int32).tobytes() + P.tobytes() + Q.tobytes()
    args = [repr(float(delta)), repr(float(overlap)), str(int(sample_size))]
    return cpp_main.Reader(cpp_main.run(exe, workdir, payload, args, preload))


def run(exe, workdir, P, Q, delta, overlap, sample_size, preload=None):
    """ComputeTransformation + getCorrespondences -> dict(threw_before, score, T, C (centred), sP, sQ, nearest, sq,
    nearest2 (the call without sq_dist))"""
    r = run_pair(exe, workdir, P, Q, delta, overlap, sample_size, preload)
    take = r.take
    out = dict(threw_before=int(take(np.int32, 1)[0]), score=take(np.float32, 1)[0], T=take(np.float32, 16),
               C=take(np.float32, 16))
    out["sP"] = take(np.float32, 3 * int(take(np.int32, 1)[0])).reshape(-1, 3)
    out["sQ"] = take(np.float32, 3 * int(take(np.int32, 1)[0])).reshape(-1, 3)
    nq = len(out["sQ"])
    out["nearest"], out["sq"], out["nearest2"] = take(np.int32, nq), take(np.float32, nq), take(np.int32, nq)
    assert r.done()
    return out
