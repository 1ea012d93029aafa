"""Timing of s4g_nearest on cfg2 (1M x 1M pair, delta = 0.003), one JSON line per figure, with the card's name and power
limit:

  self      1M sampled-P points, each excluding itself, at MeanDistance's squared radius 0.2 x diameter (here the largest
            extent of P)
  near_gt   1M unbounded queries T q, T near the ground truth
  wrong     1M unbounded queries T q, T a random (wrong) transform

GPU: CUDA events around `reps` calls of s4g_nearest_dev after one warm-up call; the mean number of P points tested and of
coarse blocks scanned per query from s4g_nearest_probe_stats.  CPU (the figure to beat, when the compiled reference is
present): the reference's kd-tree (KdTree::doQueryRestrictedClosestIndex) for the same queries, one thread, wall clock.

usage: python scripts/nearest_bench.py [reps]
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from super4pcs_b200 import Context, synth  # noqa: E402


def main(reps=10):
    import torch
    from oracle import nearest_any as ona
    n, delta = 1_000_000, 0.003
    d = synth.make_pair(n, 0.3, seed=42)
    P, cp = synth.center(d["P"])
    Q, cq = synth.center(d["Q"])
    M = synth.candidate_transforms(2, delta, seed=7, n_near=1, centroid_p=cp, centroid_q=cq)   # near-GT, then a random one
    T = np.ascontiguousarray(M.transpose(0, 2, 1)).reshape(-1, 16).astype(np.float32)
    ref = None
    if ona.ref_available():                 # the reference's matcher on the pair; its centred clouds are the ones timed
        ref = ona.RefNearestAny(P, Q, delta)
        P, Q = ref.sampled()
    radius = float(np.float32(np.abs(P.max(0) - P.min(0)).max()) * np.float32(0.2))
    self_ = np.arange(n, dtype=np.int32)
    cases = [("self", P, None, radius, self_), ("near_gt", Q, T[0], np.inf, None), ("wrong", Q, T[1], np.inf, None)]
    stream = torch.cuda.Stream()
    with Context(0) as ctx, torch.cuda.stream(stream):
        ctx.set_cloud_p(P, delta)
        ctx.set_stream(stream.cuda_stream)
        idx = torch.empty(n, dtype=torch.int32, device="cuda")
        sq = torch.empty(n, dtype=torch.float32, device="cuda")
        for name, X, T16, r, ex in cases:
            dX = torch.from_numpy(np.ascontiguousarray(X)).cuda()
            dT = None if T16 is None else torch.from_numpy(T16.copy()).cuda()
            dE = None if ex is None else torch.from_numpy(ex).cuda()
            call = lambda: ctx.nearest_dev(dX.data_ptr(), n, idx.data_ptr(), sq.data_ptr(), r,  # noqa: E731
                                           None if dT is None else dT.data_ptr(), None if dE is None else dE.data_ptr())
            call()
            stream.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(reps):
                call()
            e1.record(stream)
            e1.synchronize()
            ms = e0.elapsed_time(e1) / reps
            index, _, st = ctx.nearest(X, r, T16, ex, stats=True)
            assert np.array_equal(index, idx.cpu().numpy())
            row = dict(cfg="cfg2", stage="nearest", queries=name, n_p=n, n_q=n, delta=delta, sq_radius=r, ms=ms,
                       queries_per_s=n / (ms * 1e-3), found=int((index >= 0).sum()), points_tested_per_query=st["tested"] / n,
                       blocks_per_query=st["blocks"] / n, device=bench.device_info(0, 0))
            if ref is not None:
                t0 = time.perf_counter()
                ri, _ = ref.query(X, r, T16, ex)
                row["cpu_reference_kdtree_ms"] = (time.perf_counter() - t0) * 1e3
                row["cpu_reference_found"] = int((ri >= 0).sum())
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 10)
