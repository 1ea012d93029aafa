"""Timing of the range query (s4g_range_count_dev + s4g_range_fill_dev) on cfg2 (1M x 1M pair, delta = 0.003), one JSON
line per figure, with the card's name and power limit:

  self     1M sampled-P points at MeanDistance's squared radius 0.2 x diameter (here the largest extent of P).  Every list
           holds ~20 % of P, so the 1M lists (~2e11 entries) cannot be held: the count pass is timed over all 1M
           queries, count + fill over the longest leading run of (randomly ordered) queries whose lists fit in 1e9
           entries.
  near_gt  1M queries T q at delta^2, T near the ground truth
  wrong    1M queries T q at delta^2, T a random (wrong) transform

GPU: CUDA events around `reps` calls after one warm-up call; the total entries and the entries per query (mean, max) of
the same queries.  CPU (when the compiled reference is present): the reference's kd-tree (KdTree::doQueryDistIndices)
on one thread, wall clock, over all the queries at delta^2 and over the first 250 at MeanDistance's radius.

usage: python scripts/range_bench.py [reps]
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

FILL_LIMIT = 1_000_000_000   # entries (8 GB of indices and d^2)
CPU_SUBSAMPLE = 250          # queries of the reference's tree at MeanDistance's radius


def main(reps=10):
    import torch
    from oracle import range as orange
    n, delta = 1_000_000, 0.003
    d = synth.make_pair(n, 0.3, seed=42)
    P, cp = synth.center(d["P"])
    Q, cq = synth.center(d["Q"])
    M = synth.candidate_transforms(2, delta, seed=7, n_near=1, centroid_p=cp, centroid_q=cq)   # near-GT, then a random one
    T = np.ascontiguousarray(M.transpose(0, 2, 1)).reshape(-1, 16).astype(np.float32)
    ref = None
    if orange.ref_available():              # the reference's matcher on the pair; its centred clouds are the ones timed
        ref = orange.RefRange(P, Q, delta)
        P, Q = ref.sampled()
    sq_delta = float(np.float32(delta) * np.float32(delta))
    md = float(np.float32(np.abs(P.max(0) - P.min(0)).max()) * np.float32(0.2))
    perm = np.random.RandomState(0).permutation(n)
    cases = [("self", P[perm], None, md), ("near_gt", Q, T[0], sq_delta), ("wrong", Q, T[1], sq_delta)]
    stream = torch.cuda.Stream()
    with Context(0) as ctx, torch.cuda.stream(stream):
        ctx.set_cloud_p(P, delta)
        ctx.set_stream(stream.cuda_stream)

        def timed(call):
            call()
            stream.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(reps):
                call()
            e1.record(stream)
            e1.synchronize()
            return e0.elapsed_time(e1) / reps

        for name, X, T16, r in cases:
            dX = torch.from_numpy(np.ascontiguousarray(X)).cuda()
            dT = None if T16 is None else torch.from_numpy(T16.copy()).cuda()
            pT = None if dT is None else dT.data_ptr()
            off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
            count = lambda m: ctx.range_count_dev(dX.data_ptr(), m, off.data_ptr(), r, pT)  # noqa: E731
            count_ms = timed(lambda: count(n))
            stream.synchronize()
            o = off.cpu().numpy()
            lens = np.diff(o)
            m = n if o[n] <= FILL_LIMIT else int(np.searchsorted(o, FILL_LIMIT, side="right")) - 1
            total = int(o[m])
            idx = torch.empty(max(total, 1), dtype=torch.int32, device="cuda")
            sq = torch.empty(max(total, 1), dtype=torch.float32, device="cuda")

            def both():
                count(m)
                ctx.range_fill_dev(dX.data_ptr(), m, off.data_ptr(), total, idx.data_ptr(), sq.data_ptr(), r, pT)
            ms = timed(both)
            row = dict(cfg="cfg2", stage="range", queries=name, n_p=n, n_q=n, delta=delta, sq_radius=r,
                       count_ms_all=count_ms, total_all=int(o[n]), entries_per_query_mean=float(lens.mean()),
                       entries_per_query_max=int(lens.max()), queries_filled=m, total_filled=total, ms=ms,
                       device=bench.device_info(0, 0))
            if ref is not None:
                k = n if r == sq_delta else CPU_SUBSAMPLE
                t0 = time.perf_counter()
                ro, _, _ = ref.query(X[:k], r, T16)
                row["cpu_reference_kdtree_queries"] = k
                row["cpu_reference_kdtree_ms"] = (time.perf_counter() - t0) * 1e3
                row["cpu_reference_total"] = int(ro[-1])
                assert int(ro[-1]) == int(o[k])
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 10)
