"""Timing of s4g_knn on cfg2 (1M x 1M pair, delta = 0.003) for k in {1, 8, 16, 32, 64}, one JSON line per (query set, k),
with the card's name and power limit:

  self      1M sampled-P points, each excluding itself, unbounded: the normal-estimation query
  near_gt   1M unbounded queries T q, T near the ground truth
  wrong     1M unbounded queries T q, T a random (wrong) transform

GPU: CUDA events around `reps` calls of s4g_knn_dev after one warm-up call; the mean number of P points tested and of
coarse blocks scanned per query from s4g_knn_probe_stats.  CPU (a time baseline only, when scipy imports):
scipy.spatial.cKDTree(P).query(X, k) on the first CPU_QUERIES queries, with 1 thread and with all threads, wall clock,
and the share of those rows whose index set equals ours.  cKDTree works in float64, so a row can differ where distances
tie or nearly tie in fp32; it is not an oracle.

usage: python scripts/knn_bench.py [reps]
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

KS = [1, 8, 16, 32, 64]
CPU_QUERIES = 20000


def cpu_rows(tree, X, k, exclude, workers):
    """cKDTree's k nearest of X (the query's own index removed when exclude is given) -> (index [m, k], seconds)"""
    t0 = time.perf_counter()
    kk = k + 1 if exclude is not None else k
    _, idx = tree.query(X, kk, workers=workers)
    secs = time.perf_counter() - t0
    idx = idx.reshape(len(X), kk)
    if exclude is not None:
        keep = idx != exclude[:, None]
        keep[keep.all(1), -1] = False                          # the point itself was not among them: drop the last
        idx = idx[keep].reshape(len(X), k)
    return idx, secs


def main(reps=5):
    import torch
    n, delta = 1_000_000, 0.003
    d = synth.make_pair(n, 0.3, seed=42)
    P, cp = synth.center(d["P"])
    Q, cq = synth.center(d["Q"])
    M = synth.candidate_transforms(2, delta, seed=7, n_near=1, centroid_p=cp, centroid_q=cq)   # near-GT, then a random one
    T = np.ascontiguousarray(M.transpose(0, 2, 1)).reshape(-1, 16).astype(np.float32)
    P, Q = np.ascontiguousarray(P, np.float32), np.ascontiguousarray(Q, np.float32)
    self_ = np.arange(n, dtype=np.int32)
    cases = [("self", P, None, self_), ("near_gt", Q, T[0], None), ("wrong", Q, T[1], None)]
    try:
        from scipy.spatial import cKDTree
        tree = cKDTree(P.astype(np.float64))
    except ImportError:
        tree = None
    stream = torch.cuda.Stream()
    with Context(0) as ctx, torch.cuda.stream(stream):
        ctx.set_cloud_p(P, delta)
        ctx.set_stream(stream.cuda_stream)
        idx = torch.empty(n * max(KS), dtype=torch.int32, device="cuda")
        sq = torch.empty(n * max(KS), dtype=torch.float32, device="cuda")
        for name, X, T16, ex in cases:
            dX = torch.from_numpy(np.ascontiguousarray(X)).cuda()
            dT = None if T16 is None else torch.from_numpy(T16.copy()).cuda()
            dE = None if ex is None else torch.from_numpy(ex).cuda()
            Y = X if T16 is None else (X.astype(np.float64) @ T16.reshape(4, 4)[:3, :3].astype(np.float64)
                                       + T16.reshape(4, 4)[3, :3].astype(np.float64))
            for k in KS:
                call = lambda: ctx.knn_dev(dX.data_ptr(), n, k, idx.data_ptr(), sq.data_ptr(), np.inf,  # noqa: E731
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
                index, _, st = ctx.knn(X, k, np.inf, T16, ex, stats=True)
                assert np.array_equal(index.reshape(-1), idx[:n * k].cpu().numpy())
                row = dict(cfg="cfg2", stage="knn", queries=name, k=k, n_p=n, n_q=n, delta=delta, sq_radius="inf",
                           ms=ms, queries_per_s=n / (ms * 1e-3), points_tested_per_query=st["tested"] / n,
                           blocks_per_query=st["blocks"] / n, device=bench.device_info(0, 0))
                if tree is not None:
                    m = CPU_QUERIES
                    sub_ex = None if ex is None else ex[:m]
                    ci, s1 = cpu_rows(tree, Y[:m], k, sub_ex, 1)
                    _, sa = cpu_rows(tree, Y[:m], k, sub_ex, -1)
                    agree = (np.sort(ci, 1) == np.sort(index[:m], 1)).all(1).mean()
                    row.update(cpu_queries=m, cpu_ckdtree_1thread_ms=s1 * 1e3, cpu_ckdtree_all_threads_ms=sa * 1e3,
                               cpu_threads=os.cpu_count(),
                               cpu_rows_same_index_set=float(agree))
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 5)
