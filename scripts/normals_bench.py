"""Timing of s4g_normals on the cfg2 P (1M points, delta = 0.003), unbounded, k in {8, 16, 32}; one JSON line per k and
one for the grid's delta, with the card's name and power limit.

GPU, CUDA events around `reps` calls after one warm-up call:
  knn_original_ms   s4g_knn_dev of the P points in the order of the cloud (no exclusion): the rows alone
  normals_ms        the whole s4g_normals_dev (sorted queries, k_knn in the grid's order, k_normals)
and, from one torch.profiler pass over `reps` further s4g_normals_dev calls (CUPTI kernel durations, mean per call):
  kernel_ms         {k_normals_queries, k_knn (the rows in the grid's order), k_normals}
CPU baseline (when scipy imports), wall clock: scipy.spatial.cKDTree(P).query(P, k, workers=-1) and numpy float64 batched
np.linalg.eigh of each row's covariance (in chunks of 100 000 rows), and the share of points whose normals agree with ours
within 1 degree, up to sign.  cKDTree works in float64, so a row can differ where distances tie in fp32.
Grid delta (k = 16): s4g_set_cloud_p + s4g_normals_dev, wall clock to a synchronize, at the delta of
Utils::EstimateNormals's rule (0.5 E sqrt(k / n)) and at 0.5x and 2x of it, after one warm-up at each.

usage: python scripts/normals_bench.py [reps]
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

KS = [8, 16, 32]
KERNELS = ("k_normals_queries", "k_knn", "k_normals")


def cpu_normals(P, k):
    """cKDTree + float64 batched eigh -> (normals [n, 3], seconds of the tree's build and query, seconds of the PCA)"""
    from scipy.spatial import cKDTree
    t0 = time.perf_counter()
    _, idx = cKDTree(P.astype(np.float64)).query(P.astype(np.float64), k, workers=-1)
    t1 = time.perf_counter()
    P64 = P.astype(np.float64)
    out = np.empty((len(P), 3))
    for s in range(0, len(P), 100000):
        pts = P64[idx[s:s + 100000]]
        d = pts - pts.mean(1, keepdims=True)
        out[s:s + 100000] = np.linalg.eigh(np.einsum("nki,nkj->nij", d, d) / k)[1][:, :, 0]
    return out, t1 - t0, time.perf_counter() - t1


def kernel_ms(prof, reps):
    """mean device time per call of each kernel of s4g_normals_dev in a profiler trace (demangled names: k_knn<...>,
    k_normals(...), k_normals_queries(...))"""
    out = {name: 0.0 for name in KERNELS}
    for e in prof.key_averages():
        for name in KERNELS:
            if name + "<" in e.key or name + "(" in e.key:
                out[name] += e.device_time_total / 1e3 / reps
                break
    return out


def main(reps=5):
    import torch
    n, delta = 1_000_000, 0.003
    P, _ = synth.center(synth.make_pair(n, 0.3, seed=42)["P"])
    P = np.ascontiguousarray(P, np.float32)
    dev = bench.device_info(0, 0)
    stream = torch.cuda.Stream()
    dX = torch.from_numpy(P).cuda()
    idx = torch.empty(n * max(KS), dtype=torch.int32, device="cuda")
    dn = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    de = torch.empty((n, 3), dtype=torch.float32, device="cuda")

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

    with Context(0) as ctx, torch.cuda.stream(stream):
        ctx.set_stream(stream.cuda_stream)
        ctx.set_cloud_p(P, delta)
        for k in KS:
            knn_ms = timed(lambda: ctx.knn_dev(dX.data_ptr(), n, k, idx.data_ptr(), None))
            normals_ms = timed(lambda: ctx.normals_dev(k, dn.data_ptr(), de.data_ptr()))
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    ctx.normals_dev(k, dn.data_ptr(), de.data_ptr())
                stream.synchronize()
            row = dict(cfg="cfg2", stage="normals", k=k, n_p=n, delta=delta, sq_radius="inf", reps=reps,
                       knn_original_ms=knn_ms, normals_ms=normals_ms, kernel_ms=kernel_ms(prof, reps), device=dev)
            try:
                ours = dn.cpu().numpy().astype(np.float64)
                cpu, tree_s, pca_s = cpu_normals(P, k)
                live = np.abs(ours).sum(1) > 0
                agree = (np.abs((ours * cpu).sum(1)) >= np.cos(np.radians(1.0))) & live
                row.update(cpu_threads=os.cpu_count(), cpu_ckdtree_query_workers=-1, cpu_ckdtree_ms=tree_s * 1e3,
                           cpu_numpy_eigh_ms=pca_s * 1e3, cpu_total_ms=(tree_s + pca_s) * 1e3,
                           share_within_1deg=float(agree.mean()))
            except ImportError:
                pass
            print(json.dumps(row), flush=True)
        # the grid's delta of Utils::EstimateNormals (tests/normals.py grid_delta) and its neighbours
        k = 16
        E = float((P.max(0).astype(np.float64) - P.min(0).astype(np.float64)).max())
        rule = float(np.float32(0.5 * E * np.sqrt(k / n)))
        out = {}
        for f in (0.5, 1.0, 2.0):
            d = rule * f

            def once():
                t0 = time.perf_counter()
                ctx.set_cloud_p(P, d)
                ctx.normals_dev(k, dn.data_ptr(), None)
                stream.synchronize()
                return (time.perf_counter() - t0) * 1e3
            once()
            out["x%g" % f] = dict(delta=d, ms=float(np.median([once() for _ in range(reps)])))
        print(json.dumps(dict(cfg="cfg2", stage="normals_grid_delta", k=k, n_p=n, rule="0.5 E sqrt(k / n)", reps=reps,
                              runs=out, device=dev)), flush=True)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 5)
