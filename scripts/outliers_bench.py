"""Timing of the outlier filters (s4g_statistical_outliers, s4g_radius_outliers) on two clouds, one JSON line per case,
each with the card's name and power limit:
  cfg2   the cfg2 P (1M points, centred, delta = 0.003)
  cfg3   the cfg3 P (200 000 points, 20 % uniform outliers, centred, delta = 0.01)

GPU, CUDA events around `reps` calls of the _dev form after one warm-up call, then one torch.profiler pass over `reps`
further calls (CUPTI kernel durations, mean per call) split into stages:
  statistical, k in {8, 16, 32}, std_ratio = 1:
    rows        k_normals_queries + k_outlier_exclude + k_knn (the self-excluded k-nearest rows in the grid's order)
    mean        k_outlier_mean
    reductions  k_outlier_runs + k_outlier_moments (mu, then sigma) + k_outlier_flags
    compaction  cub's DeviceSelect (the kept j in ascending order)
  radius, sq_radius in {delta^2, (3 delta)^2} x min_neighbors in {4, 16}:
    capped      the filter as shipped: k_radius_count stops at min_neighbors
    full        the same kernel with min_neighbors = 2^31 - 1, which no count reaches: every neighbour is counted, i.e.
                the cost without the early exit (its keep list is empty; only the time is reported)
CPU baseline (when scipy imports), wall clock: scipy.spatial.cKDTree(P, float64) built and queried with workers=16, plus
numpy's mean / std (statistical: k + 1 nearest, self dropped; radius: query_ball_point(return_length=True) minus 1), and
the agreement of its mask with ours.

usage: python scripts/outliers_bench.py [reps]
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
STAGES = {"rows": ("k_normals_queries", "k_outlier_exclude", "k_knn"), "mean": ("k_outlier_mean",),
          "reductions": ("k_outlier_runs", "k_outlier_moments", "k_outlier_flags"),
          "compaction": ("DeviceSelect", "DeviceCompactInit")}
WORKERS = 16


def clouds():
    P2, _ = synth.center(synth.make_pair(1_000_000, 0.3, seed=42)["P"])
    P3, _ = synth.center(synth.make_pair(200_000, 0.4, seed=43, noise_sigma=0.005, outlier_frac=0.2)["P"])
    return [("cfg2", np.ascontiguousarray(P2, np.float32), 0.003), ("cfg3", np.ascontiguousarray(P3, np.float32), 0.01)]


def stage_ms(prof, reps):
    out = {s: 0.0 for s in STAGES}
    for e in prof.key_averages():
        for s, names in STAGES.items():
            if any(nm in e.key for nm in names):
                out[s] += e.device_time_total / 1e3 / reps
                break
    return out


def cpu_statistical(P, k, std_ratio):
    from scipy.spatial import cKDTree
    t0 = time.perf_counter()
    X = P.astype(np.float64)
    d, _ = cKDTree(X).query(X, k + 1, workers=WORKERS)
    mean = d[:, 1:].mean(1)
    mask = mean <= mean.mean() + std_ratio * mean.std(ddof=1)
    return mask, (time.perf_counter() - t0) * 1e3


def cpu_radius(P, sq_radius, min_neighbors):
    from scipy.spatial import cKDTree
    t0 = time.perf_counter()
    X = P.astype(np.float64)
    c = cKDTree(X).query_ball_point(X, float(np.sqrt(sq_radius)), workers=WORKERS, return_length=True) - 1
    return c >= min_neighbors, (time.perf_counter() - t0) * 1e3


def main(reps=5):
    import torch
    dev = bench.device_info(0, 0)
    stream = torch.cuda.Stream()

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

    for cfg, P, delta in clouds():
        n = len(P)
        keep = torch.empty(n, dtype=torch.int32, device="cuda")
        nk = torch.empty(1, dtype=torch.int64, device="cuda")
        mean = torch.empty(n, dtype=torch.float64, device="cuda")
        counts = torch.empty(n, dtype=torch.int32, device="cuda")
        with Context(0) as ctx, torch.cuda.stream(stream):
            ctx.set_stream(stream.cuda_stream)
            ctx.set_cloud_p(P, delta)
            for k in KS:
                call = lambda: ctx.statistical_outliers_dev(k, 1.0, keep.data_ptr(), nk.data_ptr(), mean.data_ptr())  # noqa: E731
                ms = timed(call)
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(reps):
                        call()
                    stream.synchronize()
                ours = np.zeros(n, bool)
                ours[keep[:int(nk.item())].cpu().numpy()] = True
                row = dict(cfg=cfg, stage="statistical_outliers", k=k, std_ratio=1.0, n_p=n, delta=delta, reps=reps,
                           total_ms=ms, stage_ms=stage_ms(prof, reps), kept=int(ours.sum()), device=dev)
                try:
                    mask, cpu_ms = cpu_statistical(P, k, 1.0)
                    row.update(cpu_workers=WORKERS, cpu_ckdtree_numpy_ms=cpu_ms, mask_agreement=float((mask == ours).mean()))
                except ImportError:
                    pass
                print(json.dumps(row), flush=True)
            for r in (delta * delta, 9 * delta * delta):
                for mn in (4, 16):
                    capped = timed(lambda: ctx.radius_outliers_dev(r, mn, keep.data_ptr(), nk.data_ptr(), counts.data_ptr()))
                    ours = np.zeros(n, bool)
                    ours[keep[:int(nk.item())].cpu().numpy()] = True
                    full = timed(lambda: ctx.radius_outliers_dev(r, 2 ** 31 - 1, keep.data_ptr(), nk.data_ptr(),
                                                                 counts.data_ptr()))
                    row = dict(cfg=cfg, stage="radius_outliers", sq_radius=r, radius_in_delta=float(np.sqrt(r) / delta),
                               min_neighbors=mn, n_p=n, delta=delta, reps=reps, capped_ms=capped, full_count_ms=full,
                               early_exit_speedup=full / capped, kept=int(ours.sum()), device=dev)
                    try:
                        mask, cpu_ms = cpu_radius(P, r, mn)
                        row.update(cpu_workers=WORKERS, cpu_ckdtree_ms=cpu_ms, mask_agreement=float((mask == ours).mean()))
                    except ImportError:
                        pass
                    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 5)
