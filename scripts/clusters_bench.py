"""Timing of the Euclidean clusters (s4g_euclidean_clusters) on two clouds, one JSON line per case, each with the card's
name and power limit:
  cfg2   the cfg2 P (1M points, centred, delta = 0.003) at radius delta, 2 delta and 3 delta, min_size = 1
  cfg3   the cfg3 P (200 000 points, 20 % uniform outliers, centred, delta = 0.01) at radius 0.01 and 0.02, min_size 1
         and 100

GPU, CUDA events around `reps` calls of the _dev form after one warm-up call, then one torch.profiler pass over `reps`
further calls (CUPTI kernel durations, mean per call) split into stages:
  link            k_cluster_link (the box descent and the union-find hooks)
  compress_sizes  k_cluster_init + k_cluster_compress + k_cluster_flags
  ordering_csr    the two radix sorts, the offsets' scan, k_cluster_sizes, k_cluster_rank, k_cluster_labels
  copies          the memsets and the device-to-device copy of the members
Yardstick: s4g_range_count_dev over the same points at the same radius (the same descent and point test, no union-find;
plus its scan), the queries in brick order so that their locality matches the link kernel's grid order.  The gap between
the two is the cost of the hooks.
CPU baseline (when scipy imports), wall clock: scipy.spatial.cKDTree(P, float64).query_pairs(r, output_type='ndarray') +
scipy.sparse.csgraph.connected_components, and the number of points whose component differs from ours (the float64
test can disagree with the fp32 one at the boundary, so this is reported, not asserted).

usage: python scripts/clusters_bench.py [reps]
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

STAGES = {"link": ("k_cluster_link",), "compress_sizes": ("k_cluster_init", "k_cluster_compress", "k_cluster_flags"),
          "ordering_csr": ("RadixSort", "DeviceScan", "k_cluster_sizes", "k_cluster_rank", "k_cluster_labels"),
          "copies": ("Memset", "Memcpy")}


def clouds():
    P2, _ = synth.center(synth.make_pair(1_000_000, 0.3, seed=42)["P"])
    P3, _ = synth.center(synth.make_pair(200_000, 0.4, seed=43, noise_sigma=0.005, outlier_frac=0.2)["P"])
    return [("cfg2", np.ascontiguousarray(P2, np.float32), 0.003, [0.003, 0.006, 0.009], [1]),
            ("cfg3", np.ascontiguousarray(P3, np.float32), 0.01, [0.01, 0.02], [1, 100])]


def stage_ms(prof, reps):
    out = {s: 0.0 for s in STAGES}
    for e in prof.key_averages():
        for s, names in STAGES.items():
            if any(nm in e.key for nm in names):
                out[s] += e.device_time_total / 1e3 / reps
                break
    return out


def brick_order(P, delta):
    """the points sorted by bricks of 4 cells of edge 2.02 delta (z, y, x): about the grid's order"""
    b = np.floor((P - P.min(0)) / (4 * 2.02 * delta)).astype(np.int64)
    return np.lexsort((b[:, 0], b[:, 1], b[:, 2]))


def cpu_components(P, radius):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    from scipy.spatial import cKDTree
    t0 = time.perf_counter()
    X = P.astype(np.float64)
    pairs = cKDTree(X).query_pairs(radius, output_type="ndarray")
    n = len(X)
    _, lab = connected_components(coo_matrix((np.ones(len(pairs), np.int8), (pairs[:, 0], pairs[:, 1])), shape=(n, n)),
                                  directed=False)
    ms = (time.perf_counter() - t0) * 1e3
    first = np.full(lab.max() + 1, n, np.int64)
    np.minimum.at(first, lab, np.arange(n))
    return first[lab], ms


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

    for cfg, P, delta, rs, mins in clouds():
        n = len(P)
        labels, root, members = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3))
        offsets, nc = torch.empty(n + 1, dtype=torch.int64, device="cuda"), torch.empty(1, dtype=torch.int64, device="cuda")
        xyz = torch.from_numpy(P[brick_order(P, delta)].copy()).cuda()
        qoff = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        with Context(0) as ctx, torch.cuda.stream(stream):
            ctx.set_stream(stream.cuda_stream)
            ctx.set_cloud_p(P, delta)
            for r in rs:
                sq = float(np.float32(r) * np.float32(r))
                for mn in mins:
                    call = lambda: ctx.euclidean_clusters_dev(sq, labels.data_ptr(), nc.data_ptr(), root.data_ptr(),  # noqa: E731
                                                              offsets.data_ptr(), members.data_ptr(), mn)
                    ms = timed(call)
                    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                        for _ in range(reps):
                            call()
                        stream.synchronize()
                    rc = timed(lambda: ctx._chk(ctx._L.s4g_range_count_dev(ctx.h, xyz.data_ptr(), n, None, sq,
                                                                            qoff.data_ptr())))
                    k = int(nc.item())
                    sizes = np.diff(offsets[:k + 1].cpu().numpy())
                    ours = root.cpu().numpy()
                    row = dict(cfg=cfg, n_p=n, delta=delta, radius=r, radius_in_delta=r / delta, sq_radius=sq, min_size=mn,
                               reps=reps, total_ms=ms, stage_ms=stage_ms(prof, reps), range_count_ms=rc,
                               link_minus_range_count_ms=stage_ms(prof, reps)["link"] - rc,
                               components=int((ours == np.arange(n)).sum()), n_clusters=k,
                               largest=int(sizes[0]) if k else 0, edges_x2=int(qoff[n].item()) - n, device=dev)
                    if mn == mins[0]:
                        try:
                            cpu_root, cpu_ms = cpu_components(P, float(np.sqrt(np.float64(sq))))
                            row.update(cpu_ckdtree_csgraph_ms=cpu_ms, cpu_points_differing=int((cpu_root != ours).sum()))
                        except ImportError:
                            pass
                    print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 5)
