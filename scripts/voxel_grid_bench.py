"""Timing of voxel-grid downsampling (s4g_voxel_grid), one JSON line per case, each with the card's name and power limit.

Clouds: n in {10^6, 10^7, 5 10^7} points uniform in the unit cube, with unit normals and rgb, at leaves that put about
1, 8 and 64 points in a voxel; min_points = 1, every output requested.

GPU, CUDA events around `reps` calls after one warm-up call:
  dev_ms        the _dev form on device arrays (the library's own work)
  host_ms       the host form (adds the copies of the inputs and outputs)
  sample_ms     s4g_voxel_sample at the same n and leaf (host form; it keeps the first point of each voxel)
then one torch.profiler pass over `reps` further _dev calls (CUPTI kernel durations, mean per call) split into stages:
  keys          k_vg_init + k_vg_bounds + k_vg_keys
  sort          cub's radix sort of the (key, index) pairs, 63 bits
  segments      k_vg_heads + k_vg_starts + the two cub scans (voxel of each sorted position, output index of each voxel)
  gather        k_vg_gather (xyz, normals and rgb into sorted order)
  sums          k_vg_runs + k_vg_final
  outputs       k_vg_flags + k_vg_count + k_vg_voxel_of
Bytes: io_bytes is what any implementation has to move, computed from the shapes: the inputs once (36 bytes per point),
every output once (40 bytes per voxel: centroid, normal, rgb, count, first) and voxel_of (4 bytes per point).
io_tb_per_s = io_bytes / dev time, against the H100 SXM data sheet's 3.35 TB/s of HBM3.
CPU: the port (oracle/voxel_grid_port.cc, one thread) on the same arrays, its wall clock, and whether every output of the
GPU equals it bit for bit; `first_equals_voxel_sample` compares `first` with s4g_voxel_sample's output.

usage: python scripts/voxel_grid_bench.py [reps]
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import voxel_grid as ovg  # noqa: E402
from super4pcs_b200 import Context  # noqa: E402

NS = [1_000_000, 10_000_000, 50_000_000]
PPVS = [1, 8, 64]
HBM_TBS = 3.35
STAGES = {"keys": ("k_vg_init", "k_vg_bounds", "k_vg_keys"), "sort": ("DeviceRadixSort",),
          "segments": ("k_vg_heads", "k_vg_starts", "DeviceScan"), "gather": ("k_vg_gather",),
          "sums": ("k_vg_runs", "k_vg_final"), "outputs": ("k_vg_flags", "k_vg_count", "k_vg_voxel_of")}


def cloud(n, seed):
    rng = np.random.RandomState(seed)
    X = rng.random_sample((n, 3)).astype(np.float32)
    N = rng.normal(0, 1, (n, 3)).astype(np.float32)
    N /= np.linalg.norm(N, axis=1, keepdims=True)
    R = rng.random_sample((n, 3)).astype(np.float32)
    return X, N, R


def stage_ms(prof, reps):
    out = {s: 0.0 for s in STAGES}
    for e in prof.key_averages():
        for s, names in STAGES.items():
            if any(nm in e.key for nm in names):
                out[s] += e.device_time_total / 1e3 / reps
                break
    return out


def equal(a, b):
    for x, y in zip(a, b):
        if x is None and y is None:
            continue
        if x is None or y is None or x.shape != y.shape or not np.array_equal(np.asarray(x).view(np.uint32),
                                                                              np.asarray(y).view(np.uint32)):
            return False
    return True


def main(reps=10):
    import torch
    dev = bench.device_info(0, 0)
    stream = torch.cuda.Stream()

    def timed(call, k):
        call()
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(k):
            call()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / k

    for n in NS:
        X, N, R = cloud(n, seed=n % 1000)
        k = reps if n <= 10_000_000 else max(2, reps // 2)
        dX, dN, dR = (torch.from_numpy(a).cuda() for a in (X, N, R))
        oX, oN, oR = (torch.empty((n, 3), dtype=torch.float32, device="cuda") for _ in range(3))
        cnt, fst, vof = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(3))
        m = torch.empty(1, dtype=torch.int64, device="cuda")
        for ppv in PPVS:
            leaf = float((ppv / n) ** (1.0 / 3.0))
            with Context(0) as ctx, torch.cuda.stream(stream):
                ctx.set_stream(stream.cuda_stream)
                call = lambda: ctx.voxel_grid_dev(dX.data_ptr(), n, leaf, oX.data_ptr(), m.data_ptr(),  # noqa: E731
                                                  dN.data_ptr(), dR.data_ptr(), oN.data_ptr(), oR.data_ptr(),
                                                  cnt.data_ptr(), fst.data_ptr(), vof.data_ptr())
                dev_ms = timed(call, k)
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(k):
                        call()
                    stream.synchronize()
                stages = stage_ms(prof, k)
                got = None

                def host():
                    nonlocal got
                    got = ctx.voxel_grid(X, leaf, N, R)
                host_ms = timed(host, k)
                sample = None

                def vs():
                    nonlocal sample
                    sample = ctx.voxel_sample(X, leaf)
                sample_ms = timed(vs, k)
            n_out = len(got[0])
            dev_out = (oX[:n_out].cpu().numpy(), oN[:n_out].cpu().numpy(), oR[:n_out].cpu().numpy(),
                       cnt[:n_out].cpu().numpy(), fst[:n_out].cpu().numpy(), vof.cpu().numpy())
            t0 = time.perf_counter()
            want = ovg.port(X, leaf, N, R)
            port_ms = (time.perf_counter() - t0) * 1e3
            io_bytes = 36 * n + 40 * n_out + 4 * n
            row = dict(stage="voxel_grid", n=n, leaf=leaf, points_per_voxel_target=ppv, n_out=n_out,
                       mean_points_per_voxel=n / n_out, reps=k, dev_ms=dev_ms, host_ms=host_ms, sample_ms=sample_ms,
                       points_per_s=n / (dev_ms / 1e3), stage_ms=stages, io_bytes=io_bytes,
                       io_tb_per_s=io_bytes / (dev_ms / 1e3) / 1e12, io_share_of_hbm=io_bytes / (dev_ms / 1e3) / 1e12 / HBM_TBS,
                       port_ms_1_thread=port_ms, host_equals_port=equal(got, want), dev_equals_port=equal(dev_out, want),
                       first_equals_voxel_sample=bool(np.array_equal(got[4], sample)), device=dev)
            print(json.dumps(row), flush=True)
        del dX, dN, dR, oX, oN, oR, cnt, fst, vof
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 10)
