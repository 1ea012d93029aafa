"""Timing of the plane segmentation (s4g_segment_planes), one round (max_planes = 1, refine on), one JSON line per case,
each with the card's name, power limit and largest SM clock:
  cfg2   the cfg2 P (1M points, centred), threshold 0.003 (delta)
  room   a 1M-point room (tests/planes.py: a floor and two walls, noise 0.002), threshold 0.01
at n_hypotheses H = 256, 1024 and 4096.

GPU, CUDA events around `reps` calls of the _dev form after one warm-up call, then one torch.profiler pass over `reps`
further calls (CUPTI kernel durations, mean per call) split into stages:
  count          k_plane_count (the H x nP tests)
  active_draws   k_plane_active + the select of the active points + k_plane_gather + k_plane_hypotheses + k_plane_argmax
  refit_label    k_plane_inliers + the select of the inliers + k_plane_runs + k_plane_centroid + k_plane_refit +
                 k_plane_final + k_plane_accept + k_plane_label
  members        k_plane_member_keys + the radix sort
  copies         the memsets and the device-to-device copy of the members
Rate: tests/s = H nP / count time.  Bound: a test is 3 FMUL + 3 FADD, unfused (the contract forbids FMA), so at most
132 SMs x 128 fp32 lanes x the largest SM clock (nvidia-smi clocks.max.sm) such instructions per second; the share is
that bound's time over the count time (the compare and the counter increment are not counted in the bound).
CPU baseline: oracle/planes_port.cc (OpenMP on every core) on the same cloud, wall clock, and whether its outputs equal
the device's (labels, plane bits, members, hyp_counts).

usage: python scripts/planes_bench.py [reps]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from super4pcs_b200 import Context, s4g, synth  # noqa: E402

STAGES = {"count": ("k_plane_count",),
          "active_draws": ("k_plane_active", "k_plane_gather", "k_plane_hypotheses", "k_plane_argmax"),
          "refit_label": ("k_plane_inliers", "k_plane_runs", "k_plane_centroid", "k_plane_refit", "k_plane_final",
                          "k_plane_accept", "k_plane_label"),
          "members": ("k_plane_member_keys", "RadixSort"),
          "copies": ("Memset", "Memcpy")}
SELECT = ("DeviceSelect", "DeviceCompact", "Select")      # CUB's select kernels: split between the two selects


def clouds():
    from tests import planes as tp
    P2, _ = synth.center(synth.make_pair(1_000_000, 0.3, seed=42)["P"])
    room = tp.room(1_000_000, noise=0.002, seed=3)[0]
    return [("cfg2", np.ascontiguousarray(P2, np.float32), 0.003), ("room", room, 0.01)]


def stage_ms(prof, reps):
    out = {s: 0.0 for s in STAGES}
    out["selects"] = 0.0
    for e in prof.key_averages():
        for s, names in STAGES.items():
            if any(nm in e.key for nm in names):
                out[s] += e.device_time_total / 1e3 / reps
                break
        else:
            if any(nm in e.key for nm in SELECT):
                out["selects"] += e.device_time_total / 1e3 / reps
    return out


def max_sm_clock_mhz():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=60)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def main(reps=10):
    import torch
    from oracle import planes as op
    dev = bench.device_info(0, 0)
    dev["max_sm_clock_mhz"] = max_sm_clock_mhz()
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

    for cfg, P, thr in clouds():
        n = len(P)
        labels, members = (torch.empty(n, dtype=torch.int32, device="cuda") for _ in range(2))
        offsets, n_planes = torch.empty(2, dtype=torch.int64, device="cuda"), torch.empty(1, dtype=torch.int32, device="cuda")
        planes = torch.empty(64, dtype=torch.uint8, device="cuda")
        with Context(0) as ctx, torch.cuda.stream(stream):
            ctx.set_stream(stream.cuda_stream)
            ctx.set_cloud_p(P, 0.01)
            for H in (256, 1024, 4096):
                counts = torch.empty(H, dtype=torch.int32, device="cuda")
                call = lambda: ctx.segment_planes_dev(thr, labels.data_ptr(), planes.data_ptr(), n_planes.data_ptr(),  # noqa: E731
                                                      offsets.data_ptr(), members.data_ptr(), counts.data_ptr(), H)
                ms = timed(call)
                with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                    for _ in range(reps):
                        call()
                    stream.synchronize()
                st = stage_ms(prof, reps)
                k = int(n_planes.item())
                rec = planes.cpu().numpy().view(s4g.PLANE_DTYPE)[:k]
                off = offsets[:k + 1].cpu().numpy()
                got = (labels.cpu().numpy(), rec, off, members[:off[-1]].cpu().numpy(),
                       counts.cpu().numpy().view(np.uint32).reshape(1, H))
                tests = float(H) * n
                row = dict(cfg=cfg, n_p=n, threshold=thr, n_hypotheses=H, reps=reps, call_ms=ms, stage_ms=st,
                           tests_per_s=tests / (st["count"] / 1e3) if st["count"] else None,
                           n_inliers=int(rec[0]["n_inliers"]) if k else 0,
                           hypothesis_inliers=int(rec[0]["hypothesis_inliers"]) if k else 0, device=dev)
                if dev["max_sm_clock_mhz"] and st["count"]:
                    lanes_per_s = dev["sm_count"] * 128 * dev["max_sm_clock_mhz"] * 1e6
                    bound_ms = 6 * tests / lanes_per_s * 1e3
                    row.update(fp32_issue_bound_ms=bound_ms, share_of_fp32_issue_bound=bound_ms / st["count"])
                t0 = time.perf_counter()
                want = op.planes(P, thr, H, hyp_counts=True)
                row.update(cpu_port_ms=(time.perf_counter() - t0) * 1e3, cpu_threads=os.cpu_count(),
                           cpu_port_equal=all(a.tobytes() == b.tobytes() for a, b in zip(got, want)))
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 10)
