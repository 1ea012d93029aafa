"""Timing of s4g_fpfh and s4g_fpfh_match on the cfg2 P (1M points, delta = 0.003), unbounded, on the s4g_normals
(k = 16) of the same cloud oriented by s4g_orient_normals (k = 16); one JSON line per measurement, with the card's name
and power limit.

GPU, CUDA events around `reps` calls after one warm-up call:
  fpfh      s4g_fpfh_dev at k in {16, 32, 64}: dev_ms the whole call, and from one torch.profiler pass over `reps`
            further calls (CUPTI kernel durations, mean per call) stage_ms: rows = k_normals_queries + k_outlier_exclude +
            k_knn; spfh = k_fpfh_spfh; fpfh = k_fpfh_gather.  At k = 16 every output is compared with the port's on the
            GPU's rows (dev_equals_port).
  fpfh_small  the same call on the first 10^5 points (their own resident cloud), against the port on one thread
            (oracle/fpfh_port.cc with its brute-force rows replaced by the GPU's), timed by the wall clock.
  match     s4g_fpfh_match_dev at n_a = n_b in {10^4, 10^5} (rows of the k = 32 descriptors: a the first n, b the next n),
            mutual off and on.  A tested pair issues 33 x 3 FP32 instructions (-fmad=false); the issue bound is
            132 SMs x 128 lanes x 1.98 GHz, and bound_share = (pairs x 99 / that rate) / dev time.  At 10^4 the outputs
            are compared with the port's (one thread).

usage: python scripts/fpfh_bench.py [reps]
"""
import json
import os
import sys
import time

os.environ.setdefault("OMP_NUM_THREADS", "1")   # the port's timings are single-threaded

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import fpfh as ofpfh  # noqa: E402
from super4pcs_b200 import Context, synth  # noqa: E402

KS = [16, 32, 64]
STAGES = {"rows": ("k_normals_queries", "k_outlier_exclude", "k_knn"), "spfh": ("k_fpfh_spfh",),
          "fpfh": ("k_fpfh_gather",)}
ISSUE_RATE = 132 * 128 * 1.98e9          # FP32 instructions per second, H100 SXM at its boost clock


def stage_ms(prof, reps):
    out = {s: 0.0 for s in STAGES}
    for e in prof.key_averages():
        for s, names in STAGES.items():
            if any(nm in e.key for nm in names):
                out[s] += e.device_time_total / 1e3 / reps
                break
    return out


def bits_equal(a, b):
    return bool(np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)))


def main(reps=5):
    import torch
    n, delta = 1_000_000, 0.003
    P, _ = synth.center(synth.make_pair(n, 0.3, seed=42)["P"])
    P = np.ascontiguousarray(P, np.float32)
    dev = bench.device_info(0, 0)
    stream = torch.cuda.Stream()
    dX = torch.from_numpy(P).cuda()
    excl = torch.arange(n, dtype=torch.int32, device="cuda")
    idx = torch.empty(n * max(KS), dtype=torch.int32, device="cuda")
    sq = torch.empty(n * max(KS), dtype=torch.float32, device="cuda")
    dN = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    dF = torch.empty((n, 33), dtype=torch.float32, device="cuda")
    out2 = torch.empty(2, dtype=torch.int64, device="cuda")

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

    F32 = None
    with Context(0) as ctx, torch.cuda.stream(stream):
        ctx.set_stream(stream.cuda_stream)
        ctx.set_cloud_p(P, delta)
        ctx.normals_dev(16, dN.data_ptr())
        ctx.orient_normals_dev(dN.data_ptr(), 16, dN.data_ptr(), out2.data_ptr())
        stream.synchronize()
        N = dN.cpu().numpy()
        for k in KS:
            call = lambda: ctx.fpfh_dev(dN.data_ptr(), k, dF.data_ptr())  # noqa: E731
            dev_ms = timed(call)
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    call()
                stream.synchronize()
            row = dict(cfg="cfg2", stage="fpfh", k=k, n_p=n, delta=delta, sq_radius="inf", reps=reps, dev_ms=dev_ms,
                       stage_ms=stage_ms(prof, reps), device=dev)
            got = dF.cpu().numpy()
            if k == 32:
                F32 = got.copy()
            if k == 16:
                ctx.knn_dev(dX.data_ptr(), n, k, idx.data_ptr(), sq.data_ptr(), d_exclude_ptr=excl.data_ptr())
                stream.synchronize()
                rows = idx[:n * k].cpu().numpy().reshape(n, k)
                sqs = sq[:n * k].cpu().numpy().reshape(n, k)
                t0 = time.perf_counter()
                want = ofpfh.port(P, N, k, rows=rows, sq=sqs)
                row.update(port_ms_1_thread=(time.perf_counter() - t0) * 1e3, dev_equals_port=bits_equal(got, want))
            print(json.dumps(row), flush=True)

    m = 100_000
    with Context(0) as ctx, torch.cuda.stream(stream):
        ctx.set_stream(stream.cuda_stream)
        ctx.set_cloud_p(P[:m], float(delta * np.sqrt(n / m)))
        for k in KS:
            call = lambda: ctx.fpfh_dev(dN.data_ptr(), k, dF.data_ptr())  # noqa: E731
            dev_ms = timed(call)
            got = dF[:m].cpu().numpy()
            r, s = ctx.knn(P[:m], k, exclude=np.arange(m, dtype=np.int32))
            t0 = time.perf_counter()
            want = ofpfh.port(P[:m], N[:m], k, rows=r, sq=s)
            print(json.dumps(dict(cfg="cfg2[:1e5]", stage="fpfh_small", k=k, n_p=m, dev_ms=dev_ms,
                                  port_ms_1_thread=(time.perf_counter() - t0) * 1e3, dev_equals_port=bits_equal(got, want),
                                  device=dev)), flush=True)

    with Context(0) as ctx, torch.cuda.stream(stream):
        ctx.set_stream(stream.cuda_stream)
        dA = torch.from_numpy(F32).cuda()
        di = torch.empty(n, dtype=torch.int32, device="cuda")
        ds = torch.empty(n, dtype=torch.float32, device="cuda")
        for nm in (10_000, 100_000):
            a, b = dA[:nm], dA[nm:2 * nm]
            for mutual in (False, True):
                call = lambda: ctx.fpfh_match_dev(a.data_ptr(), nm, b.data_ptr(), nm, di.data_ptr(), ds.data_ptr(),  # noqa
                                                  mutual=mutual)
                dev_ms = timed(call)
                pairs = nm * nm * (2 if mutual else 1)
                bound_ms = pairs * 99 / ISSUE_RATE * 1e3
                row = dict(stage="fpfh_match", n_a=nm, n_b=nm, mutual=mutual, reps=reps, dev_ms=dev_ms,
                           pairs_per_s=pairs / (dev_ms / 1e3), fp32_issue_bound_ms=bound_ms,
                           bound_share=bound_ms / dev_ms, matched=int((di[:nm] >= 0).sum()), device=dev)
                if nm == 10_000:
                    t0 = time.perf_counter()
                    want = ofpfh.match_port(F32[:nm], F32[nm:2 * nm], mutual)
                    row.update(port_ms_1_thread=(time.perf_counter() - t0) * 1e3,
                               dev_equals_port=bool(np.array_equal(di[:nm].cpu().numpy(), want[0])) and
                               bits_equal(ds[:nm].cpu().numpy(), want[1]))
                print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 5)
