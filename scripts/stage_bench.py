"""Secondary stage figures of SURVEY.md 8(d) (not the headline metric, see bench.py):

  cfg1  50K-pt pair, 40 % overlap, delta=0.01: ExtractPairs d=1.0 (ordered pairs/s), one whole base
        (pairs x2 -> quads -> TryCongruentSet) at |sampled_Q| = 3000 / 10000, Verify at 50K x 50K
  cfg3  200K-pt pair + noise + outliers, normals on (max_normal_difference = 30 deg), n = 10000
  cfg2  1M x 1M pair, delta=0.003: the nearest P point within delta of every query (s4g_verify_nearest_dev), ms per
        transform for a near-ground-truth and a wrong transform, CUDA events, with the card's name and power limit
  cfg4  10M-pt pair: grid build (points/s) and the counting-only shell query at eps = 2e-4

usage: python scripts/stage_bench.py [cfg1] [cfg2] [cfg3] [cfg4]   -> one JSON line per figure
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from super4pcs_b200 import Context, PairFilters, synth  # noqa: E402


def timed(fn, reps=3):
    fn()
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        r = fn()
        ts.append(time.perf_counter() - t)
    return r, min(ts)


def out(**kw):
    print(json.dumps(kw), flush=True)


def hbm_peak():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 6650.0


def roofline(algorithmic_bytes, kernel_ms):
    """SURVEY.md 8(d): achieved = algorithmic bytes / device time, against the measured HBM copy peak"""
    gbs = algorithmic_bytes / (kernel_ms * 1e-3) / 1e9 if kernel_ms else None
    return {"algorithmic_bytes": algorithmic_bytes, "achieved_gbs": gbs, "hbm_peak_gbs": hbm_peak(),
            "hbm_frac": gbs / hbm_peak() if gbs else None}


def whole_base(ctx, P, rng, delta, filters=None, normals=None):
    diameter = float(np.linalg.norm(P.max(0) - P.min(0)))
    psub = P[rng.choice(len(P), min(len(P), 20000), replace=False)]
    ids, inv1, inv2 = bench.select_base(psub, rng, diameter)
    bx = psub[ids]
    b9 = [np.concatenate([bx[i], [0, 0, 0], [-1, -1, -1]]).astype(np.float32) for i in range(4)]
    d1, d2 = bench._eigen_norm(bx[0] - bx[1]), bench._eigen_norm(bx[2] - bx[3])
    t0 = time.perf_counter()
    n1 = ctx.extract_pairs(d1, 0.0, 2 * delta, b9[0], b9[1], filters, slot=0, fetch=False)
    n2 = ctx.extract_pairs(d2, 0.0, 2 * delta, b9[2], b9[3], filters, slot=1, fetch=False)
    t1 = time.perf_counter()
    nq = ctx.find_quads(inv1, inv2, 2 * delta, bx, fetch=False)
    t2 = time.perf_counter()
    r = ctx.try_congruent_set_resident(bx, 2 * delta)
    t3 = time.perf_counter()
    tm = ctx.timings()
    nQ = ctx.nQ
    # SURVEY.md 8(d) algorithmic bytes: quads (n1+n2)(8 + 2*16) + n1*8 + K*16; rigid 16 + 48 read per quad, 56 written per pass
    return dict(pairs=[n1, n2], quads=nq, verified=r["n_gate_pass"], best_lcp=r["best_count"] / max(1, r["n_q"]),
                pairs_s=t1 - t0, quads_s=t2 - t1, tcs_s=t3 - t2,
                device_ms=dict(pairs_last_call=tm["pairs_ms"], quads=tm["quads_ms"], rigid=tm["rigid_ms"], verify=tm["verify_ms"]),
                roofline_pairs_last_call=roofline(nQ * 64.0 + n2 * 8.0, tm["pairs_ms"]),
                roofline_quads=roofline((n1 + n2) * 40.0 + n1 * 8.0 + nq * 16.0, tm["quads_ms"]),
                roofline_rigid=roofline(nq * 64.0 + r["n_gate_pass"] * 56.0, tm["rigid_ms"]))


def cfg1():
    n, delta = 50_000, 0.01
    d = synth.make_pair(n, 0.4, seed=42)
    P, cp = synth.center(d["P"])
    Q, cq = synth.center(d["Q"])
    with Context(0) as ctx:
        ctx.set_cloud_p(P, delta)
        ctx.set_cloud_q(Q)
        k, t = timed(lambda: ctx.extract_pairs(1.0, 0.0, 2 * delta, fetch=False))
        km = ctx.timings()["pairs_ms"]
        # SURVEY.md 8(d): B_pairs = N_Q (16 pos + 3 x 16 side arrays) read + 8 B per ordered pair written (the output dominates)
        out(cfg="cfg1", stage="ExtractPairs", n_q=n, d=1.0, eps=2 * delta, ordered_pairs=k, seconds=t,
            pairs_per_s=k / t, kernel_ms=km, reference_pairs_per_s_1thread=1.0e7, roofline=roofline(n * 64.0 + k * 8.0, km))
        T = bench.make_candidates(256, P, Q, cp, cq, 7, bench.GpuStages(0))[0]
        c, t = timed(lambda: ctx.verify(T))
        out(cfg="cfg1", stage="Verify", n_p=n, n_q=n, candidates=len(T), seconds=t, candidates_per_s=len(T) / t,
            kernel_ms=ctx.timings()["verify_ms"])
        for ns in (3000, 10000):
            rng = np.random.RandomState(ns)
            ctx.set_cloud_q(Q[rng.choice(n, ns, replace=False)])
            for b in range(3):
                out(cfg="cfg1", stage="base", sample_size=ns, base=b, **whole_base(ctx, P, rng, delta))


def cfg2(reps=20):
    import torch
    n, delta = 1_000_000, 0.003
    d = synth.make_pair(n, 0.3, seed=42)
    P, cp = synth.center(d["P"])
    Q, cq = synth.center(d["Q"])
    M = synth.candidate_transforms(2, delta, seed=7, n_near=1, centroid_p=cp, centroid_q=cq)   # near-GT, then a random one
    T = np.ascontiguousarray(M.transpose(0, 2, 1)).reshape(-1, 16)
    stream = torch.cuda.Stream()            # an explicit stream: handle 0 would mean the context's own stream
    with Context(0) as ctx, torch.cuda.stream(stream):
        ctx.set_cloud_p(P, delta)
        ctx.set_cloud_q(Q)
        ctx.set_stream(stream.cuda_stream)
        gs = ctx.grid_stats()
        counts = ctx.verify(T)
        idx = torch.empty(n, dtype=torch.int32, device="cuda")
        sq = torch.empty(n, dtype=torch.float32, device="cuda")
        cnt = torch.empty(1, dtype=torch.int32, device="cuda")
        for k, which in enumerate(("near_gt", "wrong")):
            dT = torch.from_numpy(T[k:k + 1].copy()).cuda()
            call = lambda: ctx.verify_nearest_dev(dT.data_ptr(), 1, idx.data_ptr(), sq.data_ptr(), cnt.data_ptr())  # noqa: E731
            call()
            stream.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(reps):
                call()
            e1.record(stream)
            e1.synchronize()
            ms = e0.elapsed_time(e1) / reps
            hits = int(cnt.item())
            assert hits == int(counts[k]), "nearest count differs from Verify's"
            # bytes model: every query read (16 B) and its index + sq_dist written (8 B), plus the grid and the sorted P
            # (the resident bytes of the grid statistics) read once -- an upper-end model for a wrong transform, whose
            # queries mostly land outside the occupied cells and read little of the grid
            out(cfg="cfg2", stage="verify_nearest", transform=which, n_p=n, n_q=n, delta=delta, inliers=hits,
                ms_per_transform=ms, queries_per_s=n / (ms * 1e-3), roofline=roofline(n * 24.0 + gs["resident_bytes"], ms),
                device=bench.device_info(0, 0))


def cfg3():
    n, delta = 200_000, 0.01
    d = synth.make_pair(n, 0.4, seed=43, noise_sigma=0.005, outlier_frac=0.2, with_normals=True)
    P, _ = synth.center(d["P"])
    Q, _ = synth.center(d["Q"])
    rng = np.random.RandomState(3)
    sel = rng.choice(n, 10000, replace=False)
    Qn = d["Qn"][sel] / np.linalg.norm(d["Qn"][sel], axis=1, keepdims=True)
    with Context(0) as ctx:
        ctx.set_cloud_p(P, delta)
        ctx.set_cloud_q(Q[sel], normals=Qn.astype(np.float32))
        f = PairFilters(30.0, -1, -1, -1)
        for b in range(3):
            out(cfg="cfg3", stage="base", sample_size=10000, base=b, normals=True, **whole_base(ctx, P, rng, delta, f))


def cfg4():
    n = 10_000_000
    d = synth.make_pair(n, 0.2, seed=44)
    P, _ = synth.center(d["P"])
    Q, _ = synth.center(d["Q"])
    with Context(0) as ctx:
        _, t = timed(lambda: ctx.set_cloud_p(P, 0.001), reps=2)
        out(cfg="cfg4", stage="grid_build_P", n=n, delta=0.001, seconds=t, points_per_s=n / t, grid=ctx.grid_stats(),
            note="includes the H2D copy of 120 MB and the host-side bounding box")
        _, t = timed(lambda: ctx.set_cloud_q(Q), reps=2)
        out(cfg="cfg4", stage="morton_index_Q", n=n, seconds=t, points_per_s=n / t)
        k, t = timed(lambda: ctx.count_pairs(1.0, 2e-4), reps=1)
        out(cfg="cfg4", stage="count_pairs", n=n, d=1.0, eps=2e-4, ordered_pairs=k, seconds=t, pairs_per_s=k / t)


if __name__ == "__main__":
    which = sys.argv[1:] or ["cfg1"]
    for w in which:
        {"cfg1": cfg1, "cfg2": cfg2, "cfg3": cfg3, "cfg4": cfg4}[w]()
