"""Round-2 measurement of row e INSIDE the C++ layer (S4PCS_DEVICES, DESIGN.md section 6): times
Match4PCSBase::TryCongruentSet -- rigid fits + gate + Verify + arg-max of one congruent set -- through the header-compatible
C++ layer (TestMatcher-style harness, oracle/_dropin) for several device-context specs on the cfg2-sized pair, and checks
that every spec returns the same winner.  One JSON line per spec.

  python scripts/devices_bench.py --points 1000000 --devices "1 2 2+nccl 4 8 8+nccl 0,0"
  LD_PRELOAD=tests/_build/libs4g_oracle_shim.so python scripts/devices_bench.py --points 20000 --delta 0.02 --neigh 3   # CPU dry run

The congruent set is synthetic: a wide base of P, and for each of its four points the `neigh` sampled-Q points nearest to
its ground-truth pre-image -- neigh^4 quads, most of which pass the rms gate, i.e. that many full Verify passes per call.
Test / measurement infrastructure (it drives the product through the oracle's harness); not part of the product."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import _build, ref as oref  # noqa: E402
from super4pcs_b200 import synth  # noqa: E402


def congruent_set(Ps, Qs, cp, cq, neigh, seed=3):
    from scipy.spatial import cKDTree
    rng = np.random.RandomState(seed)
    gt = synth.gt_transform()
    R, t = gt[:3, :3], gt[:3, 3]
    tree = cKDTree(Qs.astype(np.float64))
    best = None
    for _ in range(200):                                   # a wide base whose pre-images all lie on the overlap
        ids = rng.randint(0, len(Ps), 4)
        pre = (Ps[ids].astype(np.float64) + cp - t) @ R - cq          # R^T (p + cP - t) - cQ, row-vector form
        d, nn = tree.query(pre, k=neigh)
        nn = nn.reshape(4, -1)
        spread = np.linalg.norm(Ps[ids][:, None] - Ps[ids][None], axis=2)
        score = spread[np.triu_indices(4, 1)].min() - 50.0 * np.max(d)
        if best is None or score > best[0]:
            best = (score, ids, nn)
    _, ids, nn = best
    quads = np.stack(np.meshgrid(nn[0], nn[1], nn[2], nn[3], indexing="ij"), -1).reshape(-1, 4)
    return ids.astype(np.int32), np.ascontiguousarray(quads, np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1000000)
    ap.add_argument("--delta", type=float, default=0.003)
    ap.add_argument("--overlap", type=float, default=0.3)
    ap.add_argument("--neigh", type=int, default=8, help="neigh^4 quads in the congruent set")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--devices", default="1 2 4 8", help="space-separated S4PCS_DEVICES values")
    args = ap.parse_args()
    if _build.build_dropin_harness() is None:
        raise SystemExit("drop-in harness not built (needs Eigen at build time; run __graft_entry__.build() where the reference is)")
    d = synth.make_pair(args.points, args.overlap, seed=42)
    _, cp = synth.center(d["P"])
    _, cq = synth.center(d["Q"])
    opt = oref.make_options(delta=args.delta, sample_size=10 ** 9, overlap=args.overlap)
    base = quads = first = None
    for spec in args.devices.split():
        # "4" = host merge of the shard records (default); "4+nccl" = S4PCS_NCCL=1, reduction inside libs4g over NCCL
        os.environ["S4PCS_DEVICES"] = spec.split("+")[0]   # read by the matcher's constructor
        os.environ["S4PCS_NCCL"] = "1" if spec.endswith("+nccl") else "0"
        t0 = time.perf_counter()
        m = oref.RefMatcher(d["P"], d["Q"], opt, libpath=_build.DROPIN_SO)
        setup = time.perf_counter() - t0
        if quads is None:
            Ps, _, _ = m.sampled_p()
            Qs, _, _ = m.sampled_q()
            base, quads = congruent_set(Ps, Qs, cp.astype(np.float64), cq.astype(np.float64), args.neigh)
        t0 = time.perf_counter()
        r = m.try_congruent_set(base, quads)               # warm-up: peers (and the communicator) are created, scratch grows
        first_call = time.perf_counter() - t0
        ms = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            r = m.try_congruent_set(base, quads)
            ms.append(1e3 * (time.perf_counter() - t0))
        m.close()
        sig = (float(np.float32(r["best_lcp"])), int(r["n_gate"]), [int(x) for x in r["congruent"]],
               [int(x) for x in r["T"].view(np.uint32)])
        first = first or sig
        ms.sort()
        print(json.dumps({"devices": spec, "points": args.points, "delta": args.delta, "quads": int(len(quads)),
                          "gate_passing": sig[1], "best_lcp": sig[0], "median_ms": round(ms[len(ms) // 2], 3),
                          "min_ms": round(ms[0], 3), "verified_per_s": round(sig[1] / (1e-3 * ms[len(ms) // 2]), 1),
                          "setup_s": round(setup, 3), "first_call_s": round(first_call, 3),
                          "identical_to_first": sig == first}), flush=True)


if __name__ == "__main__":
    main()
