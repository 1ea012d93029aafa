"""Where k_verify's cycles go, per phase, on bench.py's workload (1M x 1M points, the same seeded 4096 candidates).

Builds libs4g with -DS4G_VERIFY_CLOCKS=1 into a temporary directory (the tree's library is left as it is), runs Verify
--warmup + --steps times with the L2 flushed before every step, and prints one JSON line: the SM cycles of every warp of
the timed launches summed per phase of k_verify (super4pcs_b200/csrc/verify.cu, g_verify_clocks) and their shares, with
the card's name, power limit and median SM clock.  The clock reads cost a few instructions per tile, so the kernel time
printed beside the split is that of the instrumented build, not of the shipped one.

    python scripts/verify_phases.py [--steps 10] [--warmup 3]
"""
import argparse
import ctypes as C
import json
import os
import shutil
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from super4pcs_b200 import build, s4g  # noqa: E402

PHASES = ("stage_and_cull", "lookups", "queue_and_exact", "rest")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("verify_phases.py: no CUDA device")
    tmp = tempfile.mkdtemp(prefix="s4g_phases_")
    try:
        lib = build.build_lib(force=True, extra_flags=("-DS4G_VERIFY_CLOCKS=1",), out_dir=tmp)
        s4g.lib_path = lambda: lib                 # every Context of this process loads the instrumented build
        L = s4g.load_library()
        L.s4g_verify_clocks.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
        L.s4g_verify_clocks.restype = C.c_int

        _, P, Q, cp, cq = bench.build_workload(bench.N_POINTS)
        gs = bench.GpuStages(0)
        T, _ = bench.make_candidates(bench.CANDIDATES_PER_GPU, P, Q, cp, cq, 7, gs)   # bench.py's list on rank 0
        gs.ctx.close()
        ctx = s4g.Context(0)
        ctx.set_cloud_p(P, bench.DELTA)
        ctx.set_cloud_q(Q)
        dev = torch.device("cuda", 0)
        d_T = torch.from_numpy(np.ascontiguousarray(T)).to(dev)
        d_counts = torch.zeros(len(T), dtype=torch.int32, device=dev)
        flush = torch.empty(bench.L2_FLUSH_BYTES // 4, dtype=torch.float32, device=dev)
        clocks = np.zeros(4, np.uint64)

        def read_clocks(reset):
            rc = L.s4g_verify_clocks(ctx.h, clocks.ctypes.data, int(reset))
            if rc != 0:
                raise RuntimeError("s4g_verify_clocks: %d" % rc)
            return clocks.copy()

        for _ in range(args.warmup):
            ctx.verify_dev(d_T.data_ptr(), len(T), d_counts.data_ptr())
        torch.cuda.synchronize()
        read_clocks(True)
        sampler = bench.ClockSampler(0)
        sampler.start()
        kernel_ms = 0.0
        for _ in range(args.steps):
            flush.fill_(1.0)
            torch.cuda.synchronize()
            ctx.verify_dev(d_T.data_ptr(), len(T), d_counts.data_ptr())
            ctx.synchronize()
            kernel_ms += ctx.timings()["verify_ms"]
        sampler.stop_flag.set()
        sampler.join(timeout=5)
        c = read_clocks(True).astype(np.float64)
        split = dict(zip(PHASES[:3], c[:3]))
        split["rest"] = c[3] - c[:3].sum()
        print(json.dumps({
            "what": "k_verify warp-cycles per phase, bench.py workload (%d candidates, %d points)" % (len(T), bench.N_POINTS),
            "steps": args.steps,
            "cycles_per_step": {k: v / args.steps for k, v in split.items()},
            "share": {k: round(v / c[3], 4) for k, v in split.items()},
            "kernel_ms_instrumented": kernel_ms / args.steps,
            "device": bench.device_info(0, 0),
            "clocks": sampler.summary(),
        }), flush=True)
        ctx.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
