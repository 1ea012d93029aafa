#!/usr/bin/env python
"""bench.py -- candidate transforms LCP-verified per second at 1M points (BASELINE.json metric).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
           --master-port P bench.py --gpus N --steps K --warmup W

Workload (BASELINE.json configs[2], SURVEY.md 8(d) cfg2): synthetic bumpy-sphere pair, 1M points
each, 30 % overlap, delta = 0.003, |sampled_P| = |sampled_Q| = 1e6 (whole clouds), clouds + grid
replicated in every GPU's HBM.  A step = one pass of the hot path (Match4PCSBase::Verify, a8) over
a batch of 4096 candidate transforms PER GPU (weak scaling: candidate sets shard embarrassingly),
followed by the one collective of the path: a max-allreduce of the packed (count, index) key --
since round 2 inside libs4g (ncclAllReduce on the stream of the Verify kernel, csrc/comm.cu).

  value  : candidates/s with the transforms already resident in HBM (s4g_verify_best_dev).
  e2e    : the same metric through the host-buffer C-ABI call s4g_verify_best (pinned host transforms
           + indices in, host counts + key out: the H2D and D2H copies are inside the timed region).
  roofline: Verify kernel, algorithmic bytes N_Q (16 + 8 C + 16 k) per candidate with C, k measured
           on the built grid by the kernel's own statistics variant (DESIGN.md section 5).
  device : name, SM count and power limit of the GPU the numbers were measured on.
  cpu_baseline: the reference's own Verify (oracle/_ref, unmodified reference, OpenMP over
           candidates = the reference's own parallelisation) on a bounded sample of the SAME
           candidates, on this box's host cores.

--impl reference runs only that CPU arm, with the same config/metric/unit.
--dump-outputs DIR writes what the last timed step computed (the counts and the winner of the resident call) as
DIR/<name>.npy in float64; the inputs are seeded, so two builds can be compared output for output.
Only the cpu_baseline / --impl reference legs touch oracle/ (as the thing being compared against).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

# The CPU arm binds its OpenMP threads to physical cores (one thread per core, no SMT siblings, no migration): the
# unbound all-hyperthreads run of round 1 moved 5x between two boxes.  Must be in the environment before libgomp starts.
# Only where the CPU arm can run in this process (N = 1, or --impl reference): under torchrun with N > 1 the binding would
# pin the main thread of every rank to the first core.
if int(os.environ.get("WORLD_SIZE", "1") or 1) == 1 or "reference" in sys.argv:
    os.environ.setdefault("OMP_PROC_BIND", "close")
    os.environ.setdefault("OMP_PLACES", "cores")

if int(os.environ.get("WORLD_SIZE", "1") or 1) > 1:
    # NCCL's own log (communicator ranks, transports, NVLS) at INFO unless the caller chose a level; set before torch /
    # NCCL are loaded.  It goes to stderr with everything else that writes to fd 1 (isolate_stdout).
    # (S4_NCCL_DEBUG overrides; a pre-set VERSION / WARN -- some images export one -- is raised to INFO so that the
    # communicator's rank count can be read from the log.)
    if os.environ.get("S4_NCCL_DEBUG"):
        os.environ["NCCL_DEBUG"] = os.environ["S4_NCCL_DEBUG"]
    elif os.environ.get("NCCL_DEBUG", "").upper() in ("", "VERSION", "WARN"):
        os.environ["NCCL_DEBUG"] = "INFO"

try:                                   # before libgomp binds the main thread to its first place
    _CPUS = sorted(os.sched_getaffinity(0))
except AttributeError:
    _CPUS = list(range(os.cpu_count() or 1))

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

METRIC = "candidate transforms LCP-verified/sec at 1M pts"
UNIT = "candidates/s"
N_POINTS = 1_000_000
OVERLAP = 0.30
DELTA = 0.003
CANDIDATES_PER_GPU = 4096
N_NEAR = 64
L2_FLUSH_BYTES = 256 << 20
H100_HBM_GBS = 3350.0   # NVIDIA H100 SXM data sheet; the fallback peak when no measured one is at hand


def host_threads():
    """CPUs this process may run on (torchrun pins OMP_NUM_THREADS=1, so the OpenMP default cannot be trusted; the
    count is passed explicitly to num_threads())"""
    return max(1, len(_CPUS))


def physical_cores():
    """physical cores among the CPUs this process may run on (SMT siblings counted once): the thread count of the
    CPU arm.  Falls back to host_threads() when /sys is not readable."""
    seen = set()
    for c in _CPUS:
        try:
            base = "/sys/devices/system/cpu/cpu%d/topology/" % c
            seen.add((open(base + "physical_package_id").read().strip(), open(base + "core_id").read().strip()))
        except OSError:
            return host_threads()
    return max(1, len(seen))


def _env_int(name, default):
    try:
        return int(os.environ.get(name, default))
    except ValueError:
        return default


def build_workload(n_points, seed=42):
    from super4pcs_b200 import synth
    d = synth.make_pair(n_points, OVERLAP, seed=seed)
    P, cp = synth.center(d["P"])
    Q, cq = synth.center(d["Q"])
    return d, P, Q, cp, cq


EXTRACT_N = 3000        # |sampled_Q| of the extraction that feeds the candidate list (SURVEY 8(d) cfg2)
EXTRACT_DELTA = 0.01


def _closest_params(a, b, c, d):
    """parameters (s, t) in [0,1] of the closest points of segments ab and cd (float64)"""
    u, v, w = b - a, d - c, a - c
    A, B, C, D, E = u @ u, u @ v, v @ v, u @ w, v @ w
    den = A * C - B * B
    s = 0.5 if den < 1e-12 else np.clip((B * E - C * D) / den, 0.0, 1.0)
    t = np.clip((B * s + E) / C, 0.0, 1.0)
    s = np.clip((B * t - D) / A, 0.0, 1.0)
    return float(s), float(t), float(np.linalg.norm(w + s * u - t * v))


def select_base(P, rng, diameter):
    """a wide, near-planar 4-point base of P with its two invariants (host side of the RANSAC loop;
    workload generator only -- the drop-in C++ layer has the reference-exact selection)"""
    n = len(P)
    for _ in range(200):
        i0 = rng.randint(n)
        c = rng.randint(n, size=(512, 2))
        u, w = P[c[:, 0]] - P[i0], P[c[:, 1]] - P[i0]
        wide = np.linalg.norm(np.cross(u, w), axis=1)
        wide[(np.linalg.norm(u, axis=1) > 0.7 * diameter) | (np.linalg.norm(w, axis=1) > 0.7 * diameter)] = -1
        k = int(np.argmax(wide))
        if wide[k] <= 0:
            continue
        i1, i2 = int(c[k, 0]), int(c[k, 1])
        nrm = np.cross(P[i1] - P[i0], P[i2] - P[i0]).astype(np.float64)
        nrm /= np.linalg.norm(nrm)
        dist = np.abs((P - P[i0]).astype(np.float64) @ nrm)
        far = np.ones(n, bool)
        for i in (i0, i1, i2):
            far &= np.linalg.norm(P - P[i], axis=1) > 0.2 * diameter
        if not far.any():
            continue
        dist[~far] = np.inf
        i3 = int(np.argmin(dist))
        ids = [i0, i1, i2, i3]
        best = None
        for (a, b, cc, d) in ((0, 1, 2, 3), (0, 2, 1, 3), (0, 3, 1, 2)):
            s_, t_, dd = _closest_params(*(P[ids[j]].astype(np.float64) for j in (a, b, cc, d)))
            if best is None or dd < best[0]:
                best = (dd, [ids[a], ids[b], ids[cc], ids[d]], s_, t_)
        return np.array(best[1], np.int32), np.float32(best[2]), np.float32(best[3])
    raise RuntimeError("no base found")


def _eigen_norm(v):
    v = v.astype(np.float32)
    return np.sqrt(np.float32(v[0] * v[0]) + (np.float32(v[1] * v[1]) + np.float32(v[2] * v[2])))


def make_candidates(k, P, Q, cp, cq, seed, stages):
    """SURVEY.md 8(d) cfg2 candidate list (column-major 16 floats each): N_NEAR perturbations of the
    ground truth, then transforms derived from congruent quads of an n=3000 extraction on the same
    clouds (rigid fits that pass the rms gate), padded with random rigid motions.
    `stages(Qsub)` returns an object with extract_pairs / find_quads / rigid_batch for the sub-sampled
    Q (the GPU context in our arm, the CPU oracle in the reference arm: same inputs, bit-identical
    stage outputs, hence the same candidate list in both arms)."""
    from super4pcs_b200 import synth
    rng = np.random.RandomState(seed)
    near = synth.candidate_transforms(N_NEAR, DELTA, seed=seed, n_near=N_NEAR, centroid_p=cp, centroid_q=cq)
    out = [np.ascontiguousarray(near.transpose(0, 2, 1)).reshape(-1, 16)]
    have = N_NEAR
    qsub = Q[rng.choice(len(Q), EXTRACT_N, replace=False)]
    psub = P[rng.choice(len(P), 20000, replace=False)]
    st = stages(psub, qsub, EXTRACT_DELTA)
    diameter = float(np.linalg.norm(psub.max(0) - psub.min(0)))
    target, per_base, tries = int(0.75 * (k - N_NEAR)), 384, 0
    got = 0
    while got < target and tries < 64:
        tries += 1
        ids, inv1, inv2 = select_base(psub, rng, diameter)
        bx = psub[ids]
        b9 = [np.concatenate([bx[i], [0, 0, 0], [-1, -1, -1]]).astype(np.float32) for i in range(4)]
        d1, d2 = _eigen_norm(bx[0] - bx[1]), _eigen_norm(bx[2] - bx[3])
        quads = st.quads_for_base(d1, d2, 2 * EXTRACT_DELTA, b9, inv1, inv2, bx)
        if len(quads) == 0:
            continue
        T, rms, ok = st.rigid_batch(ids, bx, quads)
        gate = np.nonzero(ok & (rms >= 0) & (rms < 2 * EXTRACT_DELTA))[0]
        if len(gate) == 0:
            continue
        take = gate[np.linspace(0, len(gate) - 1, min(per_base, len(gate))).astype(int)]
        out.append(T[take])
        got += len(take)
    have += got
    if have < k:
        rnd = synth.candidate_transforms(k - have, DELTA, seed=seed + 1, n_near=0, centroid_p=cp, centroid_q=cq)
        out.append(np.ascontiguousarray(rnd.transpose(0, 2, 1)).reshape(-1, 16))
    T = np.ascontiguousarray(np.concatenate(out)[:k].astype(np.float32))
    import hashlib
    return T, {"near_gt": N_NEAR, "quad_derived": int(min(got, k - N_NEAR)),
               "random": int(max(0, k - N_NEAR - got)), "bases_tried": tries,
               # both arms must print the same digest: same inputs + bit-identical stages => same list
               "sha1": hashlib.sha1(T.tobytes()).hexdigest()[:16]}


class GpuStages:
    """stage provider for make_candidates backed by libs4g (our arm)"""

    def __init__(self, device):
        self.device = device

    def __call__(self, psub, qsub, delta):
        from super4pcs_b200 import Context
        self.ctx = Context(self.device)
        self.ctx.set_cloud_p(psub, delta)
        self.ctx.set_cloud_q(qsub)
        return self

    def quads_for_base(self, d1, d2, eps, b9, inv1, inv2, bx):
        self.ctx.extract_pairs(d1, 0.0, eps, b9[0], b9[1], slot=0, fetch=False)
        self.ctx.extract_pairs(d2, 0.0, eps, b9[2], b9[3], slot=1, fetch=False)
        return self.ctx.find_quads(inv1, inv2, eps, bx)

    def rigid_batch(self, ids, bx, quads):
        return self.ctx.rigid_batch(bx, quads)


class OracleStages:
    """stage provider backed by the CPU oracle (reference arm only)"""

    def __call__(self, psub, qsub, delta):
        from oracle import port as oport
        self.pt = oport.Port(psub, qsub, delta)
        return self

    def quads_for_base(self, d1, d2, eps, b9, inv1, inv2, bx):
        p1 = self.pt.extract_pairs(d1, 0.0, eps, b9[0], b9[1])
        p2 = self.pt.extract_pairs(d2, 0.0, eps, b9[2], b9[3])
        return self.pt.find_quads(inv1, inv2, eps, bx, p1, p2)

    def rigid_batch(self, ids, bx, quads):
        return self.pt.rigid_batch(ids, quads)


class ClockSampler(threading.Thread):
    """SM clocks / throttle reasons DURING the timed region: NVML polled in-process
    every 5 ms (nvidia-smi takes longer to start than a timed region lasts); falls back to nvidia-smi."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,"
         "clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index):
        super().__init__(daemon=True)
        self.gpu = gpu_index
        self.stop_flag = threading.Event()
        self.sm, self.mx, self.reasons, self.power = [], [], set(), []
        self.source = "nvml"
        try:
            import pynvml
            pynvml.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = gpu_index
            if vis:
                try:
                    phys = int(vis.split(",")[gpu_index])
                except (ValueError, IndexError):
                    phys = gpu_index
            self.nv = pynvml
            self.h = pynvml.nvmlDeviceGetHandleByIndex(phys)
            self.max_sm = float(pynvml.nvmlDeviceGetMaxClockInfo(self.h, pynvml.NVML_CLOCK_SM))
        except Exception:
            self.nv = None
            self.source = "nvidia-smi"

    def _poll_nvml(self):
        nv = self.nv
        self.sm.append(float(nv.nvmlDeviceGetClockInfo(self.h, nv.NVML_CLOCK_SM)))
        self.mx.append(self.max_sm)
        try:
            self.power.append(nv.nvmlDeviceGetPowerUsage(self.h) / 1000.0)
        except Exception:
            pass
        try:
            r = nv.nvmlDeviceGetCurrentClocksThrottleReasons(self.h)
        except Exception:
            r = 0
        for name, bit in (("hw_slowdown", 0x8), ("sw_power_cap", 0x4), ("sw_thermal_slowdown", 0x20),
                          ("hw_thermal_slowdown", 0x40)):
            if r & bit:
                self.reasons.add(name)

    def _poll_smi(self):
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + self.Q, "--format=csv,noheader,nounits",
                              "-i", str(self.gpu)], capture_output=True, text=True, timeout=5).stdout
        for line in out.strip().splitlines():
            r = [c.strip() for c in line.split(",")]
            self.sm.append(float(r[1]))
            self.mx.append(float(r[2]))
            for name, v in zip(["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"], r[5:9]):
                if v.lower().startswith("active"):
                    self.reasons.add(name)

    def run(self):
        while not self.stop_flag.is_set():
            try:
                if self.nv is not None:
                    self._poll_nvml()
                else:
                    self._poll_smi()
            except Exception:
                pass
            self.stop_flag.wait(0.005 if self.nv is not None else 0.2)

    def summary(self):
        return {"sm_mhz": float(np.median(self.sm)) if self.sm else None,
                "sm_max_mhz": max(self.mx) if self.mx else None, "reasons": sorted(self.reasons),
                "samples": len(self.sm), "power_w_max": max(self.power) if self.power else None,
                "source": self.source}


def _ref_matcher(raw):
    """(object with verify_batch(T, best_lcp, nthreads) -> (lcp, seconds), kind, closer)"""
    from oracle import ref as oref
    if oref.available():
        opt = oref.make_options(delta=DELTA, sample_size=10 ** 9, overlap=OVERLAP)
        m = oref.RefMatcher(raw["P"], raw["Q"], opt)      # reference init(): centring, kd-tree
        return m.verify_batch, "reference", m.close
    from oracle import port as oport
    from super4pcs_b200 import synth
    P, _ = synth.center(raw["P"])
    Q, _ = synth.center(raw["Q"])
    pt = oport.Port(P, Q, DELTA)

    def vb(T, best, nthreads=1):
        lcp, _, secs = pt.verify_batch(T, best, nthreads=nthreads)
        return lcp, secs
    return vb, "port", (lambda: None)


def cpu_reference_arm(raw, T_colmajor, per_thread=4, reps=3, threads=None, early_exit=True, one_thread=True):
    """Times the reference's own Verify (match4pcsBase.cc:508-567) on an evenly spaced sample of the candidates.
    Headline: OpenMP over candidates (the reference's own parallelisation of this loop, match4pcsBase.hpp:390-393) on
    every PHYSICAL core, threads bound (OMP_PROC_BIND=close, OMP_PLACES=cores), `per_thread` candidates per thread with
    dynamic scheduling, best of `reps` passes; every candidate runs to the end, like the GPU arm.
    Side figures: `as_shipped_1thread` -- MatchSuper4PCS pins this loop to ONE thread (super4pcs.cc:70-72): a few
    candidates on one thread; `early_exit` -- the same sample with best_LCP preset to the sample's best LCP, so that every
    candidate stops once it cannot beat it (match4pcsBase.cc:558-560), the most favourable state of the reference's loop.
    Returns a dict with value / sample indices / lcp (for the parity check of the GPU counts)."""
    verify_batch, kind, close = _ref_matcher(raw)
    cores = threads or physical_cores()
    sample = min(len(T_colmajor), max(1, cores * per_thread))
    idx = np.unique(np.linspace(0, len(T_colmajor) - 1, sample).astype(int))
    Ts = np.ascontiguousarray(T_colmajor[idx])
    verify_batch(Ts[:max(1, cores)], 0.0, nthreads=cores)          # warm caches / threads
    lcp, best_secs, all_secs = None, None, []
    for _ in range(max(1, reps)):
        lcp, secs = verify_batch(Ts, 0.0, nthreads=cores)
        all_secs.append(secs)
        best_secs = secs if best_secs is None else min(best_secs, secs)
    out = {"value": len(idx) / best_secs, "unit": UNIT, "cores": cores, "kind": kind, "seconds": best_secs,
           "seconds_all": all_secs, "idx": idx, "lcp": np.asarray(lcp, np.float32),
           "sample": ("%d of the %d candidates (evenly spaced over near-GT + quad-derived + random), full %d x %d Verify "
                      "each, no early exit, OpenMP over candidates on %d physical cores (threads bound: OMP_PROC_BIND=%s "
                      "OMP_PLACES=%s; %d hardware threads visible), dynamic schedule, best of %d passes"
                      % (len(idx), len(T_colmajor), len(raw["P"]), len(raw["Q"]), cores, os.environ.get("OMP_PROC_BIND"),
                         os.environ.get("OMP_PLACES"), host_threads(), max(1, reps)))}
    if one_thread:
        k1 = Ts[np.linspace(0, len(Ts) - 1, min(len(Ts), 3)).astype(int)]
        verify_batch(k1[:1], 0.0, nthreads=1)
        _, s1 = verify_batch(k1, 0.0, nthreads=1)
        out["as_shipped_1thread"] = {"value": len(k1) / s1, "unit": UNIT, "cores": 1,
                                     "note": "MatchSuper4PCS runs this loop on one thread (super4pcs.cc:70-72): %d candidates "
                                             "of the sample, one thread" % len(k1)}
    if early_exit:
        try:
            best = float(np.max(lcp))
            _, secs_ee = verify_batch(Ts, best, nthreads=cores)
            out["early_exit"] = {"value": len(idx) / secs_ee, "unit": UNIT, "best_lcp": best,
                                 "note": "same sample, best_LCP preset to the sample's best LCP: every candidate stops "
                                         "once it cannot beat it"}
        except Exception:
            out["early_exit"] = None
    close()
    return out


def cpu_public(d):
    """the JSON-able part of cpu_reference_arm()'s result"""
    return {k: v for k, v in d.items() if k not in ("idx", "lcp", "seconds_all", "seconds")}


def run_reference(args):
    """--impl reference: the reference's own Verify on this box's host cores.  Headline `value` = the reference AS IT RUNS
    INSIDE ITS OWN LOOP, i.e. with its early exit against the best LCP seen (match4pcsBase.cc:558-560; best_LCP preset to the
    best LCP of the sample = the most favourable state of that loop; round-1 ADVICE: do not quote the speed-up against a
    reference whose early exit is disabled); `cpu_baseline.no_early_exit` = every candidate verified to the end, the work the
    GPU arm does."""
    rank = _env_int("RANK", 0)
    if rank != 0:
        return 0
    raw, P, Q, cp, cq = build_workload(args.points)
    K = args.candidates if args.scaling == "weak" else args.strong_candidates
    T, mix = make_candidates(K, P, Q, cp, cq, 7, OracleStages())
    verify_batch, kind, close = _ref_matcher(raw)
    cores = physical_cores()
    n = min(len(T), max(1, cores * args.ref_per_thread))
    idx = np.unique(np.linspace(0, len(T) - 1, n).astype(int))
    Ts = np.ascontiguousarray(T[idx])
    lcp, secs_full = verify_batch(Ts, 0.0, nthreads=cores)          # untimed pass 0: warms caches / threads, gives the best LCP
    best = float(np.max(lcp))
    times = []
    for it in range(args.warmup + args.steps):
        _, secs = verify_batch(Ts, best, nthreads=cores)
        if it >= args.warmup:
            times.append(secs)
    _, secs_full = verify_batch(Ts, 0.0, nthreads=cores)             # the same sample without early exit (side figure)
    k1 = Ts[np.linspace(0, len(Ts) - 1, min(len(Ts), 3)).astype(int)]
    _, s1 = verify_batch(k1, 0.0, nthreads=1)
    close()
    value = len(idx) * len(times) / sum(times)
    cpu = {"value": value, "unit": UNIT, "cores": cores, "kind": kind,
           "sample": ("%d of the %d candidates (evenly spaced over near-GT + quad-derived + random) per step, %d x %d Verify "
                      "each WITH the reference's early exit (best_LCP preset to the sample's best LCP %.4f), OpenMP over "
                      "candidates on %d physical cores (threads bound: OMP_PROC_BIND=%s OMP_PLACES=%s; %d hardware threads "
                      "visible), dynamic schedule" % (len(idx), len(T), len(raw["P"]), len(raw["Q"]), best, cores,
                                                     os.environ.get("OMP_PROC_BIND"), os.environ.get("OMP_PLACES"), host_threads())),
           "no_early_exit": {"value": len(idx) / secs_full, "unit": UNIT, "note": "same sample, every candidate verified to the end"},
           "as_shipped_1thread": {"value": len(k1) / s1, "unit": UNIT, "cores": 1,
                                  "note": "MatchSuper4PCS runs this loop on one thread (super4pcs.cc:70-72): %d candidates, no early exit" % len(k1)}}
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * sum(times) / len(times),
        "higher_is_better": True, "scaling": args.scaling, "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": dict(workload_config(args, max(1, args.gpus)), candidate_mix=mix),
        "cpu_baseline": cpu,
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    emit(line)
    return 0


def workload_config(args, world):
    strong = args.scaling == "strong"
    per_gpu = args.candidates if not strong else (args.strong_candidates + world - 1) // world
    total = args.candidates * world if not strong else args.strong_candidates
    return {"workload": "cfg2: synthetic bumpy-sphere pair, %d pts each, 30%% overlap, delta=%.4g, "
                        "|sampled_P|=|sampled_Q|=%d, %s "
                        "(%d near-GT, then rigid fits of congruent quads from an n=3000 extraction, random padding), "
                        "Verify without early exit"
                        % (args.points, DELTA, args.points,
                           ("%d candidate transforms per GPU per step" % args.candidates) if not strong else
                           ("ONE list of %d candidate transforms per step, sharded index %% n_gpus" % args.strong_candidates),
                           N_NEAR),
            "n_points": args.points, "delta": DELTA, "overlap": OVERLAP,
            "candidates_per_gpu_per_step": per_gpu, "global_candidates_per_step": total,
            "sharding": "candidate sets sharded across GPUs, clouds+grid replicated, 1 allreduce(MAX) of the "
                        "packed (count,index) key per step",
            "l2": "flushed between timed steps (256 MiB write)"}


def device_info(dev, local):
    """what the numbers were measured on: name, SM count, power limit (NVML, when it can be read)"""
    import torch
    p = torch.cuda.get_device_properties(dev)
    out = {"name": p.name, "sm_count": p.multi_processor_count, "memory_gb": round(p.total_memory / 1e9, 1),
           "power_limit_w": None}
    try:
        import pynvml
        pynvml.nvmlInit()
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        phys = int(vis.split(",")[local]) if vis else local
        out["power_limit_w"] = pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(phys)) / 1000.0
    except Exception:
        pass
    return out


def dump_outputs(out_dir, counts, key):
    """the arrays the resident call (s4g_verify_best_dev) hands its caller in the last timed step: the inlier count of
    every candidate and the winner's packed key, decoded into (count, candidate index); float64 holds both exactly"""
    os.makedirs(out_dir, exist_ok=True)
    np.save(os.path.join(out_dir, "counts.npy"), np.asarray(counts, np.float64))
    np.save(os.path.join(out_dir, "winner.npy"), np.array([key >> 32, 0xFFFFFFFF - (key & 0xFFFFFFFF)], np.float64))


def run_ours(args):
    import torch
    import torch.distributed as dist
    from super4pcs_b200 import Context

    world = _env_int("WORLD_SIZE", 1)
    rank = _env_int("RANK", 0)
    local = _env_int("LOCAL_RANK", 0)
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device (the product has no CPU path; use --impl reference for the CPU arm)")
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)    # NCCL_DEBUG: see the top of this file

    strong = args.scaling == "strong"
    raw, P, Q, cp, cq = build_workload(args.points)
    gs = GpuStages(local)
    if strong:
        # ONE candidate list for the whole job (same seed on every rank); rank r verifies the candidates index % world == r
        T_all, mix = make_candidates(args.strong_candidates, P, Q, cp, cq, 7, gs)
        my_idx = np.arange(rank, len(T_all), world)
        T_host = np.ascontiguousarray(T_all[my_idx])
    else:
        T_all = None
        T_host, mix = make_candidates(args.candidates, P, Q, cp, cq, 7 + 1000 * rank, gs)
        my_idx = np.arange(len(T_host))
    gs.ctx.close()
    K = len(T_host)

    ctx = Context(local)
    # ONE explicit stream for libs4g's launches, torch's glue ops, the timing events and (through torch's stream
    # synchronisation) NCCL.  (Round-1 bug, found in round 2: torch's DEFAULT stream has the handle 0, which s4g_set_stream
    # reads as "use the context's own non-blocking stream" -- the key reduction then was not ordered after k_verify and the
    # step time was bracketed on another stream than the kernel's; the numbers came out right only because a 250K-CTA
    # kernel leaves no SM free for anything else until it is almost over.)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.set_stream(stream)
    assert stream.cuda_stream != 0
    ctx.set_stream(stream.cuda_stream)
    t0 = time.time()
    ctx.set_cloud_p(P, DELTA)
    ctx.set_cloud_q(Q)
    setup_s = time.time() - t0
    gstats = ctx.grid_stats()

    # The one collective of the path (max of the packed key over the ranks) runs INSIDE libs4g, on the stream of k_verify:
    # rank 0 draws an NCCL id through the library, torch.distributed only ships those 128 bytes (plumbing), every rank
    # attaches its context (s4g_comm_init_rank).  --collective torch keeps round 1's torch glue ops + dist.all_reduce for A/B.
    native = args.collective == "native"
    if native and world > 1:
        from super4pcs_b200 import s4g as _s4g
        idt = torch.zeros(_s4g.COMM_ID_BYTES, dtype=torch.uint8, device=dev)
        if rank == 0:
            idt.copy_(torch.frombuffer(bytearray(_s4g.comm_unique_id()), dtype=torch.uint8))
        dist.broadcast(idt, src=0)
        ctx.comm_init_rank(idt.cpu().numpy().tobytes(), world, rank)
    comm_info = ctx.comm_info()

    d_T = torch.from_numpy(T_host).to(dev)
    d_counts = torch.zeros(K, dtype=torch.int32, device=dev)
    idx_desc = (0xFFFFFFFF - torch.from_numpy(my_idx.astype(np.int64)).to(dev))   # global candidate index in the key
    my_idx32 = np.ascontiguousarray(my_idx.astype(np.uint32))
    d_idx32 = torch.from_numpy(my_idx32.view(np.int32)).to(dev)
    d_key = torch.zeros(1, dtype=torch.int64, device=dev)
    flush = torch.empty(L2_FLUSH_BYTES // 4, dtype=torch.float32, device=dev)
    T_pinned = torch.from_numpy(T_host).pin_memory()
    T_pinned_np = T_pinned.numpy()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def step_resident():
        if native:                                 # k_pack_T12, k_verify, k_argmax_n, ncclAllReduce: one stream-ordered chain
            ctx.verify_best_dev(d_T.data_ptr(), K, d_idx32.data_ptr(), d_counts.data_ptr(), d_key.data_ptr())
            return d_key
        ctx.verify_dev(d_T.data_ptr(), K, d_counts.data_ptr())
        key = ((d_counts.to(torch.int64) & 0xFFFFFFFF) << 32 | idx_desc).max().reshape(1)
        if world > 1:
            dist.all_reduce(key, op=dist.ReduceOp.MAX)
        return key

    def step_e2e():
        if native:                                 # H2D transforms + indices, kernels, allreduce, D2H counts + key, sync
            return ctx.verify_best(T_pinned_np, my_idx32)[1]
        counts = ctx.verify(T_pinned_np)          # H2D transforms, kernels, D2H counts, sync
        k = int(np.argmax(counts))                 # first maximum = smallest index among ties
        key = (int(counts[k]) << 32) | (0xFFFFFFFF - int(my_idx[k]))
        if world > 1:
            kt = torch.tensor([key], dtype=torch.int64, device=dev)
            dist.all_reduce(kt, op=dist.ReduceOp.MAX)
            key = int(kt.item())
        return key

    def timed(step_fn, steps, warmup, sampler=None):
        for _ in range(warmup):
            step_fn()
        barrier()
        if sampler:
            sampler.start()
        total_ms, kernel_ms = 0.0, 0.0
        l0 = ctx.timings()["launches"]
        for _ in range(steps):
            flush.fill_(1.0)                       # evict L2 between timed steps (untimed)
            barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            last_key = step_fn()
            e1.record(stream)
            barrier()
            total_ms += e0.elapsed_time(e1)
            kernel_ms += ctx.timings()["verify_ms"]   # this step's k_verify (events recorded inside libs4g on this stream)
        if sampler:
            sampler.stop_flag.set()
            sampler.join(timeout=5)
        launches = ctx.timings()["launches"] - l0
        t = torch.tensor([total_ms], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item()), launches, kernel_ms / steps, last_key

    sampler = ClockSampler(local) if rank == 0 else None
    ms_res, launches, kernel_ms, key_res = timed(step_resident, args.steps, args.warmup, sampler)
    ms_e2e, _, _, key_e2e = timed(step_e2e, args.steps, max(1, args.warmup // 2))
    n_global = world * K if not strong else args.strong_candidates
    value = n_global * args.steps / (ms_res * 1e-3)
    e2e = n_global * args.steps / (ms_e2e * 1e-3)
    counts_host = d_counts.cpu().numpy().astype(np.int64)       # last resident step's counts of this rank
    key_res = int(key_res.item())
    if key_res != int(key_e2e):
        raise SystemExit("bench.py: the resident and the host-buffer step disagree on the winner key (%x vs %x)"
                         % (key_res, int(key_e2e)))

    line = None
    if rank == 0:
        # roofline of the Verify kernel: algorithmic bytes from the look-ups this grid really performs
        sub = np.linspace(0, K - 1, 64).astype(int)
        ps = ctx.verify_probe_stats(T_host[sub])
        nq = args.points
        npair = float(len(sub) * nq)
        c_bar = ps["ranges_read"] / npair
        k_bar = ps["points_tested"] / npair
        r_bar = ps["brick_entries_read"] / npair
        b_bar = ps["bitmap_words_read"] / npair
        # SURVEY.md 8(d): N_Q (16 + 8 C + 16 k) per candidate, with the lookups this hierarchy really performs: 4-byte
        # words of the delta-field / v-brick table / occupancy map, 4-byte brick-table entries, 8-byte (start,end) ranges
        bytes_per_cand = nq * (16.0 + 4.0 * b_bar + 4.0 * r_bar + 8.0 * c_bar + 16.0 * k_bar)
        peaks = {}
        try:
            peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        except Exception:
            pass
        peak = float(peaks.get("hbm_gbs", H100_HBM_GBS))
        achieved = K * bytes_per_cand / (kernel_ms * 1e-3) / 1e9
        roofline = {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                    "kernel": "k_verify", "kernel_ms": kernel_ms,
                    "kernel_ms_source": "mean over the timed resident steps (CUDA events inside libs4g, launching stream)",
                    "peak_source": "MEASURED_PEAKS.json hbm_gbs (measured)" if peaks else
                                   "H100 SXM data sheet, 3.35 TB/s (not a measured peak)",
                    "algorithmic_bytes_per_candidate": bytes_per_cand,
                    "cell_ranges_per_query": c_bar, "points_tested_per_query": k_bar,
                    "brick_entries_per_query": r_bar, "field_words_per_query": b_bar,
                    "tile_candidate_pairs_culled_frac": ps["tile_pairs_culled"] / (len(sub) * ((nq + 31) // 32)),   # cull unit = the 32 queries of one warp
                    "survey_literal_bytes_per_candidate": nq * (16.0 + 8.0 * 8 + 16.0 * k_bar)}
        cpu, parity = None, None
        if not args.no_cpu_baseline and world == 1:      # reported on rank 0 at N=1 only
            r = cpu_reference_arm(raw, T_host, per_thread=args.ref_per_thread_inrun, reps=3)
            cpu = cpu_public(r)
            # parity on the timed workload: the reference's Verify of the sampled candidates at full 1M x 1M against the
            # counts the timed kernel produced (LCP = float(count) / float(N), match4pcsBase.cc:566)
            mine = (counts_host[r["idx"]].astype(np.float32) / np.float32(nq)).astype(np.float32)
            bad = int(np.count_nonzero(mine != r["lcp"]))
            parity = {"parity_checked": int(len(r["idx"])), "mismatches": bad,
                      "against": "%s Verify, full %d x %d, same candidates" % (r["kind"], nq, nq)}
            if bad:
                k = int(np.flatnonzero(mine != r["lcp"])[0])
                raise SystemExit("bench.py: PARITY FAILURE -- %d of %d sampled candidates differ from the reference "
                                 "(first: candidate %d, ours %r, reference %r)" % (bad, len(r["idx"]), int(r["idx"][k]),
                                                                                  float(mine[k]), float(r["lcp"][k])))
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms_res / args.steps, "higher_is_better": True,
            "scaling": args.scaling, "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": dict(workload_config(args, world), candidate_mix=mix),
            "e2e": {"value": e2e, "unit": UNIT, "h2d_bytes_per_step": int(K * 64 + (K * 4 if native else 0)),
                    "d2h_bytes_per_step": int(K * 4 + (8 if native else 0)), "ms_per_step": ms_e2e / args.steps},
            "gpu_launches": int(launches),
            "collective": ({"where": "inside libs4g on the stream of k_verify: ncclAllReduce(ncclMax, uint64) of the packed key "
                                     "(s4g_verify_best*, csrc/comm.cu); torch.distributed only ships the 128-byte NCCL id",
                            "comm_ranks": comm_info["ranks"], "nccl_version": comm_info["nccl_version"],
                            "enqueued_by_rank0": ctx.comm_info()["collectives"] - comm_info["collectives"]}
                           if native else {"where": "torch glue ops + torch.distributed.all_reduce(MAX) (--collective torch)"}),
            "roofline": roofline, "cpu_baseline": cpu,
            "clocks": sampler.summary() if sampler else None,
            "device": device_info(dev, local),
            "grid": gstats, "setup_seconds": setup_s,
            "winner_key": "%016x" % key_res,
        }
        if parity:
            line.update(parity)
        if args.dump_outputs:
            dump_outputs(args.dump_outputs, counts_host, key_res)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    ctx.close()
    if line is not None:
        emit(line)
    return 0


_REAL_STDOUT = None


def isolate_stdout():
    """Everything any library prints on fd 1 (e.g. NCCL's version banner) goes to stderr; the ONE
    JSON line of the contract is written to the original stdout by emit()."""
    global _REAL_STDOUT
    if _REAL_STDOUT is None:
        sys.stdout.flush()
        _REAL_STDOUT = os.fdopen(os.dup(1), "w")
        os.dup2(2, 1)


def emit(line):
    out = _REAL_STDOUT if _REAL_STDOUT is not None else sys.stdout
    out.write(json.dumps(line) + "\n")
    out.flush()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--points", type=int, default=N_POINTS, help="debug only; the metric is quoted at 1M")
    ap.add_argument("--candidates", type=int, default=CANDIDATES_PER_GPU)
    ap.add_argument("--scaling", default="weak", choices=["weak", "strong"],
                    help="weak: --candidates per GPU per step; strong: ONE list of --strong-candidates sharded index %% world")
    ap.add_argument("--strong-candidates", type=int, default=32768)
    ap.add_argument("--collective", default="native", choices=["native", "torch"],
                    help="native: key argmax + ncclAllReduce inside libs4g (s4g_verify_best*); torch: round 1's torch ops + dist.all_reduce")
    ap.add_argument("--ref-per-thread", type=int, default=2, help="--impl reference: candidates per physical core per step")
    ap.add_argument("--ref-per-thread-inrun", type=int, default=4, help="in-run cpu_baseline: candidates per physical core (best of 3)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write what the last timed step computed as DIR/<name>.npy (float64)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    isolate_stdout()
    if args.warmup < 3 and args.impl == "ours":
        args.warmup = 3
    if args.impl == "reference":
        return run_reference(args)
    return run_ours(args)


if __name__ == "__main__":
    sys.exit(main())
