"""TEST INFRASTRUCTURE, not collected by pytest; needs an H100: time-boxed fuzz of every device stage through the C ABI against the oracle port -- pairs with random filters,
quads, rigid fits, Verify counts, TryCongruentSet winners -- over random clouds / deltas / bases, including tiny and
degenerate clouds.  The CPU-side twin (port vs compiled reference) is tests/fuzz_port_vs_reference.py.
  python tests/fuzz_gpu_vs_port.py [seed] [seconds]"""
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import port as oport  # noqa: E402
from super4pcs_b200 import Context, PairFilters, synth  # noqa: E402

bits = lambda a: np.ascontiguousarray(a, np.float32).view(np.uint32)  # noqa: E731
rng = np.random.RandomState(int(sys.argv[1]) if len(sys.argv) > 1 else 0)
budget = float(sys.argv[2]) if len(sys.argv) > 2 else 120
t0, n_cfg, bad = time.time(), 0, 0


def report(what, **kw):
    global bad
    bad += 1
    print("DIFF", what, kw, flush=True)


with Context(0) as ctx:
    while time.time() - t0 < budget:
        n = int(rng.choice([rng.randint(5, 60), rng.randint(60, 3000), rng.randint(3000, 20000)]))
        normals = bool(rng.randint(0, 2))
        delta = float(rng.choice([0.003, 0.01, 0.03, 0.08]))
        seed = int(rng.randint(1, 10 ** 6))
        d = synth.make_pair(n, float(rng.choice([0.3, 0.6, 0.9])), seed=seed, with_normals=normals,
                            noise_sigma=float(rng.choice([0, 0.003])), outlier_frac=float(rng.choice([0, 0.15])))
        P, _ = synth.center(d["P"])
        Q, _ = synth.center(d["Q"])
        if rng.randint(0, 8) == 0:
            Q[::3] = Q[0]                                    # duplicates
        if rng.randint(0, 8) == 0:
            P[:, 2] = 0                                      # planar P
        Qn = None
        if normals:
            Qn = (d["Qn"] / np.linalg.norm(d["Qn"], axis=1, keepdims=True)).astype(np.float32)
        rgb = rng.uniform(0, 255, Q.shape).astype(np.float32) if rng.randint(0, 4) == 0 else None
        ctx.set_cloud_p(P, delta)
        ctx.set_cloud_q(Q, normals=Qn, rgb=rgb)
        pt = oport.Port(P, Q, delta, Qn=Qn, Qrgb=rgb)
        filt = (float(rng.choice([-1, 20.0, 60.0])) if normals else -1.0, float(rng.choice([-1, -1, 1.5])),
                float(rng.choice([-1, -1, 70.0])), float(rng.choice([-1, 150.0])) if rgb is not None else -1.0)
        tag = dict(n=n, delta=delta, seed=seed, filt=filt)
        for _ in range(3):
            ids = rng.randint(0, len(P), 4)
            bx = P[ids]
            bn = rng.standard_normal((4, 3)).astype(np.float32)
            bn /= np.linalg.norm(bn, axis=1, keepdims=True)
            brgb = rng.uniform(0, 255, (4, 3)).astype(np.float32)
            b9 = lambda i: np.concatenate([bx[i], bn[i], brgb[i]]).astype(np.float32)  # noqa: E731
            d1, d2 = float(np.linalg.norm(bx[0] - bx[1])), float(np.linalg.norm(bx[2] - bx[3]))
            a1, a2 = float(np.linalg.norm(bn[0] - bn[1])), float(np.linalg.norm(bn[2] - bn[3]))
            eps = 2 * delta
            if not (d1 > 0 and d2 > 0):
                continue
            p1 = ctx.extract_pairs(d1, a1, eps, b9(0), b9(1), PairFilters(*filt), slot=0)
            p2 = ctx.extract_pairs(d2, a2, eps, b9(2), b9(3), PairFilters(*filt), slot=1)
            if len(Q) <= 6000:                               # the port's pair sweep is brute force
                w1, w2 = pt.extract_pairs(d1, a1, eps, b9(0), b9(1), filt), pt.extract_pairs(d2, a2, eps, b9(2), b9(3), filt)
                if not (np.array_equal(p1, w1) and np.array_equal(p2, w2)):
                    report("pairs", **tag)
                    continue
            if len(p1) == 0 or len(p2) == 0 or len(p1) * len(p2) > 2e8:
                continue
            inv1, inv2 = float(rng.uniform(0, 1)), float(rng.uniform(0, 1))
            q = ctx.find_quads(inv1, inv2, eps, bx)
            if len(p1) * len(p2) <= 4e7:
                wq = pt.find_quads(inv1, inv2, eps, bx, p1, p2)
                if not np.array_equal(q, wq):
                    report("quads", got=len(q), want=len(wq), **tag)
                    continue
            if len(q) == 0:
                continue
            qs = q[:3000]
            T, rms, ok = ctx.rigid_batch(bx, qs, max_angle_deg=filt[2])
            Tp, rp, okp = pt.rigid_batch(ids, qs, max_angle_deg=filt[2])
            sel = okp & (rp < 1e8)
            if filt[2] < 0 and not (np.array_equal(ok, okp) and np.array_equal(bits(rms[sel]), bits(rp[sel])) and
                                    np.array_equal(bits(T[sel]), bits(Tp[sel]))):
                report("rigid", **tag)                        # (max_angle >= 0: device atan2f is within 2 ulp, not bit-exact)
                continue
            gate = okp & (rp >= 0) & (rp < eps)
            if gate.any():
                Tg = Tp[gate][:64]
                c = ctx.verify(Tg)
                _, good, _ = pt.verify_batch(Tg, 0.0, nthreads=oport.num_threads())
                if not np.array_equal(c, good):
                    report("verify", **tag)
                    continue
            if filt[2] < 0:
                r = ctx.try_congruent_set(bx, qs, eps)
                _, g_all, _ = pt.verify_batch(Tp[gate], 0.0, nthreads=oport.num_threads()) if gate.any() else (None, np.zeros(0, np.uint32), None)
                want_gate = int(gate.sum())
                want_best = int(g_all.max()) if want_gate else 0
                want_idx = int(np.nonzero(gate)[0][int(np.argmax(g_all))]) if want_gate else -1
                if not (r["n_gate_pass"] == want_gate and r["best_count"] == want_best and r["best_index"] == want_idx):
                    report("tcs", got=(r["n_gate_pass"], r["best_count"], r["best_index"]), want=(want_gate, want_best, want_idx), **tag)
        n_cfg += 1
print("configs", n_cfg, "bad", bad, "secs", round(time.time() - t0, 1))
