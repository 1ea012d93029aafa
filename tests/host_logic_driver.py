"""Subprocess body of tests/test_host_logic_cpu.py and tests/test_zz_lanes_gpu.py: drives the header-compatible C++
layer through the drop-in harness (oracle/_dropin/libb200_harness.so) and prints one JSON line.  Run with
LD_PRELOAD=tests/_build/libs4g_oracle_shim.so it exercises the HOST logic on the CPU oracle; run without, the real
CUDA library.  S4PCS_LANES / S4PCS_FUSED are read by the C++ layer from the environment."""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import _build, ref as oref  # noqa: E402


def _h(a):
    return hashlib.sha1(np.ascontiguousarray(a).tobytes()).hexdigest()[:16]


def run(which, libpath):
    gold = os.path.join(ROOT, "tests", "golden")
    out = {}
    if which == "hippo":
        h = np.load(os.path.join(gold, "hippo.npz"))
        opt = oref.make_options(delta=0.01, overlap=0.7, sample_size=200, max_time_seconds=1000)
        score, T, Qt = oref.compute_transformation(h["P"], h["Q"], opt, libpath=libpath)
        out = dict(score=float(np.float32(score)), T=[int(x) for x in T.view(np.uint32)], Q=_h(Qt))
    elif which == "trace":
        h = np.load(os.path.join(gold, "hippo.npz"))
        opt = oref.make_options(delta=0.01, overlap=0.7, sample_size=200, max_time_seconds=1000, random_seed=77)
        score, T, tr = oref.compute_transformation_traced(h["P"], h["Q"], opt, libpath=libpath)
        out = dict(score=float(np.float32(score)), T=[int(x) for x in T.view(np.uint32)], n=len(tr), trace=_h(tr))
    elif which == "steps":
        # stepwise use (Meshlab pattern) + early termination in the middle of a speculative batch, then the RNG /
        # base state is probed by selecting the next base by hand
        h = np.load(os.path.join(gold, "hippo.npz"))
        opt = oref.make_options(delta=0.01, sample_size=200, overlap=0.5, terminate_threshold=0.55, random_seed=3,
                                max_time_seconds=1000)
        m = oref.RefMatcher(h["P"], h["Q"], opt, identity_sampler=False, libpath=libpath)
        log = []
        for n in (1, 3, 2, 7, 40, 100):
            r = m.perform_n_steps(n)
            ok, i1, i2, ids = m.select_quadrilateral()
            bx, _, _ = m.base3d()
            log.append([r["ret"], float(np.float32(r["best_lcp"])), r["n_progress"], _h(r["T"]), bool(ok),
                        float(np.float32(i1)), float(np.float32(i2)), [int(x) for x in ids], _h(bx)])
        out = dict(log=log)
        m.close()
    elif which == "prealigned":
        # the initial LCP (identity alignment) already exceeds the terminate threshold: the reference keeps drawing bases until
        # one reaches TryCongruentSet (a base without pairs or without congruent quads returns false, hpp:335-347) -- return
        # values, progress reports and the RNG state (probed by selecting the next base by hand) must follow it
        h = np.load(os.path.join(gold, "hippo.npz"))
        opt = oref.make_options(delta=0.004, sample_size=60, overlap=0.5, terminate_threshold=0.04, random_seed=11,
                                max_time_seconds=1000)
        m = oref.RefMatcher(h["P"], h["P"].copy(), opt, identity_sampler=False, libpath=libpath)
        log = [float(np.float32(m.init_state()["best_lcp"]))]
        for n in (1, 1, 1, 2, 3, 5, 40, 200):
            r = m.perform_n_steps(n)
            ok, i1, i2, ids = m.select_quadrilateral()
            log.append([r["ret"], float(np.float32(r["best_lcp"])), r["n_progress"], r["n_candidates"], bool(ok),
                        [int(x) for x in ids]])
        out = dict(log=log)
        m.close()
    elif which == "patches":
        # a sampled Q of 3500 points = 4 of Verify's 1024-query super-tiles (S4G_VERIFY_PATCHES > 1 splits them into
        # patches; s4g_try_bases is on by default at this size): 9 bases in four stepwise calls, a few seconds on the CPU
        # (the whole run would try 72 bases, some with 80K candidates)
        from super4pcs_b200 import synth
        d = synth.make_pair(12000, 0.8, seed=4)
        opt = oref.make_options(delta=0.007, overlap=0.8, sample_size=3500, random_seed=21, max_time_seconds=10000)
        m = oref.RefMatcher(d["P"], d["Q"], opt, identity_sampler=False, libpath=libpath)
        log = [m.nQ, _h(m.sampled_q()[0])]
        for n in (2, 2, 3, 2):
            r = m.perform_n_steps(n)
            log.append([r["ret"], float(np.float32(r["best_lcp"])), r["n_progress"], [int(x) for x in r["T"].view(np.uint32)]])
        out = dict(log=log)
        m.close()
    elif which.startswith("synth"):
        # whole pipeline on a synthetic pair: voxel sampler, shuffle + truncation, RNG-driven bases, filters
        from super4pcs_b200 import synth
        seed, normals = int(which[5]), which.endswith("n")
        d = synth.make_pair(30000, 0.6, seed=seed, with_normals=normals)
        kw = dict(delta=0.02, overlap=0.6, sample_size=300, max_time_seconds=10000, random_seed=100 + seed)
        if normals:
            kw["max_normal_difference"] = 40.0
        score, T, Qt = oref.compute_transformation(d["P"], d["Q"], oref.make_options(**kw), Pn=d["Pn"], Qn=d["Qn"],
                                                   libpath=libpath)
        out = dict(score=float(np.float32(score)), T=[int(x) for x in T.view(np.uint32)], Q=_h(Qt))
    elif which == "whole":
        # sample_size larger than the clouds (both used whole), then the demo's literal defaults (LCP 1 at identity),
        # then an empty cloud (kLargeNumber sentinel)
        from super4pcs_b200 import synth
        d = synth.make_pair(400, 0.9, seed=5)
        opt = oref.make_options(delta=0.02, overlap=0.9, sample_size=10 ** 6, max_time_seconds=10000, random_seed=7)
        s1, T1, Q1 = oref.compute_transformation(d["P"], d["Q"], opt, libpath=libpath)
        h = np.load(os.path.join(gold, "hippo.npz"))
        opt = oref.make_options(delta=5.0, overlap=0.2, sample_size=200, max_time_seconds=10)
        s2, T2, _ = oref.compute_transformation(h["P"], h["Q"], opt, libpath=libpath)
        s3, _, _ = oref.compute_transformation(np.zeros((0, 3), np.float32), np.zeros((5, 3), np.float32), opt, libpath=libpath)
        out = dict(s1=float(np.float32(s1)), T1=_h(T1), Q1=_h(Q1), s2=float(s2), T2=_h(T2), s3=float(s3))
    elif which == "trials":
        # init(): sampler, centring, diameter estimate, number of trials, initial LCP over a sweep of overlaps
        from super4pcs_b200 import synth
        d = synth.make_pair(1500, 0.5, seed=3)
        rows = []
        for ov in (0.1, 0.2, 0.35, 0.5, 0.62, 0.75, 0.9, 1.0):
            opt = oref.make_options(delta=0.03, overlap=ov, sample_size=400, random_seed=99)
            m = oref.RefMatcher(d["P"], d["Q"], opt, identity_sampler=False, libpath=libpath)
            st = m.init_state()
            rows.append([st["number_of_trials"], float(np.float32(st["best_lcp"])), float(np.float32(st["diameter"])), m.nP, m.nQ,
                         _h(m.sampled_q()[0]), _h(m.sampled_p()[0]), _h(st["centroid_p"]), _h(st["centroid_q"])])
            m.close()
        out = dict(rows=rows)
    elif which.startswith("sweep"):
        # randomised whole-pipeline sweep: small clouds, random delta / overlap / sample size / seed / filters
        from super4pcs_b200 import synth
        rng = np.random.RandomState(int(which[5:]))
        rows = []
        for _ in range(6):
            n = int(rng.randint(250, 900))
            ov = float(rng.choice([0.3, 0.5, 0.7, 0.9]))
            normals = bool(rng.randint(0, 2))
            d = synth.make_pair(n, ov, seed=int(rng.randint(1, 10 ** 6)), with_normals=normals,
                                noise_sigma=float(rng.choice([0.0, 0.002])), outlier_frac=float(rng.choice([0.0, 0.1])))
            kw = dict(delta=float(rng.choice([0.02, 0.04, 0.07])), overlap=ov, sample_size=int(rng.choice([60, 150, 10 ** 6])),
                      max_time_seconds=10000, random_seed=int(rng.randint(0, 2 ** 31 - 1)),
                      terminate_threshold=float(rng.choice([1.0, 1.0, max(ov, 0.8)])))
            if normals and rng.randint(0, 2):
                kw["max_normal_difference"] = float(rng.choice([20.0, 45.0]))
            if rng.randint(0, 3) == 0:
                kw["max_translation_distance"] = 3.0
            score, T, Qt = oref.compute_transformation(d["P"], d["Q"], oref.make_options(**kw), Pn=d["Pn"], Qn=d["Qn"],
                                                       libpath=libpath)
            rows.append([float(np.float32(score)), _h(T), _h(Qt)])
        out = dict(rows=rows)
    elif which == "ties":
        # four inputs (found by tests/fuzz_pipeline_vs_reference.py) where two candidates with DIFFERENT transforms tie for the
        # final best inlier count: the winner then depends on the candidate order (DESIGN.md section 4)
        g = np.load(os.path.join(gold, "tie_cases.npz"), allow_pickle=True)
        rows = []
        for k in (1, 2, 3, 4):
            kw = eval(str(g["c%d_kw" % k]))
            Pn = g["c%d_Pn" % k] if ("c%d_Pn" % k) in g else None
            Qn = g["c%d_Qn" % k] if ("c%d_Qn" % k) in g else None
            score, T, _ = oref.compute_transformation(g["c%d_P" % k], g["c%d_Q" % k], oref.make_options(**kw), Pn=Pn, Qn=Qn,
                                                      libpath=libpath)
            rows.append([bool(np.float32(score) == g["c%d_score" % k]),
                         bool(np.array_equal(T.view(np.uint32), g["c%d_T" % k].view(np.uint32)))])
        out = dict(rows=rows)
    elif which == "bigpairs":
        # a base whose one diagonal's pair band covers every pair of a line of 8200 points (67,231,800 >= 2^26 ordered
        # pairs) and whose other diagonal's band holds none: the batched pass must refuse it and the per-base chain take it
        Q = np.zeros((8200, 3), np.float32)
        Q[:, 0] = np.linspace(-0.49, 0.49, 8200, dtype=np.float32)
        P = np.array([[-0.25, 0, 0], [0.25, 0, 0], [0, 0.75, 0], [0, -0.75, 0]], np.float32)   # diagonals 0.5 and 1.5
        opt = oref.make_options(delta=0.25, overlap=1.0, sample_size=10 ** 6, max_time_seconds=10000, random_seed=5)
        score, T, Qt = oref.compute_transformation(P, Q, opt, libpath=libpath)
        out = dict(score=float(np.float32(score)), T=[int(x) for x in T.view(np.uint32)], Q=_h(Qt))
    elif which == "pairtest":
        # the reference's own ExtractPairs test (tests/pair_extraction.cc:239-314) through MatchSuper4PCS::ExtractPairs
        from tests.test_oracle_golden import _bruteforce_pairs, _sphere_cloud
        P, Q = _sphere_cloud(200, 1), _sphere_cloud(150, 101)
        m = oref.RefMatcher(P, Q, oref.make_options(delta=0.1, overlap=0.5, sample_size=10 ** 8), libpath=libpath)
        out = dict(equal=[bool(np.array_equal(m.extract_pairs(d, a, 0.2, 0, 1), _bruteforce_pairs(Q, d, 0.2)))
                          for d, a in ((0.3, 0.6), (0.5, 0.4))])
        m.close()
    else:
        raise SystemExit("unknown scenario " + which)
    return out


if __name__ == "__main__":
    which, target = sys.argv[1], sys.argv[2]
    libpath = _build.DROPIN_SO if target == "dropin" else None     # None = the compiled reference
    print("RESULT " + json.dumps(run(which, libpath)))
