"""CPU test of bench.py's workload builders (base selection, candidate list through the oracle stages)
so that the benchmark code paths stay importable and sane without a GPU."""
import numpy as np

import bench


def test_candidate_list_from_oracle_stages():
    raw, P, Q, cp, cq = bench.build_workload(20000)
    T, mix = bench.make_candidates(128, P, Q, cp, cq, 7, bench.OracleStages())
    assert T.shape == (128, 16) and T.dtype == np.float32
    assert mix["near_gt"] == bench.N_NEAR and mix["near_gt"] + mix["quad_derived"] + mix["random"] == 128
    M = T.reshape(-1, 4, 4).transpose(0, 2, 1)
    R = M[:, :3, :3].astype(np.float64)
    assert np.abs(np.einsum("kij,klj->kil", R, R) - np.eye(3)).max() < 1e-4     # rigid motions
    assert np.allclose(M[:, 3], [0, 0, 0, 1])


def test_select_base_is_wide_and_deterministic():
    raw, P, Q, cp, cq = bench.build_workload(5000)
    d = float(np.linalg.norm(P.max(0) - P.min(0)))
    a = bench.select_base(P, np.random.RandomState(3), d)
    b = bench.select_base(P, np.random.RandomState(3), d)
    assert np.array_equal(a[0], b[0]) and a[1] == b[1] and a[2] == b[2]
    assert len(set(a[0].tolist())) == 4 and 0.0 <= a[1] <= 1.0 and 0.0 <= a[2] <= 1.0


def test_reference_arm_prints_the_contract_line():
    """`bench.py --impl reference` on a reduced debug size (the metric itself is quoted at 1M points on the GPU box):
    one JSON line on stdout with every key of the contract, nothing else"""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--impl", "reference", "--points", "20000",
                        "--candidates", "64", "--ref-per-thread", "1", "--steps", "2", "--warmup", "1"],
                       capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [ln for ln in r.stdout.splitlines() if ln.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("impl", "metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "cpu_baseline", "e2e", "gpu_launches"):
        assert k in d, k
    assert d["impl"] == "reference" and d["steps"] == 2 and d["warmup"] == 1 and d["value"] > 0
    assert d["cpu_baseline"]["kind"] in ("reference", "port") and d["cpu_baseline"]["cores"] >= 1
    assert d["e2e"]["h2d_bytes_per_step"] == 0 and d["config"]["workload"].startswith("cfg2")
    assert "20000 x" in d["cpu_baseline"]["sample"] and "physical cores" in d["cpu_baseline"]["sample"]
    assert d["cpu_baseline"]["as_shipped_1thread"]["cores"] == 1 and d["cpu_baseline"]["as_shipped_1thread"]["value"] > 0
    assert d["cpu_baseline"]["no_early_exit"]["value"] > 0 and "early exit" in d["cpu_baseline"]["sample"]


def test_physical_cores_counts_smt_siblings_once():
    assert 1 <= bench.physical_cores() <= bench.host_threads()

