"""GPU tests collected AFTER every other GPU test (file name order).  The a1 normalisation,
the GPU variant of the randomised pipeline sweep and the exact-order tie cases (see tests/test_host_logic_cpu.py for the
CPU twins on the oracle stand-in)."""
import os

import numpy as np
import pytest

from oracle import _build
from oracle import port as oport
from tests import common
from tests.test_host_logic_cpu import ROOT, run_driver, timings_report

pytestmark = pytest.mark.gpu

needs_ref = pytest.mark.skipif(_build.build_ref() is None, reason="oracle/_ref (compiled reference) not present")


@pytest.fixture(scope="module")
def ctx(s4g_lib):
    from super4pcs_b200 import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def built(s4g_lib):
    from super4pcs_b200 import build_cpp
    if build_cpp.build_all()["lib"] is None or _build.build_dropin_harness() is None:
        pytest.skip("C++ layer not available")


@pytest.mark.parametrize("n,seed,shift", [(3000, 1, 0.0), (777, 5, 12.5), (4097, 4, -3.25)])
def test_q_normalization_matches_oracle(ctx, n, seed, shift):
    """a1 (PairCreationFunctor::synch3DContent, pairCreationFunctor.h:90-122): _gcenter and _ratio bit for bit -- the
    host replay of S4PCS_EXACT_ORDER rebuilds the unit-cube coordinates from exactly these numbers"""
    sc = common.scenario(n, 0.4, 0.02, seed=seed)
    Q = (sc["Q"] + np.float32(shift)).astype(np.float32)
    ctx.set_cloud_p(sc["P"], 0.02)
    ctx.set_cloud_q(Q)
    g, ratio = ctx.q_normalization()
    wg, wratio = oport.Port(sc["P"], Q, 0.02).normalization()
    assert np.array_equal(np.asarray(g, np.float32).view(np.uint32), np.asarray(wg, np.float32).view(np.uint32))
    assert np.float32(ratio) == np.float32(wratio)


@needs_ref
@pytest.mark.parametrize("seed,lanes", [(2, 3), (3, 1)])
def test_randomised_pipeline_sweep_on_the_gpu_matches_reference(built, seed, lanes):
    """the randomised whole-pipeline sweep of tests/test_host_logic_cpu.py on the real CUDA library"""
    want = run_driver("sweep%d" % seed, "reference")
    assert run_driver("sweep%d" % seed, "dropin", lanes=lanes) == want


@needs_ref
def test_exact_order_mode_resolves_equal_count_ties_like_the_reference_on_the_gpu(built):
    """Equal-count ties on the real CUDA library (see tests/test_host_logic_cpu.py::test_equal_count_ties_...): the four
    committed tie cases come out bit-identical to the reference with NO environment variable (exact order is the default
    since round 2); with the replay turned off (S4PCS_EXACT_ORDER=0) only the score is."""
    same = {"rows": [[True, True]] * 4}
    off = run_driver("ties", "dropin", extra_env={"S4PCS_EXACT_ORDER": "0"})
    assert all(score_equal for score_equal, _ in off["rows"])
    for lanes, fused in ((1, 1), (3, 1), (1, 0)):
        assert run_driver("ties", "dropin", lanes=lanes, fused=fused) == same


def test_stage_timings_report_on_the_gpu(built, tmp_path):
    """S4PCS_TIMINGS=1 on the real library: the counts of the report (ordered pairs, quads, verified candidates, bases) do not
    depend on the lane count, the device times are real (> 0) and their sum stays below the wall clock"""
    import re
    from super4pcs_b200 import build_cpp
    demo = build_cpp.build_all()["demo"]
    if not demo:
        pytest.skip("demo binary not available")
    assert timings_report(demo, tmp_path) is None

    def parse(rows):
        ms = [float(re.search(r":\s*([0-9.eE+-]+)", r).group(1)) for r in rows[:4]]
        counts = [re.search(r"\(device; (.*)\)", r).group(1) for r in rows[:3]] + [rows[4].split(":")[1].strip()]
        return ms, counts

    ms1, c1 = parse(timings_report(demo, tmp_path, S4PCS_TIMINGS="1"))
    ms2, c2 = parse(timings_report(demo, tmp_path, S4PCS_TIMINGS="1", S4PCS_LANES="3"))
    assert c1 == c2 and c1[3] == "139"
    assert all(m > 0 for m in ms1) and sum(ms1) < 60000
