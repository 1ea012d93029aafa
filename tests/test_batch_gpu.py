"""Row f1, single-launch form (s4g_try_bases): B bases through ONE launch chain -- base index as a grid dimension /
key prefix, three read-backs per batch -- must give, per base, exactly what the per-base chain
s4g_extract_pairs x2 -> s4g_find_quads -> s4g_try_congruent_set_resident gives (pair counts, quad count, gate passes,
winner index / count / transform bits), and the C++ layer with S4PCS_BATCH must reproduce the golden hippo result and
the reference's traces."""
import os

import numpy as np
import pytest

import bench
from oracle import _build
from tests import common
from tests.test_host_logic_cpu import ROOT, run_driver

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(_build.build_ref() is None, reason="oracle/_ref (compiled reference) not present")


def _bases(P, Pn, rng, k, diameter):
    out = []
    sub = rng.choice(len(P), min(len(P), 20000), replace=False)
    while len(out) < k:
        ids, inv1, inv2 = bench.select_base(P[sub], rng, diameter)
        pid = sub[ids]
        bx = P[pid]
        bn = np.zeros((4, 3), np.float32) if Pn is None else (Pn[pid] / np.linalg.norm(Pn[pid], axis=1, keepdims=True)).astype(np.float32)
        b9 = np.concatenate([bx, bn, -np.ones((4, 3), np.float32)], axis=1).astype(np.float32)
        out.append(dict(d1=bench._eigen_norm(bx[0] - bx[1]), d2=bench._eigen_norm(bx[2] - bx[3]),
                        na1=bench._eigen_norm(bn[0] - bn[1]), na2=bench._eigen_norm(bn[2] - bn[3]),
                        b9=b9, bxp=bx, inv1=inv1, inv2=inv2))
    return out


@pytest.mark.parametrize("n,ns,delta,normals,nb,patches", [
    pytest.param(20000, 400, 0.02, False, 7, None, id="20000-400-0.02-False-7"),
    pytest.param(50000, 3000, 0.01, False, 5, None, id="50000-3000-0.01-False-5"),
    pytest.param(30000, 2000, 0.015, True, 9, None, id="30000-2000-0.015-True-9"),
    pytest.param(5000, 70, 0.05, False, 33, None, id="5000-70-0.05-False-33"),
    # Verify's queries in 3 / 2 patches (S4G_VERIFY_PATCHES): the batched chain runs them with its device-side candidate
    # count and candidates beyond it keyed last, the per-base chain with a host count
    pytest.param(50000, 3000, 0.01, False, 5, 3, id="50000-3000-0.01-False-5-patches3"),
    pytest.param(30000, 2000, 0.015, True, 9, 2, id="30000-2000-0.015-True-9-patches2")])
def test_try_bases_equals_the_per_base_chain(s4g_lib, monkeypatch, n, ns, delta, normals, nb, patches):
    from super4pcs_b200 import Context, PairFilters
    if patches is not None:
        monkeypatch.setenv("S4G_VERIFY_PATCHES", str(patches))
    sc = common.scenario(n, 0.5, delta, seed=n % 97, normals=normals)
    rng = np.random.RandomState(ns)
    sel = rng.choice(n, ns, replace=False)
    Qs = np.ascontiguousarray(sc["Q"][sel])
    Qn = None
    if normals:
        Qn = (sc["Qn"][sel] / np.linalg.norm(sc["Qn"][sel], axis=1, keepdims=True)).astype(np.float32)
    filt = PairFilters(35.0, -1, -1, -1) if normals else PairFilters(-1, -1, -1, -1)
    diameter = float(np.linalg.norm(sc["P"].max(0) - sc["P"].min(0)))
    bases = _bases(sc["P"], sc["Pn"] if normals else None, rng, nb, diameter)
    eps = 2 * delta
    with Context(0) as ctx:
        ctx.set_cloud_p(sc["P"], delta)
        ctx.set_cloud_q(Qs, normals=Qn)
        got = ctx.try_bases(bases, eps, eps, eps, filters=filt)
        assert len(got) == nb
        some_quads = 0
        for b, g in zip(bases, got):
            n1 = ctx.extract_pairs(b["d1"], b["na1"], eps, b["b9"][0], b["b9"][1], filt, slot=0, fetch=False)
            n2 = ctx.extract_pairs(b["d2"], b["na2"], eps, b["b9"][2], b["b9"][3], filt, slot=1, fetch=False)
            assert g["n_pairs"] == [n1, n2]
            nq = ctx.find_quads(b["inv1"], b["inv2"], eps, b["b9"][:, :3], fetch=False) if n1 and n2 else 0
            assert g["n_quads"] == nq
            if nq == 0:
                assert g["tcs"]["best_index"] == -1 and g["tcs"]["n_gate_pass"] == 0
                continue
            some_quads += 1
            w = ctx.try_congruent_set_resident(b["bxp"], eps)
            t = g["tcs"]
            for k in ("key", "best_count", "best_index", "n_gate_pass", "n_q"):
                assert t[k] == w[k], k
            assert np.array_equal(t["T"].view(np.uint32), w["T"].view(np.uint32))
            assert np.array_equal(t["quad"], w["quad"]) and np.float32(t["rms"]) == np.float32(w["rms"]) or w["best_index"] < 0
            assert np.array_equal(t["centroid1"].view(np.uint32), w["centroid1"].view(np.uint32))
            assert np.array_equal(t["centroid2"].view(np.uint32), w["centroid2"].view(np.uint32))
        assert some_quads >= 1
        # a second batch on the same context (buffers are reused) and a batch of one
        again = ctx.try_bases(bases[:1], eps, eps, eps, filters=filt)
        assert again[0]["n_pairs"] == got[0]["n_pairs"] and again[0]["tcs"]["key"] == got[0]["tcs"]["key"]


def test_try_bases_argument_limits(s4g_lib):
    from super4pcs_b200 import Context, S4GError
    sc = common.scenario(3000, 0.4, 0.02)
    b = _bases(sc["P"], None, np.random.RandomState(1), 1, 2.0)
    with Context(0) as ctx:
        ctx.set_cloud_p(sc["P"], 0.02)
        ctx.set_cloud_q(sc["Q"])
        with pytest.raises(S4GError):
            ctx.try_bases(b * 65, 0.04, 0.04, 0.04)                    # more than 64 bases
        with pytest.raises(S4GError):
            ctx.try_bases(b, 0.04, 2.0 ** -16 * 2.3, 0.04)             # quad grid deeper than the batched keys allow


@pytest.fixture(scope="module")
def built(s4g_lib):
    from super4pcs_b200 import build_cpp
    if build_cpp.build_all()["lib"] is None or _build.build_dropin_harness() is None:
        pytest.skip("C++ layer not available")


@pytest.mark.parametrize("batch,lanes", [(8, 1), (3, 1), (64, 1)])
def test_hippo_with_batched_bases_matches_golden(built, batch, lanes):
    g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
    r = run_driver("hippo", "dropin", lanes=lanes, extra_env={"S4PCS_BATCH": str(batch)}, timeout=300)
    assert np.float32(r["score"]) == g["score"] == np.float32(0.64)
    assert np.array_equal(np.array(r["T"], np.uint32), g["T_colmajor"].view(np.uint32))


@needs_ref
@pytest.mark.parametrize("which", ["trace", "steps", "ties", "sweep1", "prealigned"])
def test_batched_bases_match_reference_traces(built, which):
    want = run_driver(which, "reference")
    if which == "ties":
        want = {"rows": [[True, True]] * 4}
    assert run_driver(which, "dropin", extra_env={"S4PCS_BATCH": "8"}, timeout=600) == want
