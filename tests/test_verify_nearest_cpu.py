"""The nearest P point within delta of every transformed Q point (s4g_verify_nearest, Match4PCSBase::getCorrespondences)
without a GPU: the port's brute force against the compiled reference's own kd-tree query, and the C++ layer's
getCorrespondences on the oracle stand-in of libs4g.

Contract (include/s4g.h): index = the P point with the smallest d^2 <= delta^2, equal d^2 -> the smallest index, -1 when
none; sq_dist = that d^2 bit for bit (+inf for -1).  The reference keeps the last point of equal distance its traversal
visits, so its index may differ from ours only inside a tie, and then ours is the smaller one."""
import os

import numpy as np
import pytest

from oracle import nearest as onear
from oracle import port as oport
from tests import common, correspondences

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
needs_ref = pytest.mark.skipif(not onear.ref_available(), reason="oracle/_ref (compiled reference) not present")


def check_against_reference(P, index, sq, ref_index, ref_sq, T16, Q):
    """index / sq (ours) against the reference's: same hits, bit-equal sq_dist, a different index only inside a tie
    (both points at the same d^2) and then ours is the smaller one.  Returns the number of rows decided by a tie."""
    assert np.array_equal(index >= 0, ref_index >= 0)
    assert np.array_equal(common.bits(sq), common.bits(ref_sq))
    k, i = np.nonzero(index != ref_index)
    for kk, ii in zip(k, i):
        T = T16[kk].reshape(4, 4).T
        t = (((T[:3, 0] * Q[ii, 0]).astype(np.float32) + (T[:3, 1] * Q[ii, 1]).astype(np.float32)).astype(np.float32)
             + (T[:3, 2] * Q[ii, 2]).astype(np.float32)).astype(np.float32) + T[:3, 3]
        d = (t.astype(np.float32) - P[[index[kk, ii], ref_index[kk, ii]]]).astype(np.float32)
        d2 = (d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])).astype(np.float32)
        assert d2[0] == d2[1] == sq[kk, ii] and index[kk, ii] < ref_index[kk, ii]
    return len(k)


def ref_and_port(P, Q, delta, T16):
    """the reference matcher on (P, Q) with every point kept; the port on the reference's centred sampled clouds"""
    m = onear.RefNearest(P, Q, delta)
    sP, sQ = m.sampled()
    ri, rs = m.query(T16)
    pi, ps, pc = onear.bruteforce(sP, sQ, delta, T16)
    _, good, _ = oport.Port(sP, sQ, delta).verify_batch(T16, 0.0)
    assert np.array_equal(pc, good)                         # count = Verify's count
    assert np.array_equal((pi >= 0).sum(1), pc)
    assert np.array_equal(common.bits(ps[pi < 0]), common.bits(np.full((pi < 0).sum(), np.inf, np.float32)))
    return sP, sQ, pi, ps, ri, rs


@needs_ref
@pytest.mark.parametrize("n,delta,seed", [(2000, 0.02, 1), (3000, 0.01, 4)])
def test_port_matches_reference_kdtree_on_seeded_clouds(n, delta, seed):
    sc = common.scenario(n, 0.4, delta, seed=seed)
    T16 = np.concatenate([common.candidates_colmajor(sc, 24, seed=seed, n_near=12),
                          np.eye(4, dtype=np.float32).reshape(1, 16)])     # near-GT, random, identity
    sP, sQ, pi, ps, ri, rs = ref_and_port(sc["raw"]["P"], sc["raw"]["Q"], delta, T16)
    assert (pi[:12] >= 0).sum() > 0.01 * len(sQ) * 12                       # the near-GT transforms find neighbours
    check_against_reference(sP, pi, ps, ri, rs, T16, sQ)


@needs_ref
def test_port_matches_reference_kdtree_on_hippo_samples():
    g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
    P, Q = g["stage_P"], g["stage_Q"]
    rng = np.random.RandomState(5)
    T = [g["stage_b0_tcs_T"], np.eye(4, dtype=np.float32).reshape(16)]
    T += list(g["stage_b0_verify_T"])
    for _ in range(6):                                                      # random rotations about the cloud
        A = np.linalg.qr(rng.standard_normal((3, 3)))[0]
        M = np.eye(4)
        M[:3, :3] = A * np.sign(np.linalg.det(A))
        M[:3, 3] = rng.uniform(-0.05, 0.05, 3)
        T.append(M.astype(np.float32).T.reshape(16))
    T16 = np.ascontiguousarray(T, np.float32)
    sP, sQ, pi, ps, ri, rs = ref_and_port(P, Q, 0.01, T16)
    assert (pi[0] >= 0).sum() > 0
    check_against_reference(sP, pi, ps, ri, rs, T16, sQ)


@needs_ref
def test_exact_ties_resolve_to_the_smallest_index():
    """duplicated P points: every neighbour that has a copy is a tie; ours is the first copy, the reference's is one of
    the copies (the one its traversal visits last)"""
    sc = common.scenario(1500, 0.4, 0.02, seed=9)
    P0 = sc["raw"]["P"]
    P = np.concatenate([P0, P0[::2]])                                       # copies at the end: larger indices
    T16 = np.concatenate([common.candidates_colmajor(sc, 8, seed=2, n_near=8), np.eye(4, dtype=np.float32).reshape(1, 16)])
    sP, sQ, pi, ps, ri, rs = ref_and_port(P, sc["raw"]["Q"], 0.02, T16)
    check_against_reference(sP, pi, ps, ri, rs, T16, sQ)
    hit = pi >= 0
    assert hit.sum() > 100
    assert (pi[hit] < len(P0)).all()                                        # never a later copy
    dup = hit & (pi < len(P0)) & (pi % 2 == 0)                              # neighbours that have a copy
    assert dup.sum() > 50
    assert ((ri[dup] == pi[dup]) | (ri[dup] == len(P0) + pi[dup] // 2)).all()
    assert (ri[dup] != pi[dup]).sum() > 0                                  # the reference did pick later copies


@pytest.fixture(scope="module")
def program(s4g_lib, tmp_path_factory):
    from tests import build_shim
    d = tmp_path_factory.mktemp("corr")
    exe = correspondences.build(d)
    if exe is None:
        pytest.skip("C++ layer not buildable here (no Eigen)")
    return exe, build_shim.build()


def test_get_correspondences_on_oracle_shim_hippo(program, tmp_path):
    """the run-example options (-o 0.7 -d 0.01 -n 200): the golden registration, 0.64 x 200 = 128 correspondences, equal
    to the port's brute force on getFirstSampled() / getSecondSampled() under the centred transform behind the score"""
    exe, shim = program
    h = np.load(os.path.join(ROOT, "tests", "golden", "hippo.npz"))
    g = np.load(os.path.join(ROOT, "tests", "golden", "hippo_result.npz"))
    r = correspondences.run(exe, tmp_path, h["P"], h["Q"], 0.01, 0.7, 200, preload=shim)
    assert r["threw_before"] == 1                                           # no registration yet: throws
    assert r["score"] == g["score"] == np.float32(0.64)
    assert np.array_equal(common.bits(r["T"]), common.bits(g["T_colmajor"]))
    assert len(r["sP"]) == int(g["nP"]) and len(r["sQ"]) == int(g["nQ"]) == 200
    assert (r["nearest"] >= 0).sum() == 128
    pi, ps, pc = onear.bruteforce(r["sP"], r["sQ"], 0.01, r["C"])
    assert np.array_equal(r["nearest"], pi[0])
    assert np.array_equal(common.bits(r["sq"]), common.bits(ps[0]))
    assert np.array_equal(r["nearest2"], r["nearest"])
