"""The quad search's edge fixtures of tests/quads.py and its restatement, checked without a GPU: on every fixture the
restatement's quads equal the port's and, where the reference is built, the reference's own
FindCongruentQuadrilaterals; every family puts some decision between neighbouring floats; the restatement agrees with a
float64 evaluation away from the boundaries; every catchable wrong form of a decision changes some fixture;
and a host emulation of the batched quad keys and offsets shows the two limits the batched chain has to enforce."""
import numpy as np
import pytest

from oracle import port as oport
from oracle import ref as oref
from tests import edges as E
from tests import quads as T


def _supported(fx):
    return 0 <= T.grid(fx["thr2"], T.normalization(fx["Q"])[1])[0] <= 18


@pytest.mark.parametrize("family", list(T.FAMILIES))
def test_restatement_equals_the_port(family):
    ports = {}
    for fx in T.fixtures(family):
        if not _supported(fx):
            with pytest.raises(ValueError):
                T.run(fx)
            continue
        key = fx["Q"].tobytes()
        if key not in ports:
            ports[key] = oport.Port(fx["Q"][:1], fx["Q"], 0.01)
        got = ports[key].find_quads(fx["inv1"], fx["inv2"], fx["thr2"], fx["base"], fx["pairs1"], fx["pairs2"])
        assert np.array_equal(got, T.run(fx)), fx["name"]


@pytest.mark.skipif(not oref.available(), reason="oracle/_ref (compiled reference) not present")
@pytest.mark.parametrize("family", list(T.FAMILIES))
def test_restatement_equals_the_reference(family):
    """RefMatcher on the fixture's cloud: its init centres Q, so the restatement runs on the reference's sampled Q.  The
    reference allocates a dense egSize^3 grid on every call: depths beyond 8 are not run through it"""
    refs = {}
    opt = oref.make_options(delta=0.01, sample_size=10 ** 8)
    for fx in T.fixtures(family):
        if not _supported(fx):
            continue
        key = fx["Q"].tobytes()
        if key not in refs:
            m = oref.RefMatcher(fx["Q"], fx["Q"], opt)
            refs[key] = (m, m.sampled_q()[0])
        m, Qs = refs[key]
        gc, ratio = T.normalization(Qs)
        if not 0 <= T.grid(fx["thr2"], ratio)[0] <= 8:
            continue
        m.set_base3d(fx["base"])
        want = m.find_quads(fx["inv1"], fx["inv2"], fx["thr2"], fx["thr2"], fx["pairs1"], fx["pairs2"])
        mine = T.find_quads(Qs, gc, ratio, fx["pairs1"], fx["pairs2"], fx["inv1"], fx["inv2"], fx["thr2"], fx["base"])
        assert np.array_equal(want, mine), fx["name"]


def _flips(family):
    """{group: {k: decision}} of the family's fixtures at k floats from their boundary"""
    out = {}
    for fx in T.fixtures(family):
        if fx["k"] is not None and (fx["probe"] is not None or fx["decide"]):
            out.setdefault(fx["name"].rsplit("-k", 1)[0], {})[fx["k"]] = T.decision(fx)
    return out


def _flipping(groups, nearest=False):
    """groups decided differently at -1 and +1 floats (nearest: at the reached k closest to the boundary on each side)"""
    out = []
    for g, by_k in groups.items():
        lo = [k for k in by_k if k < 0]
        lo, hi = (max(lo) if lo and nearest else -1), 1
        if lo in by_k and hi in by_k and by_k[lo] != by_k[hi]:
            out.append(g)
    return out


@pytest.mark.parametrize("family", ["cell_face", "bin_face", "distance", "cone", "opposite", "fused", "depth"])
def test_every_family_decides_its_neighbouring_floats_differently(family):
    groups = _flips(family)
    # the query point's cell coordinate just below 2 is not reached from a float32 world coordinate in the fused family
    flipping = _flipping(groups, nearest=family == "fused")
    assert flipping, family
    if family == "cell_face":                       # both invariant points, every axis, every depth
        assert {g.split("-")[2] + g.split("-")[3] for g in flipping} == {s + "ax%d" % a for s in "PQ" for a in range(3)}
    if family == "bin_face":                        # a P-pair direction and a cone sample direction
        assert {g.split("-")[1] for g in flipping} == {"P", "S"}
    if family == "cone":                            # every step of nbSample, 2 .. 56
        assert sorted(int(g.split("-n")[1]) for g in flipping) == list(range(2, 57, 2))
    if family == "depth":                           # depth 0 / error, 14 / 15, 18 / error
        assert sorted(flipping) == ["depth-edge--1", "depth-edge-14", "depth-edge-18"]
        assert {g: (v[-1], v[1]) for g, v in groups.items()} == \
            {"depth-edge--1": (0, -1), "depth-edge-14": (15, 14), "depth-edge-18": (19, 18)}
    for g in flipping:                              # one boundary: the decision is the same on each side of it
        by_k = groups[g]
        lo = max(k for k in by_k if k < 0)
        assert all(by_k[k] == by_k[lo] for k in by_k if k < 0) and all(by_k[k] == by_k[1] for k in by_k if k > 0), g


def test_cone_corners():
    by_name = {fx["name"]: fx for fx in T.fixtures("cone")}
    got = {n: T.decision(by_name[n]) for n in ("ac_one", "ac_below_one", "ac_above_one", "ac_minus_one", "ac_zero")}
    assert got == {"ac_one": 0, "ac_below_one": 2, "ac_above_one": 0, "ac_minus_one": 56, "ac_zero": 46}
    assert T.alpha_cos(by_name["ac_above_one"]["base"]) > 1
    assert len(T.run(by_name["ac_above_one"])) == 0 and len(T.run(by_name["ac_one"])) == 0
    assert len(T.run(by_name["ac_minus_one"])) > 0


def test_the_sample_cap_never_binds():
    """nbSample is largest at alpha_cos = -1 (alpha = acosf(-1), pi rounded up), and there it is 56: the cap of 56 is
    never reached, so removing it changes nothing"""
    assert T.n_samples(np.float32(-1), "no_cap") == 56
    xs = E.step(np.float32(-1), np.arange(0, 4096))
    assert max(T.n_samples(x, "no_cap") for x in xs) == 56


@pytest.mark.parametrize("mutant", T.CATCHABLE)
def test_every_wrong_decision_changes_some_fixture(mutant):
    """'<' for '<=' in the distance test, rounded direction bins, '<=' for '<' at c = -1 + 1e-5 (the regular branch
    rotates +z about 0.07 rad away from the nearly-opposite one there) and a fused query point each change the quads of
    some fixture.  The sample cap is the one wrong form no input can tell apart (test_the_sample_cap_never_binds)."""
    changed = [fx["name"] for fx in T.all_fixtures() if _supported(fx) and
               not np.array_equal(T.run(fx, mutant), T.run(fx))]
    assert changed, mutant


@pytest.mark.parametrize("seed", range(4))
def test_float64_evaluation_agrees_away_from_the_boundaries(seed):
    """random clouds, bases, invariants and depths 0 .. 6: where every decision that (P-pair, Q-pair) depends on is at
    least 1e-4 (relative) from its boundary, the float32 restatement and the float64 predicate agree"""
    rng = np.random.RandomState(seed)
    Q, pairs = T.crowd(n=22, seed=100 + seed, spread=1.2)
    gc, ratio = T.normalization(Q)
    checked = hits = 0
    for depth in range(7):
        thr2 = np.float32(4.0 * rng.uniform(0.55, 0.95) * 2.0 ** -depth)
        base = T._alpha_base(rng.uniform(0.05, 3.0))
        inv1, inv2 = np.float32(rng.uniform(0.1, 0.9)), np.float32(rng.uniform(0.1, 0.9))
        _, info = T.find_quads(Q, gc, ratio, pairs, pairs, inv1, inv2, thr2, base, detail=True)
        hit64, margin = T.find_quads64(Q, gc, ratio, pairs, pairs, float(inv1), float(inv2), float(thr2), base)
        ok = margin >= 1e-4
        assert np.array_equal(info["hit"][ok], hit64[ok]), depth
        checked += int(ok.sum())
        hits += int(hit64[ok].sum())
    assert checked > 0.5 * 7 * len(pairs) ** 2 and hits > 100


@pytest.mark.parametrize("family", list(T.FAMILIES))
def test_float64_evaluation_agrees_on_the_fixtures_away_from_their_boundaries(family):
    """the same cross-check on the fixtures' own geometry: the pairs whose decisions are all at least 1e-4 from their
    boundaries (most pairs of the crowded fixtures, the designed pair of an edge fixture only at its far k)"""
    checked = 0
    for fx in T.fixtures(family):
        if not _supported(fx):
            continue
        gc, ratio = T.normalization(fx["Q"])
        args = (fx["pairs1"], fx["pairs2"], fx["inv1"], fx["inv2"], fx["thr2"], fx["base"])
        _, info = T.find_quads(fx["Q"], gc, ratio, *args, detail=True)
        hit64, margin = T.find_quads64(fx["Q"], gc, ratio, *args[:2], float(fx["inv1"]), float(fx["inv2"]),
                                       float(fx["thr2"]), fx["base"])
        ok = margin >= 1e-4
        assert np.array_equal(info["hit"][ok], hit64[ok]), fx["name"]
        checked += int(ok.sum())
    if family in ("cone", "depth", "crowd"):          # many pairs each; the edge fixtures are near a boundary by design
        assert checked > 0


# ---- the batched quad keys, emulated -----------------------------------------------------------------------------------
def test_a_pair_index_of_26_bits_or_more_corrupts_the_batched_quad_key():
    """k_bquad_query packs base << 52 | id << 26 | i; with one base, a P-pair index id >= 2^26 reads back as base 1 and a
    Q-pair index i >= 2^26 as another id: an extraction of 2^26 pairs or more has to be refused"""
    assert T.unpack_quad_key(T.pack_quad_key(0, 2 ** 26 - 1, 2 ** 26 - 1)) == (0, 2 ** 26 - 1, 2 ** 26 - 1)
    assert T.unpack_quad_key(T.pack_quad_key(0, 2 ** 26, 5)) == (1, 0, 5)
    assert T.unpack_quad_key(T.pack_quad_key(0, 6, 2 ** 26 + 3)) == (0, 7, 3)
    # about 8200 points whose pair band covers every distance already give 2^26 ordered pairs
    assert 8193 * 8192 >= 2 ** 26 > 8192 * 8191


def test_a_batch_of_2_32_quads_wraps_the_32_bit_offsets():
    """the per-entry quad counts are scanned in 32 bits: the collinear cloud of the GPU test (310 points, every ordered
    pair in both extractions, every Q-pair matching the P-pairs of its orientation) has about 4.6e9 quads, and the wrapped
    total passes the 2^31 - 1 check"""
    n = 310
    pairs = n * (n - 1)
    counts = np.concatenate([np.full(pairs, 0, np.uint32), np.full(pairs, pairs // 2, np.uint32)])   # P then Q entries
    exact = int(counts.astype(np.uint64).sum())
    off, total32 = T.scan32(counts)
    assert exact > 2 ** 32 and exact == pairs * (pairs // 2)
    assert total32 == exact - 2 ** 32 and total32 < 2 ** 31 - 1
    assert (np.diff(off.astype(np.int64)) < 0).any()              # the offsets run backwards: the fill overlaps itself
