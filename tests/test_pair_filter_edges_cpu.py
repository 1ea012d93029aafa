"""The pair filters' edge cases of tests/pair_filters.py and its oracle, checked without a GPU: on every case the oracle's
ordered pair set equals the port's and, where the reference is built, the reference's own ExtractPairs; and the cases
reach what the GPU tests rely on -- every threshold decided differently at 0 and +-1 floats, both p/q roles and both index
orders, both orientations, and every wrong form of a decision in tests/pair_filters.MUTANTS changes some count."""
import math

import numpy as np
import pytest

from oracle import port as oport
from oracle import ref as oref
from tests import edges as E
from tests import pair_filters as F

GROUPS = {"segments": F.segment_cases, "angle_sweep": F.angle_sweep_cases, "special": F.special_cases}
_cache = {}


def cases(group):
    if group not in _cache:
        _cache[group] = GROUPS[group]()
    return _cache[group]


@pytest.mark.parametrize("group", list(GROUPS))
def test_oracle_equals_the_port(group):
    ports = {}
    for case in cases(group):
        c = case["cloud"]
        if c["name"] not in ports:
            ports[c["name"]] = oport.Port(c["Q"][:1], c["Q"], 0.01, Qn=c["Qn"], Qrgb=c["Qrgb"])
        got = ports[c["name"]].extract_pairs(case["d"], case["na"], case["eps"], case["b1"], case["b2"], case["filters"])
        assert np.array_equal(got, F.oracle_pairs(case)), case["name"]


@pytest.mark.skipif(not oref.available(), reason="oracle/_ref (compiled reference) not present")
@pytest.mark.parametrize("group", list(GROUPS))
def test_oracle_equals_the_reference(group):
    """RefMatcher with the case's filter options, base_3D_ = (b1, b2, ., .) with rgb: the reference's pair set equals the
    oracle's on the clouds the reference holds.  Its init centres Q (the mirrored clouds stay bit-identical) and keeps a
    normal only after normalizing it, so the oracle runs on the reference's sampled normals and rgb."""
    refs = {}
    for case in cases(group):
        c = case["cloud"]
        key = (c["name"], case["filters"])
        if key not in refs:
            mnd, mtd, ma, mcd = case["filters"]
            opt = oref.make_options(delta=0.01, max_normal_difference=mnd, max_translation_distance=mtd, max_angle=ma,
                                    max_color_distance=mcd, sample_size=10 ** 8)
            m = oref.RefMatcher(c["Q"], c["Q"], opt, Qn=c["Qn"], Qrgb=c["Qrgb"])
            xyz, nrm, rgb = m.sampled_q()
            assert np.array_equal(xyz.view(np.uint32), c["Q"].view(np.uint32)), c["name"]
            if c["Qrgb"] is not None:
                assert np.array_equal(rgb.view(np.uint32), c["Qrgb"].view(np.uint32))
            refs[key] = (m, nrm, rgb)
        m, nrm, rgb = refs[key]
        b = np.zeros((4, 9), np.float32)
        b[:, 6:9] = -1
        b[0], b[1] = case["b1"], case["b2"]
        m.set_base3d(b[:, :3], b[:, 3:6], b[:, 6:9])
        want = m.extract_pairs(case["d"], case["na"], case["eps"], 0, 1)
        mine = F.ordered(*F.pair_bits(c["Q"], nrm, rgb, case["d"], case["na"], case["eps"], case["b1"], case["b2"],
                                      case["filters"]))
        assert np.array_equal(want, mine), case["name"]


def _decisions(group_cases):
    """{(filter, side, order): {k: kept}} of the designed pairs"""
    out = {}
    for case in group_cases:
        pr = case["probe"]
        if pr is None or "k" not in pr or "mixed" in pr or "filter" not in pr:
            continue
        out.setdefault((pr["filter"], pr["side"], pr.get("order")), {})[pr["k"]] = bool(F.probe_bits(case) & pr["bit"])
    return out


# which side of the threshold keeps the pair: strict '<' (translation, colour) keeps k < 0; 'nd > thr' rejects k > 0;
# 'dt >= cos_angle_min' keeps k >= 0
KEEPS = {"translation": lambda k: k < 0, "colour": lambda k: k < 0, "normal": lambda k: k <= 0,
         "normal_nonunit": lambda k: k <= 0, "angle": lambda k: k >= 0}


def test_every_threshold_flips_between_its_neighbouring_floats():
    dec = _decisions(cases("segments")) | _decisions(cases("special"))
    want = {("translation", s, o) for s in ("p", "q") for o in ("follows", "against")}
    want |= {("colour", s, o) for s in ("p", "q") for o in ("follows", "against")}
    want |= {("normal", s, o) for s in ("first", "second") for o in ("follows", "against")}
    want |= {("angle", s, o) for s in ("bit0", "bit1") for o in ("follows", "against")}
    want |= {("normal_nonunit", s, None) for s in ("first", "second")}
    assert want <= set(dec)
    # the same translation edge with another filter clearly failing (never kept) or on its passing edge (unchanged)
    for case in cases("segments"):
        pr = case["probe"]
        if "mixed" in pr:
            assert bool(F.probe_bits(case) & 1) == (pr["mixed"] is None and pr["k"] < 0), case["name"]
    for key, by_k in dec.items():
        if key[0] not in KEEPS:
            continue
        assert sorted(by_k) == list(E.KS), key
        assert {k: KEEPS[key[0]](k) for k in E.KS} == by_k, key


def test_max_angle_sweep_flips_at_cos_angle_min():
    dec = _decisions(cases("angle_sweep"))
    for ma in F.MAX_ANGLES:
        cmin = F.cos_angle_min(ma)
        for side in ("bit0", "bit1"):
            orders = [o for (f, s, o) in dec if f == "angle%g" % ma and s == side]
            assert orders, (ma, side)
            for order in orders:
                by_k = dec[("angle%g" % ma, side, order)]
                assert 0 in by_k and by_k[0], (ma, side, order)
                assert all(v == (k >= 0) for k, v in by_k.items()), (ma, side, order)
                if cmin > -1:                     # a float below cos_angle_min exists: it was reached and rejected
                    assert -1 in by_k and not by_k[-1], (ma, side, order)
    assert {o for (f, s, o) in dec if f == "angle90"} == {"axis"}
    assert F.cos_angle_min(1e-3) == 1.0          # a tiny angle keeps dt == 1 only
    assert F.cos_angle_min(200.0) == -1.0
    # acosf(-1) is pi rounded up to a float, above M_PI: at 180 degrees dt = -1 is rejected
    assert F.acosf(np.float32(-1))[()] > math.pi and F.cos_angle_min(180.0) == E.step(np.float32(-1), 1)


def test_special_cases_decide_as_intended():
    sp = {c["name"]: c for c in cases("special")}
    for ma in ("30", "0.001", "1e-20"):
        assert F.probe_bits(sp["dt_self_gt1_ma" + ma]) == 0          # fl(dt) > 1: acosf is NaN, the pair is rejected
        assert F.probe_bits(sp["dt_self_eq1_ma" + ma]) == 1          # dt == 1 passes any positive max_angle
    # segment1 = 0 (b1 == b2): dt = 0, and acosf(0) is above pi / 2 in double
    assert len(F.oracle_pairs(sp["b1_eq_b2_ma90.0"])) == 0
    assert len(F.oracle_pairs(sp["b1_eq_b2_ma%r" % float(E.step(np.float32(90), 1))])) == \
        len(F.oracle_pairs(sp["no_filters"]))
    assert len(F.oracle_pairs(sp["max_angle_0"])) == len(F.oracle_pairs(sp["no_filters"]))
    assert len(F.oracle_pairs(sp["no_normals"])) == len(F.oracle_pairs(sp["no_filters"]))
    assert len(F.oracle_pairs(sp["no_rgb"])) == len(F.oracle_pairs(sp["no_filters"]))
    # coincident points (d - eps <= 0): segment2 = 0, both orientations rise and fall together with max_angle
    c = sp["coincident_ma90.0"]["cloud"]
    co = {(int(a), int(b)) for a, b in F.oracle_pairs(sp["coincident_nofilter"])}
    assert (0, 2) in co and (2, 0) in co
    assert not {(0, 2), (2, 0)} & {tuple(p) for p in F.oracle_pairs(sp["coincident_ma90.0"]).tolist()}
    assert {(0, 2), (2, 0)} <= {tuple(p) for p in F.oracle_pairs(sp["coincident_ma120.0"]).tolist()}
    assert np.array_equal(c["Q"][0], c["Q"][2])
    # normals: skipped when a square underflows to 0, applied when it is a denormal
    Qn = sp["normals_special_na1.5"]["cloud"]["Qn"]
    kept = {tuple(p) for p in F.oracle_pairs(sp["normals_special_na1.5"]).tolist()}
    names = ("p_zero", "q_zero", "p_underflow", "q_underflow", "p_denormal_sq", "q_denormal_sq", "both_zero")
    for v, name in enumerate(names):
        i, j = 4 * v + 2, 4 * v
        assert F.sqn(Qn[j]) * F.sqn(Qn[i]) == 0 or "denormal" in name
        assert ((j, i) in kept) == ("denormal" not in name), name


def _segment_counts(mutant=None):
    return [len(F.oracle_pairs(case, mutant)) for case in cases("segments")]


@pytest.mark.parametrize("mutant", F.MUTANTS)
def test_each_wrong_decision_changes_a_segment_count(mutant):
    """the GPU batch compares per-segment counts: every mutant of tests/pair_filters changes at least one of them"""
    assert _segment_counts(mutant) != _segment_counts(), mutant


def test_slot_one_reading_slot_zero_base_points_changes_a_count():
    bases = F.batch_bases(cases("segments"), np.zeros((4, 3), np.float32))
    changed = 0
    for b in bases:
        s0, s1 = b["cases"]
        wrong = dict(s1, b1=s0["b1"], b2=s0["b2"])
        changed += len(F.oracle_pairs(wrong)) != len(F.oracle_pairs(s1))
    assert changed > 0


def test_swapping_p_and_q_flips_decisions_in_both_index_orders():
    for order in ("follows", "against"):
        seg = [c for c in cases("segments") if c["probe"].get("filter") == "translation" and c["probe"]["k"] == -1
               and c["probe"]["order"] == order and "mixed" not in c["probe"]]
        assert seg and all(F.probe_bits(c) == 1 and F.probe_bits(c, "trans_swap") == 0 for c in seg)


def test_pair_bits_reference_order():
    """normalized() keeps a zero vector, dot and squared norm are x + (y + z), acosf is glibc's (not numpy's arccos)"""
    z = np.zeros(3, np.float32)
    assert np.array_equal(F.normalized(z), z)
    rng = np.random.RandomState(0)
    a = rng.uniform(-1, 1, (20000, 3)).astype(np.float32)
    b = rng.uniform(-1, 1, (20000, 3)).astype(np.float32)
    left = (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]
    assert (F.dot(a, b) != left).any()
    assert np.array_equal(F.dot(a, a), F.sqn(a))
    # acosf: a float32 result, NaN beyond 1
    x = rng.uniform(-1, 1, 2000).astype(np.float32)
    assert np.array_equal(F.acosf(x), F.acosf(x).astype(np.float32).astype(np.float64))
    assert np.abs(F.acosf(x) - np.arccos(x.astype(np.float64))).max() < 3e-7
    assert np.isnan(F.acosf(E.step(np.float32(1), 1))[()]) and np.isnan(F.acosf(E.step(np.float32(-1), -1))[()])
