"""The point queries' edge fixtures (tests/query_edges.py) and the restatement of their lower bound, checked without a
GPU.

* On every fixture the inequalities of query.cu's header hold in exact arithmetic: the point's exact cell coordinate v
  lies within eps of the cell it is binned in, cell_of's clamps never bind, and cells_bound of every box and row the
  descent can open around the point is at most the fp32 d^2.  How close each family comes is printed (pytest -s).
* Every family is live: each wrong form of the bound drops, on some fixture, a point the brute force takes -- eps = 0,
  eps / 64 (below the worst product rounding at 2000 cells), no (1 - 2^-20) factor, x1 + eps for x1 + 1 + eps, and the
  k-nearest bound taken from the first held entry (replayed by emulate_knn on the tie fixtures).  eps / 4 is still
  sound and drops none.
* The brute forces (oracle/knn.py, range.py, outliers.radius, clusters.roots) agree with one another on every fixture.

Wrong forms that change no answer, so no fixture is built for them:
* __double2float_rn for _rd: the double bound is at most L (1 - 2^-20) - 2^-140 while the fp32 d^2 is at least
  L (1 - 5 * 2^-24); rounding to nearest moves it by 2^-24 relative, which the 2^-20 factor still covers.
* > for >= in the range drop: a box bound equal to sq_radius only drops points with d^2 >= bound = sq_radius, which the
  strict point test d^2 < sq_radius rejects anyway.
* the order of the descent (low half first, or nearer half first): the range lists, radius counts and cluster edges
  are the sets of points with d^2 < sq_radius and the k-nearest row is the lexicographic (d^2, index) minimum -- the
  header's argument fixes each answer independently of the order.
* Family C (the - 2^-140 term deciding a subnormal d^2) is not built: a subnormal d^2 needs cells near 2^-60 wide,
  where s4g_set_cloud_p cannot build its delta-field (test_subnormal_scale_has_no_grid).
"""
import numpy as np
import pytest
from fractions import Fraction as Fr

from oracle import clusters as oclusters
from oracle import knn as oknn
from oracle import outliers as ooutliers
from oracle import range as orange
from tests import edges as E
from tests import query_edges as QE

f32 = np.float32
NAMES = list(QE.REGIMES)


def decided(sc):
    """(family, kind, y, p, d2) of every fixture whose decided point has a finite d^2: the query fixtures and the
    P-to-P pairs (query b, point a)"""
    P = sc["P"]
    out = []
    for q in sc["queries"]:
        if np.isfinite(q["d2"]) and np.isfinite(q["y"]).all():
            out.append((q["family"], q["kind"], q["y"], P[q["j"]], q["d2"], q["radii"]))
    for pr in sc["pairs"]:
        out.append((pr["family"], pr["kind"], P[pr["b"]], P[pr["a"]], pr["d2"], pr["radii"]))
    return out


@pytest.mark.parametrize("name", NAMES)
def test_grid_restatement(name):
    """the host grid is the one context.cu builds: n from the float subtraction equals grid_layout's"""
    _, g = QE.regime_grid(name)
    assert g["n"] == g["n_float_sub"]
    sc = QE.scene(name)
    assert sc["g"]["n"] == g["n"] and sc["g"]["cshift"] == g["cshift"]
    assert [float(a) for a in sc["g"]["o"]] == [float(a) for a in g["o"]]


@pytest.mark.parametrize("name", NAMES)
def test_header_inequalities_hold(name):
    sc = QE.scene(name)
    g = sc["g"]
    eps = Fr(QE.eps_cells(g))
    worst = {}
    for p in sc["P"]:
        for k in range(3):
            c = QE.binned(g, p[k], k)
            assert 0 <= c <= g["n"][k] - 1                       # cell_of's clamp never binds
            v = QE.exact_v(g, p[k], k)
            assert c - eps < v < c + 1 + eps
    for fam, kind, y, p, d2, _ in decided(sc):
        cell = QE.point_cell(g, p)
        cross = max(max(Fr(cell[k]) - QE.exact_v(g, p[k], k), QE.exact_v(g, p[k], k) - Fr(cell[k] + 1))
                    for k in range(3))
        slack = None
        for box in QE.path_boxes(g, cell):
            b = QE.cells_bound(g, y, box)
            assert b <= d2, (fam, kind, box, b, d2)
            if b > 0:
                s = (Fr(float(d2)) - Fr(float(b))) / Fr(float(d2))
                slack = s if slack is None else min(slack, s)
        w = worst.setdefault(fam, [Fr(-1), None])
        w[0] = max(w[0], cross / eps)
        if slack is not None:
            w[1] = slack if w[1] is None else min(w[1], slack)
    for fam in sorted(worst):
        cross, slack = worst[fam]
        print("%s %s: binned %.3f eps across a face at most; tightest bound %s below fp32 d^2" % (
            name, fam, float(max(cross, 0)), "-" if slack is None else "%.3g x 2^-20" % (float(slack) * 2 ** 20)))


def test_families_are_built():
    """family A (and F, G on it) in every regime where a float lands within the product's or the subtraction's
    rounding of a face; downward crossings where p - o rounds near the top faces (widened, brick8).  In offcentre1e4
    the coordinates' lattice is 1/16 cell and p - o is exact: no float is binned across any face there."""
    for name in NAMES:
        sc = QE.scene(name)
        kinds = {q["kind"] for q in sc["queries"] if q["family"] == "A"}
        fams = {q["family"] for q in sc["queries"]} | {p["family"] for p in sc["pairs"]}
        assert {"B", "D", "E"} <= fams
        if name == "offcentre1e4":
            assert not kinds
            continue
        assert {"A", "F", "G"} <= fams, name
        assert any("-up-" in k for k in kinds), name
        if name in ("widened", "brick8"):   # p - o rounds near their top faces; elsewhere it is exact there
            assert any("-down-" in k for k in kinds), name
        for axis in range(3):
            assert any(k.split("-")[1] == str(axis) for k in kinds), (name, axis)
        for kind in ("box", "row", "both"):
            assert any(k.startswith(kind) for k in kinds), (name, kind)
        assert any(q["T"] for q in sc["queries"] if q["family"] == "A")


def test_subnormal_scale_has_no_grid():
    """family C: a cloud at 2^-60 whose d^2 are subnormal.  The delta-field built with the grid needs a voxel radius
    R = ceil(1 + reach / v) that does not fit an int there (reach carries an absolute 8 x 2^-20), so s4g_set_cloud_p
    cannot build it.  At any scale it can build, subnormal distances are far inside one cell, where the bound is 0."""
    P = (np.array([[1, 1, 1], [1.5, 1.25, 1.75], [1.9, 1.3, 1.1]]) * 2.0 ** -60).astype(f32)
    assert QE.field_reach_voxels(P, 2.0 ** -70) > 2.0 ** 31


def _mutant_flips(variant):
    """(family, regime, kind) of the fixtures where a form of the bound drops the decided point at a radius where the
    brute force takes it (range: d^2 < r, bound >= r; k-nearest with a row that is not full: d^2 <= r, bound > r)"""
    out = []
    for name in NAMES:
        sc = QE.scene(name)
        g = sc["g"]
        for fam, kind, y, p, d2, radii in decided(sc):
            for r in radii:
                if (d2 < r and QE.drops(g, y, p, r, True, **variant)) or \
                        (d2 <= r and QE.drops(g, y, p, r, False, **variant)):
                    out.append((fam, name, kind))
                    break
    return out


@pytest.mark.parametrize("mutant", list(QE.MUTANTS))
def test_wrong_bound_drops_a_taken_point(mutant):
    flips = _mutant_flips(QE.MUTANTS[mutant])
    by = {}
    for fam, name, _ in flips:
        by.setdefault(fam, set()).add(name)
    print(mutant, {f: sorted(v) for f, v in sorted(by.items())})
    assert flips, mutant
    if mutant in ("eps=0", "eps/64"):
        assert "widened" in by.get("A", ())
    if mutant == "no (1 - 2^-20)":
        assert "B" in by


def test_sound_variant_drops_nothing():
    for v in QE.SOUND_VARIANTS.values():
        assert _mutant_flips(v) == []


def _tie_rows(name, bound_from):
    sc = QE.scene(name)
    P, g = sc["P"], sc["g"]
    out = []
    for q in sc["queries"]:
        if q["family"] != "E":
            continue
        for k in q["ks"]:
            for r in q["radii"]:
                out.append(((q["kind"], q["T"], k, float(r)),
                            QE.emulate_knn(g, P, q["y"], k, r, q["exclude"], bound_from=bound_from)))
    return out


@pytest.mark.parametrize("name", NAMES)
def test_tie_emulation_equals_the_brute_force(name):
    """the replayed k-nearest descent returns the brute force's rows on the tie fixtures; the tie at the k-th entry
    is resolved to the smaller index although the larger one is found first"""
    sc = QE.scene(name)
    T16 = E.colmajor(sc["T34"])[0]
    rows = dict(_tie_rows(name, "kth"))
    for q in sc["queries"]:
        if q["family"] != "E":
            continue
        for k in q["ks"]:
            for r in q["radii"]:
                want = oknn.bruteforce(sc["P"], q["x"][None], k, r, T16 if q["T"] else None,
                                       np.array([q["exclude"]], np.int32))
                got = rows[(q["kind"], q["T"], k, float(r))]
                assert np.array_equal(got[0], want[0][0]) and np.array_equal(got[1].view(np.uint32),
                                                                              want[1][0].view(np.uint32))
        if q["exclude"] == -1:
            row = oknn.bruteforce(sc["P"], q["x"][None], 3, np.inf, T16 if q["T"] else None)[0][0]
            assert row[2] == q["j"]                              # the k-th entry at k = 3 is the smaller tied index


def test_first_held_bound_loses_a_tie():
    """the k-nearest bound taken from the first held entry instead of the k-th drops the smaller tied index"""
    differ = []
    for name in NAMES:
        kth, first = _tie_rows(name, "kth"), _tie_rows(name, "first")
        differ += [(name, a[0]) for a, b in zip(kth, first) if not np.array_equal(a[1][0], b[1][0])]
    assert differ


@pytest.mark.parametrize("name", NAMES)
def test_brute_forces_agree(name):
    sc = QE.scene(name)
    P = sc["P"]
    T16 = E.colmajor(sc["T34"])[0]
    for q in sc["queries"]:
        T = T16 if q["T"] else None
        ex = np.array([q["exclude"]], np.int32)
        for r in q["radii"]:
            want = oknn.bruteforce(P, q["x"][None], 64, r, T, ex)
            lists = orange.bruteforce(P, q["x"][None], oknn.range_radius(r), T)
            got = oknn.from_range(lists, 64, ex)
            # a range list cannot hold d^2 = +inf (its test is strict): at sq_radius = +inf it is the finite prefix
            m = int(np.isfinite(want[1]).sum()) if r == np.inf else 64
            assert np.array_equal(want[0][:, :m], got[0][:, :m]), (q["family"], q["kind"], r)
            assert np.array_equal(want[1][:, :m].view(np.uint32), got[1][:, :m].view(np.uint32))
            assert (got[0][:, m:] == -1).all()
    for pr in sc["pairs"]:
        for r in pr["radii"]:
            off, idx, _ = orange.bruteforce(P, P, r)
            _, counts, raw = ooutliers.radius(P, r, len(P), raw=True)
            assert np.array_equal(raw, np.diff(off) - (r > 0))    # each list holds the point itself when r > 0
            keep = idx != np.repeat(np.arange(len(P)), np.diff(off))
            own = np.concatenate([[0], np.cumsum(keep)])[off]
            assert np.array_equal(oclusters.roots(P, r), oclusters.roots_from_lists(len(P), own, idx[keep]))
            d2 = QE.d2_f32(P[pr["b"]], P[pr["a"]])
            assert (d2 < r) == (oclusters.roots(P, r)[pr["b"]] == oclusters.roots(P, r)[pr["a"]])
