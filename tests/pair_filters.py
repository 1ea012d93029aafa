"""The pair query's four filters at the floats where they flip, and an oracle of the whole predicate that shares no code
with oracle/port.cc.

After the unit-cube point test and the distance band (tests/edges.py), PairCreationFunctor::process (reference
pairCreationFunctor.h:165-212) takes four threshold decisions, each of which a single float can flip:

* normal      : nd = float(min(|fl|qn - pn|| - pna|, |fl|qn + pn|| - pna|)) in double, rejected when nd > norm_threshold;
                skipped when either normal has a squared norm of 0;
* colour      : |pc - b1_rgb| < max_color_distance and |qc - b2_rgb| < max_color_distance, only when all four rgb[0] >= 0;
* translation : |p - b1| < max_translation_distance and |q - b2| < max_translation_distance, p the point with the SMALLER
                original index;
* angle       : acosf(dt) <= max_angle * pi / 180 for dt = segment1 . segment2 and for -dt (one bit per orientation).

`pair_bits` restates all of it in numpy: float32 operations in the reference's order (x^2 + (y^2 + z^2), a zero vector
normalizes to itself), the normal distance in double, glibc's acosf through ctypes.  `mutant=` switches one decision to a
plausible wrong form, so that the tests can show which inputs tell each wrong form apart.

The builders put one designed pair at exactly 0, +-1 and +-2 floats from each threshold while every other filter passes
clearly and the pair's distance lies well inside the band.  Every cloud is its points interleaved with their negations,
so its float sum is exactly 0 and the reference's centring leaves it bit-identical.
"""
import ctypes
import math

import numpy as np

from tests import edges as E

f32 = np.float32
KS = E.KS
D, EPS = 0.5, 0.05                        # distance band of the designed pairs
FILTERS = (20.0, 0.75, 60.0, 0.3)         # (max_normal_difference, max_translation_distance, max_angle, max_color_distance)
MAX_ANGLES = (1e-3, 30.0, 60.0, 90.0, 179.9, 180.0, 200.0)
MUTANTS = ("norm_ge", "norm_first_only", "color_le", "trans_le", "trans_swap", "angle_gt", "angle_no_le1",
           "cos_up", "cos_down", "rgb_ign_p", "rgb_ign_q", "rgb_ign_b1", "rgb_ign_b2")

_libm = ctypes.CDLL("libm.so.6")
_libm.acosf.restype = ctypes.c_float
_libm.acosf.argtypes = [ctypes.c_float]


def acosf(x):
    """glibc's acosf of every element (float32 in, float64 out: the reference compares it with a double)"""
    x = np.asarray(x, f32)
    u, inv = np.unique(x, return_inverse=True)
    v = np.array([_libm.acosf(float(t)) for t in u], np.float64)
    return v[inv].reshape(x.shape)


def angle_threshold(max_angle):
    return float(f32(max_angle)) * math.pi / 180.0


def cos_angle_min(max_angle):
    """smallest float32 x in [-1, 1] with acosf(x) <= max_angle * pi / 180 (2.0 if none), by bisection over the floats"""
    thr = angle_threshold(max_angle)
    ok = lambda x: acosf(x)[()] <= thr  # noqa: E731
    if not ok(f32(1)):
        return f32(2)
    if ok(f32(-1)):
        return f32(-1)
    lo, hi = int(E.ordinal(f32(-1))), int(E.ordinal(f32(1)))
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if ok(E.from_ordinal(mid)):
            hi = mid
        else:
            lo = mid
    return f32(E.from_ordinal(hi))


# ---- float32 vector arithmetic in the reference's order ---------------------------------------------------------------
def sqn(v):
    v = np.asarray(v, f32)
    return v[..., 0] * v[..., 0] + (v[..., 1] * v[..., 1] + v[..., 2] * v[..., 2])


def norm(v):
    return np.sqrt(sqn(v))


def dot(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return a[..., 0] * b[..., 0] + (a[..., 1] * b[..., 1] + a[..., 2] * b[..., 2])


def normalized(v):
    v = np.asarray(v, f32)
    z = sqn(v)
    s = np.where(z > 0, np.sqrt(z), f32(1))
    return np.where((z > 0)[..., None], v / s[..., None], v).astype(f32)


# ---- the oracle -------------------------------------------------------------------------------------------------------
def band_pairs(Q, d, eps):
    """(I, J), I > J: the unordered pairs that pass the unit-cube point test and the distance band"""
    Q = np.asarray(Q, f32)
    n = len(Q)
    gc, ratio, nR, er2 = E.pair_params(Q, d, eps)
    U = ((Q - gc) / ratio) + f32(0.5)
    Is, Js = [], []
    for s in range(0, n, 512):
        i = np.arange(s, min(n, s + 512))
        un = norm(U[None, :, :] - U[i, None, :]) - nR
        dist = norm(Q[i, None, :] - Q[None, :, :])
        ok = (un * un < er2) & (np.abs(dist.astype(np.float64) - float(f32(d))) <= float(f32(eps)))
        ok &= np.arange(n)[None, :] < i[:, None]
        a, b = np.nonzero(ok)
        Is.append(i[a])
        Js.append(b)
    if not Is:
        return np.zeros(0, np.int64), np.zeros(0, np.int64)
    return np.concatenate(Is).astype(np.int64), np.concatenate(Js).astype(np.int64)


def pair_bits(Q, Qn, Qrgb, d, na, eps, b1, b2, filters, mutant=None):
    """(I, J, r): every unordered pair I > J the predicate keeps, with its orientation bits r (bit 0: (J, I), bit 1:
    (I, J)).  Qn / Qrgb None: zero normals / rgb -1, as when none are uploaded.  b1, b2: 9 floats (pos, normal, rgb)."""
    Q = np.asarray(Q, f32)
    I, J = band_pairs(Q, d, eps)
    b1, b2 = np.asarray(b1, f32).reshape(9), np.asarray(b2, f32).reshape(9)
    mnd, mtd, ma, mcd = (f32(x) for x in filters)
    keep = np.ones(len(I), bool)
    p, q = Q[J], Q[I]
    if mnd > 0:
        Qn_ = np.zeros_like(Q) if Qn is None else np.asarray(Qn, f32)
        pn, qn = Qn_[J], Qn_[I]
        applies = (sqn(qn) > 0) & (sqn(pn) > 0)
        thr = f32(0.5 * float(mnd) * math.pi / 180.0)
        pna = float(f32(na))
        first = np.abs(norm(qn - pn).astype(np.float64) - pna)
        second = np.abs(norm(qn + pn).astype(np.float64) - pna)
        nd = (first if mutant == "norm_first_only" else np.minimum(first, second)).astype(f32)
        bad = (nd >= thr) if mutant == "norm_ge" else (nd > thr)
        keep &= ~(applies & bad)
    if mcd > 0:
        rgb = -np.ones_like(Q) if Qrgb is None else np.asarray(Qrgb, f32)
        pc, qc = rgb[J], rgb[I]
        conds = {"p": pc[:, 0] >= 0, "q": qc[:, 0] >= 0, "b1": np.full(len(I), b1[6] >= 0), "b2": np.full(len(I), b2[6] >= 0)}
        use = np.ones(len(I), bool)
        for k, c in conds.items():
            if mutant != "rgb_ign_" + k:
                use &= c
        lt = (lambda a: a <= mcd) if mutant == "color_le" else (lambda a: a < mcd)
        good = lt(norm(pc - b1[6:9])) & lt(norm(qc - b2[6:9]))
        keep &= ~(use & ~good)
    if mtd > 0:
        pp, qq = (q, p) if mutant == "trans_swap" else (p, q)
        lt = (lambda a: a <= mtd) if mutant == "trans_le" else (lambda a: a < mtd)
        keep &= lt(norm(pp - b1[:3])) & lt(norm(qq - b2[:3]))
    r = np.full(len(I), 3, np.int64)
    if ma > 0:
        seg1 = normalized(b2[:3] - b1[:3])
        seg2 = normalized(q - p)
        dt, dtn = dot(seg1[None], seg2), dot(seg1[None], -seg2)
        if mutant in ("angle_gt", "angle_no_le1", "cos_up", "cos_down"):
            c = cos_angle_min(ma)
            c = E.step(c, 1) if mutant == "cos_up" else E.step(c, -1) if mutant == "cos_down" else c
            ge = (lambda x: x > c) if mutant == "angle_gt" else (lambda x: x >= c)
            le1 = (lambda x: np.ones(x.shape, bool)) if mutant == "angle_no_le1" else (lambda x: x <= f32(1))
            b0, bb1 = ge(dt) & le1(dt), ge(dtn) & le1(dtn)
        else:
            thr = angle_threshold(ma)
            b0, bb1 = acosf(dt) <= thr, acosf(dtn) <= thr
        r = b0.astype(np.int64) | (bb1.astype(np.int64) << 1)
    keep &= r != 0
    return I[keep], J[keep], r[keep]


def ordered(I, J, r):
    """sorted ordered pairs of pair_bits' output"""
    a = np.concatenate([np.stack([J[(r & 1) != 0], I[(r & 1) != 0]], 1), np.stack([I[(r & 2) != 0], J[(r & 2) != 0]], 1)])
    a = a.astype(np.int32).reshape(-1, 2)
    return a[np.lexsort((a[:, 1], a[:, 0]))]


def oracle_pairs(case, mutant=None):
    c = case["cloud"]
    return ordered(*pair_bits(c["Q"], c["Qn"], c["Qrgb"], case["d"], case["na"], case["eps"], case["b1"], case["b2"],
                              case["filters"], mutant))


def probe_bits(case, mutant=None):
    """orientation bits of the case's designed pair (0 if it is not kept)"""
    c = case["cloud"]
    I, J, r = pair_bits(c["Q"], c["Qn"], c["Qrgb"], case["d"], case["na"], case["eps"], case["b1"], case["b2"],
                        case["filters"], mutant)
    i, j = case["probe"]["pair"]
    hit = (I == i) & (J == j)
    return int(r[hit][0]) if hit.any() else 0


# ---- clouds -----------------------------------------------------------------------------------------------------------
def mirrored(pts, nrm=None, rgb=None):
    """pts interleaved with their negations (point m at index 2m, -point m at 2m + 1): the float sum of every coordinate
    is exactly 0, so the reference's centring moves nothing"""
    pts = np.asarray(pts, f32)
    Q = np.empty((2 * len(pts), 3), f32)
    Q[0::2], Q[1::2] = pts, -pts
    out = dict(Q=Q, Qn=None, Qrgb=None)
    if nrm is not None:
        out["Qn"] = np.repeat(np.asarray(nrm, f32), 2, axis=0)
    if rgb is not None:
        out["Qrgb"] = np.repeat(np.asarray(rgb, f32), 2, axis=0)
    return out


def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v)


def norm_threshold(mnd=FILTERS[0]):
    return f32(0.5 * float(f32(mnd)) * math.pi / 180.0)


def _normal_pair(opposite, scale=1.0):
    """(pn, qn): float32 normals with fl|qn - pn| (or, opposite, fl|qn + pn|) about 1.05 norm_threshold"""
    a = 2 * math.asin(0.525 * float(norm_threshold()) / scale)
    u = np.array([0.0, 0.6, 0.8])
    w = np.array([0.0, 0.6 * math.cos(a) - 0.8 * math.sin(a), 0.6 * math.sin(a) + 0.8 * math.cos(a)])
    pn, qn = (scale * u).astype(f32), (scale * w).astype(f32)
    return pn, (-qn if opposite else qn)


# the sites of the designed pairs: (index order, normals, rgb of p, rgb of q).  'follows': the point at the lower position
# has the smaller index (it is p); 'against': the other way round.
SITES = (("follows", "parallel", None, None), ("against", "parallel", None, None),
         ("follows", "opposite", None, None), ("against", "opposite", None, None),
         ("follows", "parallel", -1.0, None), ("against", "parallel", None, -1.0),
         ("follows", "parallel", -0.0, None), ("against", "parallel", None, float("nan")))
RGB0 = (0.5, 0.5, 0.5)


def filter_cloud():
    """the designed pairs (A, B = A + v, |v| = D) of SITES, mirrored; per site the indices (p, q) by original index"""
    pts, nrm, rgb, sites = [], [], [], []
    for k, (order, nkind, prgb, qrgb) in enumerate(SITES):
        A = np.array([0.3 + 0.9 * (k % 3), 0.3 + 0.9 * (k // 3), 0.3], f32)
        v = (D * _unit([0.8, 0.6, 0.04 * (k + 1)])).astype(f32)
        B = (A + v).astype(f32)
        pn, qn = _normal_pair(nkind == "opposite")
        pc, qc = np.array(RGB0, f32), np.array(RGB0, f32)
        if prgb is not None:
            pc[0] = prgb
        if qrgb is not None:
            qc[0] = qrgb
        first, second = (A, B) if order == "follows" else (B, A)     # first gets the smaller index: it is p
        m = len(pts)
        pts += [first, second]
        nrm += [pn, qn]
        rgb += [pc, qc]
        sites.append(dict(order=order, normals=nkind, p=2 * m, q=2 * (m + 1)))
    # one more pair whose fl(normalized(B - A) . normalized(B - A)) > 1: with b1 = A, b2 = B only dt <= 1 rejects it
    A = np.array([0.3 + 0.9 * 2, 0.3 + 0.9 * 2, 0.3], f32)
    rng = np.random.RandomState(3)
    while True:
        B = (A + (D * _unit(rng.uniform(0.1, 1, 3))).astype(f32)).astype(f32)
        if dot(normalized(B - A), normalized(B - A)) > 1:
            break
    m = len(pts)
    pts += [A, B]
    nrm += list(_normal_pair(False))
    rgb += [np.array(RGB0, f32)] * 2
    sites.append(dict(order="follows", normals="parallel", p=2 * m, q=2 * (m + 1), dt_above_one=True))
    c = mirrored(pts, nrm, rgb)
    c["sites"] = sites
    c["name"] = "filter_cloud"
    return c


def b9(pos, rgb=RGB0):
    return np.concatenate([np.asarray(pos, f32), np.zeros(3, f32), np.asarray(rgb, f32)]).astype(f32)


def _pna_exact(branch_value, target):
    """pna with |branch_value - pna| == target exactly (in double, so nd == target)"""
    pna = f32(float(branch_value) - float(target))
    assert float(branch_value) - float(pna) == float(target), "pna not exact"
    return pna


def _branches(c, site):
    pn, qn = c["Qn"][site["p"]], c["Qn"][site["q"]]
    return norm(qn - pn), norm(qn + pn)


def default_segment(c, site, filters=FILTERS):
    """a segment in which the site's pair passes every filter clearly and emits (p, q) only (bit 0)"""
    p, q = c["Q"][site["p"]], c["Q"][site["q"]]
    first, second = _branches(c, site)
    na = first if site["normals"] == "parallel" else second          # nd = 0
    b1 = b9((p + f32(0) + np.array([0, 0, 0.1], f32)).astype(f32), (0.45, 0.5, 0.5))
    b2 = b9((q + np.array([0, 0.02, 0.1], f32)).astype(f32), (0.45, 0.5, 0.5))
    return dict(cloud=c, d=D, eps=EPS, na=f32(na), b1=b1, b2=b2, filters=tuple(filters),
                probe=dict(pair=(site["q"], site["p"]), bit=1))


def _exact_offset(x0, t, sign):
    """x1 = x0 - sign * t with fl(x0 - x1) == sign * t exactly"""
    x1 = f32(x0 - f32(sign * t))
    assert f32(x0 - x1) == f32(sign * t), "offset not exact"
    return x1


def search_at_distance(c, u, target, side=12):
    """x near c + target * u with fl|c - x| == target"""
    c = np.asarray(c, f32)
    start = (c.astype(np.float64) + float(target) * _unit(u)).astype(f32)
    o = np.arange(-side, side + 1)
    g = np.meshgrid(o, o, o, indexing="ij")
    T = np.stack([E.step(start[i], g[i].ravel()) for i in range(3)], 1).astype(f32)
    hit = np.nonzero(norm(c[None] - T) == f32(target))[0]
    assert len(hit), "distance target not reached"
    dev = np.abs(g[0].ravel()) + np.abs(g[1].ravel()) + np.abs(g[2].ravel())
    return T[hit[np.argmin(dev[hit])]]


def search_b2(b1, seg2, target_dt, length, start=None, side=16):
    """b2 near b1 + length * dir with fl(segment1 . seg2) == target_dt, segment1 = normalized(b2 - b1); None if no float
    neighbour of the start reaches it"""
    seg2d = np.asarray(seg2, np.float64)
    e = _unit(np.cross(seg2d, [0.3, -0.5, 0.8]))
    th = math.acos(max(-1.0, min(1.0, float(target_dt))))
    b1 = np.asarray(b1, f32)
    if start is None:
        start = (b1.astype(np.float64) + length * (math.cos(th) * _unit(seg2d) + math.sin(th) * e)).astype(f32)
    o = np.arange(-side, side + 1)
    g = np.meshgrid(o, o, o, indexing="ij")
    T = np.stack([E.step(start[i], g[i].ravel()) for i in range(3)], 1).astype(f32)
    dt = dot(normalized(T - b1[None]), np.asarray(seg2, f32)[None])
    hit = np.nonzero(dt == f32(target_dt))[0]
    if not len(hit):
        return None
    dev = np.abs(g[0].ravel()) + np.abs(g[1].ravel()) + np.abs(g[2].ravel())
    return T[hit[np.argmin(dev[hit])]]


def segment_cases(c=None):
    """one extraction per case on filter_cloud(), all four filters on; each case's probe is the designed pair it puts
    at a threshold: dict(filter, side, k, order, pair, bit)"""
    c = filter_cloud() if c is None else c
    mnd, mtd, ma, mcd = FILTERS
    out = []

    def add(seg, filt, side, k, site, bit=1, name=None):
        seg["probe"].update(filter=filt, side=side, k=k, order=site["order"], bit=bit)
        seg["name"] = name or "%s-%s-%s-k%+d" % (filt, side, site["order"], k)
        out.append(seg)

    for site in c["sites"][:2]:
        p, q = c["Q"][site["p"]], c["Q"][site["q"]]
        away = _unit(p.astype(np.float64) - q)     # swapping p and q puts the other point D + x from the base point
        for k in KS:
            x = E.step(f32(mtd), k)
            s = default_segment(c, site)            # |p - b1| = x on the far side of p from q
            s["b1"][:3] = search_at_distance(p, away, x)
            add(s, "translation", "p", k, site)
            s = default_segment(c, site)            # |q - b2| = x on the far side of q from p
            s["b2"][:3] = search_at_distance(q, -away, x)
            add(s, "translation", "q", k, site)
            y = E.step(f32(mcd), k)                 # |pc - b1_rgb| = y (and |qc - b2_rgb|)
            for side, row, pt in (("p", "b1", site["p"]), ("q", "b2", site["q"])):
                s = default_segment(c, site)
                col = c["Qrgb"][pt]
                s[row][6] = _exact_offset(col[0], y, 1.0)
                assert norm(col - s[row][6:9]) == y
                add(s, "colour", side, k, site)
    thr = norm_threshold(mnd)
    for site in c["sites"][:4]:
        first, second = _branches(c, site)
        branch = "first" if site["normals"] == "parallel" else "second"
        for k in KS:
            s = default_segment(c, site)
            s["na"] = _pna_exact(first if branch == "first" else second, E.step(thr, k))
            add(s, "normal", branch, k, site)
    cmin = cos_angle_min(ma)
    for site in c["sites"][:2]:
        p, q = c["Q"][site["p"]], c["Q"][site["q"]]
        seg2 = normalized(q - p)
        for bit, sign, length in ((1, 1, D), (2, -1, 0.2)):
            for k in KS:
                s = default_segment(c, site)
                b2 = search_b2(s["b1"][:3], seg2, f32(sign * E.step(cmin, k)), length)
                assert b2 is not None, ("angle target not reached", bit, k)
                s["b2"][:3] = b2
                add(s, "angle", "bit%d" % (bit - 1), k, site, bit=bit)
    site = c["sites"][8]                             # angle 0 and fl(dt) > 1: acosf(dt) is NaN
    s = default_segment(c, site)
    s["b1"][:3], s["b2"][:3] = c["Q"][site["p"]], c["Q"][site["q"]]
    add(s, "angle_dt_above_one", "bit0", 0, site, name="angle-dt-above-one")
    # use_rgb: the colour test fails clearly on both sides (rgb distance 0.5), so only use_rgb decides
    for site in c["sites"][4:8]:
        s = default_segment(c, site)
        s["b1"][6:9], s["b2"][6:9] = (0.0, 0.5, 0.5), (0.0, 0.5, 0.5)
        add(s, "use_rgb", "point", 0, site, name="use_rgb-point%d" % c["sites"].index(site))
    site = c["sites"][0]
    for row in ("b1", "b2"):
        for v in (-1.0, -0.0, float("nan")):
            s = default_segment(c, site)
            s["b1"][6:9], s["b2"][6:9] = (0.0, 0.5, 0.5), (0.0, 0.5, 0.5)
            s[row][6] = v
            add(s, "use_rgb", row, 0, site, name="use_rgb-%s-%r" % (row, v))
    # mixed: one filter at its edge, another clearly failing (the pair is rejected at every k) or clearly passing
    for k in (-1, 0):
        for fail in ("colour", "normal", None):
            base = [x for x in out if x["probe"]["filter"] == "translation" and x["probe"]["side"] == "p"
                    and x["probe"]["k"] == k and x["probe"]["order"] == "follows"][0]
            s = dict(base, b1=base["b1"].copy(), b2=base["b2"].copy(), probe=dict(base["probe"]))
            if fail == "colour":
                s["b2"][6:9] = (0.0, 0.5, 0.5)
            elif fail == "normal":
                s["na"] = f32(s["na"] + f32(0.5))
            s["name"] = "mixed-translation-k%+d-%s" % (k, fail or "colour_edge")
            if fail is None:                        # the colour test at its edge too, on the passing side (k = -1)
                s["b1"][6] = _exact_offset(RGB0[0], E.step(f32(mcd), -1), 1.0)
            s["probe"]["mixed"] = fail
            out.append(s)
    return out


# ---- one-base cases beyond the shared cloud ---------------------------------------------------------------------------
def angle_sweep_cases():
    """max_angle over MAX_ANGLES (translation, colour, normal filters off): dt and -dt at 0, +-1, +-2 floats from
    cos_angle_min, where such a dt exists"""
    c = filter_cloud()
    out = []
    for ma in MAX_ANGLES:
        cmin = cos_angle_min(ma)
        for site in c["sites"][:2]:
            p, q = c["Q"][site["p"]], c["Q"][site["q"]]
            seg2 = normalized(q - p)
            for bit, sign in ((1, 1), (2, -1)):
                for k in KS:
                    t = E.step(cmin, k)
                    if abs(float(t)) > 1:
                        continue
                    s = default_segment(c, site, filters=(-1.0, -1.0, ma, -1.0))
                    b2 = search_b2(s["b1"][:3], seg2, f32(sign * t), D)
                    if b2 is None:
                        continue
                    s["b2"][:3] = b2
                    s["probe"].update(filter="angle%g" % ma, side="bit%d" % (bit - 1), k=k, order=site["order"], bit=bit)
                    s["name"] = "angle%g-bit%d-%s-k%+d" % (ma, bit - 1, site["order"], k)
                    out.append(s)
    # near 90 degrees cos_angle_min is tiny and a general dot product cannot land on its neighbours: a pair along x
    # (segment2 = +-x exactly) and segment1 = normalized((t, 1, 0)) = (t, 1, 0), so dt = t exactly
    A = np.array([0.3, 1.2, 0.3], f32)
    ax = mirrored([A, (A + np.array([D, 0, 0], f32)).astype(f32)])
    ax["name"] = "axis_pair"
    for ma in MAX_ANGLES:
        cmin = cos_angle_min(ma)
        if not 0 < abs(float(cmin)) < 2.0 ** -12:
            continue
        for bit, (i, j) in ((1, (2, 0)), (2, (3, 1))):          # the mirror pair points along -x: its -dt is t
            for k in KS:
                t = E.step(cmin, k)
                b2 = np.array([t, 1, 0], f32)
                assert np.array_equal(normalized(b2), b2)
                s = dict(cloud=ax, d=D, eps=EPS, na=f32(0), b1=b9([0, 0, 0]), b2=b9(b2), filters=(-1.0, -1.0, ma, -1.0),
                         probe=dict(pair=(i, j), bit=bit, filter="angle%g" % ma, side="bit%d" % (bit - 1), k=k, order="axis"),
                         name="angle%g-bit%d-axis-k%+d" % (ma, bit - 1, k))
                out.append(s)
    return out


def _dot_self_cloud():
    """pairs (p, q) whose fl(normalized(q - p) . normalized(q - p)) is > 1 and == 1: with b1 = p and b2 = q the angle
    is 0 and only dt <= 1 (acosf of a dt > 1 is NaN) decides"""
    rng = np.random.RandomState(5)
    found = {}
    pts, kinds = [], []
    for k, key in enumerate(("gt1", "eq1")):
        A = np.array([0.4 + 1.1 * k, 0.5, 0.3], f32)
        while True:
            B = (A + (D * _unit(rng.standard_normal(3))).astype(f32)).astype(f32)
            u = normalized(B - A)
            if (dot(u, u) > 1) == (key == "gt1") and (dot(u, u) == 1) == (key == "eq1"):
                break
        pts += [A, B]
        kinds.append(key)
    c = mirrored(pts)
    c["name"] = "dot_self"
    c["kinds"] = kinds
    return c


def special_cases():
    """the angle filter's corners, the normal filter's skipped and non-unit normals, the colour filter without rgb and
    filters off: dict(cloud, d, eps, na, b1, b2, filters, name)"""
    out = []

    def case(c, name, filters, b1, b2, na=0.0, d=D, eps=EPS, probe=None):
        out.append(dict(cloud=c, name=name, d=d, eps=eps, na=f32(na), b1=np.asarray(b1, f32), b2=np.asarray(b2, f32),
                        filters=tuple(filters), probe=probe))

    c = _dot_self_cloud()
    for k, key in enumerate(c["kinds"]):
        p, q = c["Q"][4 * k], c["Q"][4 * k + 2]
        for ma in (30.0, 1e-3, 1e-20):
            case(c, "dt_self_%s_ma%g" % (key, ma), (-1, -1, ma, -1), b9(p), b9(q), probe=dict(pair=(4 * k + 2, 4 * k), bit=1))
    fc = filter_cloud()
    p0 = fc["Q"][fc["sites"][0]["p"]]
    for ma in (60.0, 90.0, float(E.step(f32(90), 1)), 120.0, 200.0):
        case(fc, "b1_eq_b2_ma%r" % ma, (-1, -1, ma, -1), b9(p0), b9(p0))
    case(fc, "max_angle_0", (-1, -1, 0.0, -1), b9(p0), b9(fc["Q"][fc["sites"][0]["q"]]))
    # coincident pair points: d - eps <= 0, segment2 = 0
    A = np.array([0.6, 0.4, 0.3], f32)
    cc = mirrored([A, A, A, (A + np.array([0.01, 0, 0], f32)).astype(f32)])
    cc["name"] = "coincident"
    for ma in (60.0, 90.0, float(E.step(f32(90), 1)), 120.0):
        case(cc, "coincident_ma%r" % ma, (-1, -1, ma, -1), b9(A), b9(A + np.array([0.3, 0.1, 0], f32)), d=0.02, eps=0.05)
    case(cc, "coincident_nofilter", (-1, -1, -1, -1), b9(A), b9(A), d=0.02, eps=0.05)
    # normals: zero or underflowing squares in either point (skipped), a denormal square (applied), non-unit normals
    pn, qn = _normal_pair(False)
    tiny, sub = f32(1e-25), f32(1e-20)
    variants = (("p_zero", np.zeros(3, f32), qn), ("q_zero", pn, np.zeros(3, f32)),
                ("p_underflow", np.array([tiny, tiny, 0], f32), qn), ("q_underflow", pn, np.array([0, tiny, tiny], f32)),
                ("p_denormal_sq", np.array([sub, 0, 0], f32), qn), ("q_denormal_sq", pn, np.array([0, 0, sub], f32)),
                ("both_zero", np.zeros(3, f32), np.zeros(3, f32)))
    pts, nrm = [], []
    for k, (_, a, b) in enumerate(variants):
        A = np.array([0.3 + 0.9 * (k % 4), 0.3 + 0.9 * (k // 4), 0.3], f32)
        pts += [A, (A + (D * _unit([0.8, 0.6, 0.1])).astype(f32)).astype(f32)]
        nrm += [a, b]
    # non-unit normals at the threshold (both branches)
    for k, opp in enumerate((False, True)):
        A = np.array([0.3 + 0.9 * k, 2.1, 0.3], f32)
        pts += [A, (A + (D * _unit([0.8, 0.6, 0.1])).astype(f32)).astype(f32)]
        nrm += list(_normal_pair(opp, scale=3.0))
    nc = mirrored(pts, nrm)
    nc["name"] = "normals"
    far = b9([9, 9, 9])
    for na in (0.0, 1.0, 1.5):
        case(nc, "normals_special_na%g" % na, (FILTERS[0], -1, -1, -1), far, far, na=na)
    thr = norm_threshold()
    m = len(variants)
    for k, opp in enumerate((False, True)):
        i, j = 2 * (2 * (m + k) + 1), 2 * (2 * (m + k))
        first, second = norm(nc["Qn"][i] - nc["Qn"][j]), norm(nc["Qn"][i] + nc["Qn"][j])
        for kk in KS:
            na = _pna_exact(second if opp else first, E.step(thr, kk))
            case(nc, "normals_nonunit_%s_k%+d" % ("second" if opp else "first", kk), (FILTERS[0], -1, -1, -1), far, far,
                 na=na, probe=dict(pair=(i, j), bit=3, filter="normal_nonunit", side="second" if opp else "first", k=kk))
    # no normals / no rgb uploaded: those filters pass everything
    nn = dict(fc, Qn=None, name="filter_cloud_no_normals")
    case(nn, "no_normals", (FILTERS[0], -1, -1, -1), far, far, na=1.5)
    nr = dict(fc, Qrgb=None, name="filter_cloud_no_rgb")
    case(nr, "no_rgb", (-1, -1, -1, FILTERS[3]), b9([0, 0, 0], (0.0, 0.0, 0.0)), b9([0, 0, 0], (0.0, 0.0, 0.0)))
    case(fc, "no_filters", (-1, -1, -1, -1), far, far)
    return out


# ---- the batch --------------------------------------------------------------------------------------------------------
def batch_bases(cases, P):
    """the segment cases two by two as the bases of one s4g_try_bases call: slot s of base b is case 2b + s, each with
    its own b1 / b2 positions and rgb and its own normal angle; base_xyz_p = four points of P"""
    bases = []
    for b in range(0, len(cases) - 1, 2):
        s0, s1 = cases[b], cases[b + 1]
        b9s = np.stack([s0["b1"], s0["b2"], s1["b1"], s1["b2"]]).astype(f32)
        ids = np.arange(4 * (b // 2), 4 * (b // 2) + 4) % len(P)
        bases.append(dict(d1=s0["d"], d2=s1["d"], na1=float(s0["na"]), na2=float(s1["na"]), b9=b9s, bxp=P[ids].copy(),
                          inv1=0.5, inv2=0.5, cases=(s0, s1)))
    return bases


# ---- the shapes where k_pairs' schedule changes ------------------------------------------------------------------------
def dense_ball(n, seed=0):
    """n points in a ball of radius 0.1 (mirrored): with d = 0.05, eps = 0.2 every pair passes the band and the
    pre-filter, so the per-step survivors overflow the shared queue; random normals and rgb"""
    rng = np.random.RandomState(seed)
    u = rng.standard_normal((n // 2, 3))
    u *= (0.1 * rng.uniform(0, 1, (n // 2, 1)) ** (1 / 3)) / np.linalg.norm(u, axis=1, keepdims=True)
    nrm = rng.standard_normal((n // 2, 3))
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    c = mirrored(u.astype(f32), nrm.astype(f32), rng.uniform(0, 1, (n // 2, 3)).astype(f32))
    c["name"] = "dense_ball_%d" % n
    return c


def random_cloud(n, seed=0):
    """n points (the first n of a mirrored cloud) with normals and rgb, some rgb[0] negative"""
    rng = np.random.RandomState(seed + n)
    m = (n + 1) // 2
    x = rng.uniform(-0.5, 0.5, (m, 3)).astype(f32)
    nrm = rng.standard_normal((m, 3))
    nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(f32)
    rgb = rng.uniform(0, 1, (m, 3)).astype(f32)
    rgb[rng.uniform(size=m) < 0.1, 0] = -1
    c = mirrored(x, nrm, rgb)
    for k in ("Q", "Qn", "Qrgb"):
        c[k] = np.ascontiguousarray(c[k][:n])
    c["name"] = "random_%d" % n
    return c
