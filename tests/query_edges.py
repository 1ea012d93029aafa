"""Decision-edge fixtures for the box descent of the point queries (super4pcs_b200/csrc/query.cu), and an exact
restatement of the lower bound that lets the descent drop a box or a cell row.

The descent is exact only if cells_bound never exceeds a d^2 the kernel computes for a point binned in the box or row it
drops.  Random clouds never bring a decision near that bound, so this module builds such cases on purpose, on the grids
of tests/edges.py (grid_layout):

* A  P points binned across a cell face: their computed cell floor(fl(fl(p - o) * inv_h)) differs from floor(v),
     v = (p - o) * inv_h exactly -- upward (the product rounds up onto the face) or downward (the subtraction rounds
     down) -- on every axis, on a cell-row face inside a coarse block (y, z: the row test), a coarse-block face (x: the
     box test only, rows span the block on x) and a face where the two coincide (y, z), near the highest cell index;
     the query on the side the point crossed towards, 0.5 to 300 cells away, on that axis alone and diagonally.
* B  queries 10^3 to 10^6 cells out on one axis, the point chosen among neighbouring floats so that its fp32 d^2 rounds
     below the exact value: there the (1 - 2^-20) factor is what keeps the box.
* D  queries at +-FLT_MAX, +-inf and +-1e19 on one axis (every or no d^2 overflows), at sq_radius +inf and FLT_MAX.
* E  k-th ties: two points mirrored about the query on one axis (bit-identical d^2) in two coarse blocks, the larger
     index in the query's block (found first, nearer half first) behind two nearer points, so the row is full before the
     smaller index is met.
* F  radius counts: a point whose last neighbour is a family-A point across a face, at d^2 = sq_radius -+ floats.
* G  cluster links: a family-A link at sq_radius - 1 float (an edge) and at sq_radius (none), with a helper point.

Every query fixture carries the fp32 d^2 of its decided point and sq_radius at that d^2 and -2 ... +2 floats around it.
Family C (a subnormal d^2, where the -2^-140 term would decide) cannot be built through s4g_set_cloud_p: see
`field_reach_voxels`.

The restatement (`binned`, `exact_v`, `query_u`, `cells_bound`, `path_boxes`) follows the formulas of the header of
query.cu and of cell_of in context.cu, in double where the kernel computes in double (Python floats are IEEE doubles;
the library is built with -fmad=false, so no operation is fused) and in Fraction where the claim is exact.
`emulate_knn` replays the k-nearest descent on the host for the fixtures whose answer depends on its order (E).
"""
import functools
import math
from fractions import Fraction as Fr

import numpy as np

from tests import edges as E

f32 = np.float32
FLT_MAX = f32(np.finfo(f32).max)
KS = E.KS

# name -> (delta, box centre, box half extents, S4G_CSHIFT_MIN): the box's corners fix the grid
REGIMES = {
    "widened": E.REGIMES["widened"] + (1,),             # ~2000 cells on x: eps and the binning error are largest
    "offcentre1e4": E.REGIMES["offcentre1e4"] + (1,),   # p - o exact (Sterbenz): only the product rounds
    "straddle": (0.001, (0.002, -0.003, 0.001), (0.9, 0.8, 0.85), 1),   # o ~ -p: p - o a binade above p, rounds
    "brick8": E.REGIMES["brick8"] + (1,),               # 8-cell bricks, coarser blocks
    "centred-c1": E.REGIMES["centred"] + (1,),          # 2-cell coarse blocks
    "centred-c3": E.REGIMES["centred"] + (3,),          # S4G_CSHIFT_MIN = 3: 8-cell coarse blocks
}
FAMILIES = ("A", "B", "D", "E", "F", "G")


def env_cshift(name):
    """the S4G_CSHIFT_MIN a regime runs with (None: unset)"""
    c = REGIMES[name][3]
    return None if c == 1 else c


# ---- the restatement ----------------------------------------------------------------------------------------------------
def binned(g, x, axis):
    """cell of x on one axis as cell_of computes it, before its clamp"""
    with np.errstate(over="ignore", invalid="ignore"):
        return int(np.floor(f32(f32(f32(x) - g["o"][axis]) * g["inv_h"])))


def exact_v(g, x, axis):
    """the exact cell coordinate (x - o) * inv_h, with the float inv_h the kernel uses"""
    return (Fr(float(f32(x))) - Fr(float(g["o"][axis]))) * Fr(float(g["inv_h"]))


def eps_cells(g):
    return float(max(g["n"]) + 2) * 2.0 ** -21


def query_u(g, y):
    """u = (y - o) * inv_h in double, per axis (query_cells)"""
    ih = float(g["inv_h"])
    return tuple((float(f32(y[k])) - float(g["o"][k])) * ih for k in range(3))


def d2_f32(y, p):
    """the kernel's fp32 d^2: dx^2 + (dy^2 + dz^2)"""
    y, p = np.asarray(y, f32), np.asarray(p, f32)
    with np.errstate(over="ignore", invalid="ignore"):
        d = y - p
        return f32(d[0] * d[0] + f32(d[1] * d[1] + d[2] * d[2]))


def d2_exact(y, p):
    return sum((Fr(float(f32(a))) - Fr(float(f32(b)))) ** 2 for a, b in zip(y, p))


def rd_f32(b):
    """__double2float_rd"""
    with np.errstate(over="ignore"):
        f = f32(b)
    if float(f) > b:
        f = np.nextafter(f, f32(-np.inf))
    return f32(f)


# the wrong forms of the bound that must each change some answer (mutants), and eps / 4, which is still sound
MUTANTS = {
    "eps=0": dict(eps_scale=0.0),
    "eps/64": dict(eps_scale=1.0 / 64),
    "no (1 - 2^-20)": dict(factor=False),
    "x1 + eps": dict(upper_one=False),
}
SOUND_VARIANTS = {"eps/4": dict(eps_scale=0.25)}


def cells_bound(g, y, box, eps_scale=1.0, factor=True, upper_one=True, sub_term=True):
    """cells_bound(q, x0, x1, y0, y1, z0, z1) of query.cu for the query y and a box of cells ((x0, x1), (y0, y1),
    (z0, z1)): every operation in double and in the kernel's order, rounded down to fp32; the keyword arguments give
    its wrong forms"""
    u = query_u(g, y)
    e = eps_cells(g) * eps_scale
    ih = float(g["inv_h"])
    h2 = 1.0 / (ih * ih)
    gs = []
    for k in range(3):
        c0, c1 = box[k]
        top = (float(c1) + 1.0 + e) if upper_one else (float(c1) + e)
        gs.append(max(0.0, max((float(c0) - e) - u[k], u[k] - top)))
    s = (gs[0] * gs[0] + gs[1] * gs[1]) + gs[2] * gs[2]
    b = s * h2
    if factor:
        b = b * (1.0 - 2.0 ** -20)
    if sub_term:
        b = b - 2.0 ** -140
    return rd_f32(b) if b > 0.0 else f32(0.0)


def coarse_extent(g):
    cs = g["cshift"]
    return [(g["n"][k] >> cs) + 1 for k in range(3)]


def block_cells(g, lo, hi):
    """the cell ranges of a box of coarse blocks, as the kernels clip them"""
    cs = g["cshift"]
    return tuple((lo[k] << cs, min(((hi[k] + 1) << cs) - 1, g["n"][k] - 1)) for k in range(3))


def split(lo, hi):
    """the descent's halving of a box of blocks: (axis, mid) of its longest axis, x before y before z"""
    ex, ey, ez = (hi[k] - lo[k] for k in range(3))
    if ex >= ey and ex >= ez:
        a = 0
    elif ey >= ez:
        a = 1
    else:
        a = 2
    return a, (lo[a] + hi[a]) >> 1


def path_boxes(g, cell):
    """every box of cells the descent can open that holds a point binned in `cell`: the boxes of blocks from the root to
    the cell's block, then the cell's row (the block's cells on x, the cell on y and z)"""
    cs = g["cshift"]
    blk = [c >> cs for c in cell]
    lo, hi = [0, 0, 0], [c - 1 for c in coarse_extent(g)]
    out = []
    while True:
        out.append(block_cells(g, lo, hi))
        if lo == hi:
            break
        a, mid = split(lo, hi)
        if blk[a] <= mid:
            hi[a] = mid
        else:
            lo[a] = mid + 1
    bx = out[-1][0]
    out.append((bx, (cell[1], cell[1]), (cell[2], cell[2])))
    return out


def point_cell(g, p):
    return tuple(binned(g, p[k], k) for k in range(3))


def drops(g, y, p, sq_radius, strict_keep, **variant):
    """does the descent (with the given form of the bound) drop the point p for the query y at a fixed radius?  The
    boxes on p's path are nested, so the point is dropped iff one of them is: strict_keep (range, radius counts,
    cluster links) drops at bound >= sq_radius, else (k-nearest while its row is not full) at bound > sq_radius"""
    r = f32(sq_radius)
    for box in path_boxes(g, point_cell(g, p)):
        b = cells_bound(g, y, box, **variant)
        if (b >= r) if strict_keep else (b > r):
            return True
    return False


# ---- the grid -----------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def regime_grid(name):
    delta, centre, half, csm = REGIMES[name]
    corners = E._corners(centre, half)
    g = E.grid_layout(corners, delta, csm)
    mx = corners.max(0)
    # context.cu subtracts in float: n = ceil(fl(mx - o) / h) + 2
    g["n_float_sub"] = [int(math.ceil(float(f32(mx[k] - g["o"][k])) / g["h"])) + 2 for k in range(3)]
    return corners, g


def face_world(g, axis, F):
    return float(g["o"][axis]) + F / float(g["inv_h"])


def crossing_floats(g, axis, F, direction, span=256):
    """floats x near the face F with binned(x) = F while v < F ('up') or binned(x) = F - 1 while v >= F ('down'); the
    candidates are screened in double and confirmed in Fraction"""
    x = E.step(f32(face_world(g, axis, F)), np.arange(-span, span + 1)).astype(f32)
    with np.errstate(over="ignore", invalid="ignore"):
        c = np.floor(f32(f32(x - g["o"][axis]) * g["inv_h"])).astype(np.int64)
    v = (x.astype(np.float64) - float(g["o"][axis])) * float(g["inv_h"])
    near = np.nonzero((np.abs(v - F) < 1e-3) & ((c == F) | (c == F - 1)))[0]
    out = []
    for i in near:
        ci, vi = int(c[i]), exact_v(g, x[i], axis)
        if direction == "up" and ci == F and vi < F:
            out.append((f32(x[i]), F - vi))
        elif direction == "down" and ci == F - 1 and vi >= F:
            out.append((f32(x[i]), vi - F))
    return out


def face_kind_ok(g, axis, F, kind):
    blockface = F % (1 << g["cshift"]) == 0
    return {"box": axis == 0 and blockface, "row": axis != 0 and not blockface, "both": axis != 0 and blockface}[kind]


def find_crossing(g, axis, kind, direction, hi_cell, skip=0):
    """(F, x, depth): the highest face F <= hi_cell of the kind with a float x binned across it in the direction, the
    deepest such x (largest |v - F|); skip passes over that many suitable faces first"""
    for F in range(hi_cell, 2, -1):
        if not face_kind_ok(g, axis, F, kind):
            continue
        xs = crossing_floats(g, axis, F, direction)
        if xs:
            if skip:
                skip -= 1
                continue
            x, depth = max(xs, key=lambda t: t[1])
            return F, x, depth
    return None


# ---- queries through T --------------------------------------------------------------------------------------------------
def rigid_T(seed=17):
    """one rigid T (row-major 3 x 4) whose translation moves the queries back onto the cloud"""
    R = E.rotations(1, np.random.RandomState(seed))[0]
    return np.concatenate([R, np.array([[0.03125], [-0.0625], [0.015625]], f32)], 1).astype(f32)


def resolve(y0, T34):
    """(x, y): the query input x and the query y the kernels see (exact_tq(T, x), or x); y is within float steps of y0"""
    y0 = np.asarray(y0, f32)
    if T34 is None:
        return y0.copy(), y0.copy()
    R, t = T34[:, :3].astype(np.float64), T34[:, 3].astype(np.float64)
    x = (R.T @ (y0.astype(np.float64) - t)).astype(f32)
    return x, E.fp32_tq(T34, x)[0].astype(f32)


# ---- the fixtures -------------------------------------------------------------------------------------------------------
class Builder:
    """one cloud (its corners fix the grid) and the fixtures placed in it"""

    def __init__(self, name, seed=0):
        self.name = name
        self.corners, self.g = regime_grid(name)
        self.delta = REGIMES[name][0]
        self.lo, self.hi = self.corners.min(0).astype(np.float64), self.corners.max(0).astype(np.float64)
        self.P = [p for p in self.corners]
        self.rng = np.random.RandomState(seed)
        self.queries = []     # dict(family, kind, x, y, T (bool), j, d2, radii, ks, exclude)
        self.pairs = []       # dict(family, kind, a, b, d2, radii)
        self.T34 = rigid_T()
        self.sites = []

    def add(self, p):
        self.P.append(np.asarray(p, f32))
        return len(self.P) - 1

    def site(self, axis):
        """a point of the box interior, away from earlier sites on the two axes other than `axis` (40 cells, or less on
        a small grid)"""
        h = 1.0 / float(self.g["inv_h"])
        spread = min(40.0 * h, float((self.hi - self.lo).min()) / 14)
        others = [k for k in range(3) if k != axis]
        while True:
            for _ in range(200):
                s = self.rng.uniform(self.lo + 0.12 * (self.hi - self.lo), self.hi - 0.12 * (self.hi - self.lo))
                if all(max(abs(s[k] - t[k]) for k in others) > spread for t in self.sites):
                    self.sites.append(s)
                    return s
            spread /= 2

    def radii(self, d2):
        return [f32(E.step(d2, k)) for k in KS]

    def query(self, family, kind, y0, T, j, ks=(1, 64), exclude=-1):
        x, y = resolve(y0, self.T34 if T else None)
        d2 = d2_f32(y, self.P[j])
        self.queries.append(dict(family=family, kind=kind, x=x, y=y, T=T, j=j, d2=d2, radii=self.radii(d2), ks=ks,
                                 exclude=exclude))

    # A: binned across a face
    def family_a(self, T):
        g = self.g
        h = 1.0 / float(g["inv_h"])
        for axis, kind in ((0, "box"), (1, "row"), (1, "both"), (2, "row"), (2, "both")):
            top = binned(g, self.hi[axis], axis)
            for direction in ("up", "down"):
                found = find_crossing(g, axis, kind, direction, top - 1, skip=int(T))
                if found is None:
                    continue
                F, xa, _ = found
                s = self.site(axis)
                p = s.astype(f32)
                p[axis] = xa
                j = self.add(p)
                sign = -1.0 if direction == "up" else 1.0
                for dist in (0.5, 7.25, 300.0):
                    for diag in (False, True):
                        if diag and dist > 10:
                            continue
                        y0 = p.astype(np.float64)
                        y0[axis] = face_world(g, axis, F) + sign * dist * h
                        if diag:
                            b = (axis + 1) % 3
                            y0[b] += 0.75 * dist * h
                        self.query("A", "%s-%d-%s-%g%s" % (kind, axis, direction, dist, "-diag" if diag else ""),
                                   y0, T, j)

    # B: far queries whose fp32 d^2 rounds below the exact value
    def family_b(self, T):
        g = self.g
        h = 1.0 / float(g["inv_h"])
        cs = 1 << g["cshift"]
        for axis in range(3):
            for side in (1, -1):
                for far in (1e3, 3e4, 1e6):
                    s = self.site(axis)
                    if side > 0:    # the point just below the top face of a block near the cloud's top
                        F = (binned(g, self.hi[axis], axis) // cs) * cs
                        base = E.step(f32(face_world(g, axis, F)), -2)
                        while binned(g, base, axis) >= F:
                            base = E.step(base, -1)
                        cand = E.step(base, -np.arange(0, 48))
                    else:           # just above the bottom face of a block near the cloud's bottom
                        F = (binned(g, self.lo[axis], axis) // cs + 1) * cs
                        base = E.step(f32(face_world(g, axis, F)), 2)
                        while binned(g, base, axis) < F:
                            base = E.step(base, 1)
                        cand = E.step(base, np.arange(0, 48))
                    best = None
                    for xa in cand:
                        p = s.astype(f32)
                        p[axis] = xa
                        y0 = p.astype(np.float64)
                        y0[axis] += side * far * h
                        _, y = resolve(y0, self.T34 if T else None)
                        d2 = d2_f32(y, p)
                        deficit = (d2_exact(y, p) - Fr(float(d2))) / d2_exact(y, p)
                        if best is None or deficit > best[0]:
                            best = (deficit, p, y0)
                    j = self.add(best[1])
                    self.query("B", "%d-%+d-%g" % (axis, side, far), best[2], T, j)

    # D: overflow (identity only: a T would turn an infinite coordinate into NaN)
    def family_d(self):
        for axis in range(3):
            s = self.site(axis).astype(f32)
            j = self.add(s + f32(0.5 / float(self.g["inv_h"])))
            for v in (FLT_MAX, -FLT_MAX, np.inf, -np.inf, 1e19, -1e19):
                y = s.copy()
                y[axis] = f32(v)
                d2 = d2_f32(y, self.P[j])
                self.queries.append(dict(family="D", kind="%d-%g" % (axis, v), x=y, y=y, T=False, j=j, d2=d2,
                                         radii=[f32(np.inf), FLT_MAX], ks=(1, 3, 64), exclude=-1))

    # E: k-th ties across a coarse-block face
    def family_e(self, T):
        g = self.g
        h = 1.0 / float(g["inv_h"])
        cs = 1 << g["cshift"]
        for axis in range(3):
            s = self.site(axis)
            faces = [F for F in range(cs, g["n"][axis], cs) if self.lo[axis] + 2 * h < face_world(g, axis, F) < self.hi[axis] - 2 * h]
            F = min(faces, key=lambda F: abs(face_world(g, axis, F) - s[axis]))
            y0 = s.copy()
            y0[axis] = face_world(g, axis, F) - 0.3 * h          # in the block below the face, 0.3 cells from it
            _, y = resolve(y0, self.T34 if T else None)
            assert binned(g, y[axis], axis) == F - 1
            a = f32(0.75 * h)
            for _ in range(200):
                pm, pp = y.copy(), y.copy()
                pm[axis], pp[axis] = f32(y[axis] - a), f32(y[axis] + a)
                if (d2_f32(y, pm).view(np.uint32) == d2_f32(y, pp).view(np.uint32)
                        and binned(g, pp[axis], axis) >= F and binned(g, pm[axis], axis) >= F - cs):
                    break
                a = E.step(a, 1)
            else:
                raise AssertionError("no mirrored pair")
            o = (axis + 1) % 3
            near = []
            for t in (0.05, -0.1):
                q = y.copy()
                q[o] = f32(y[o] + t * h)
                near.append(q)
            jp = self.add(pp)                                    # the smaller index: in the block searched second
            for q in near:
                self.add(q)
            jm = self.add(pm)                                    # the larger index: found first
            x, _ = resolve(y0, self.T34 if T else None)
            d2 = d2_f32(y, pp)
            q = dict(family="E", kind="%d" % axis, x=x, y=y, T=T, j=jp, d2=d2, radii=self.radii(d2) + [f32(np.inf)],
                     ks=(1, 2, 3, 4, 64), exclude=-1)
            self.queries.append(q)
            for ex, what in ((jp, "small"), (jm, "large")):
                self.queries.append(dict(q, exclude=ex, kind=q["kind"] + "-excl-" + what))

    # F and G: P-to-P decisions across a face (a: the family-A point, smaller index; b: the other side)
    def family_fg(self):
        g = self.g
        h = 1.0 / float(g["inv_h"])
        for axis, kind in ((0, "box"), (1, "row"), (2, "both")):
            top = binned(g, self.hi[axis], axis)
            for direction in ("up", "down"):
                found = find_crossing(g, axis, kind, direction, top - 3, skip=2)
                if found is None:
                    continue
                F, xa, _ = found
                sign = -1.0 if direction == "up" else 1.0
                for fam, dist in (("F", 0.5), ("G", 1.5)):
                    s = self.site(axis)
                    a = s.astype(f32)
                    a[axis] = xa
                    b = a.copy()
                    b[axis] = f32(face_world(g, axis, F) + sign * dist * h)
                    helper = b.copy()
                    helper[axis] = f32(b[axis] + sign * 0.2 * h)
                    ja = self.add(a)
                    jb = self.add(b)
                    self.add(helper)
                    d2 = d2_f32(b, a)
                    self.pairs.append(dict(family=fam, kind="%s-%d-%s" % (kind, axis, direction), a=ja, b=jb, d2=d2,
                                           radii=self.radii(d2)))

    def finish(self):
        P = np.array(self.P, f32)
        assert (P.min(0) >= self.corners.min(0)).all() and (P.max(0) <= self.corners.max(0)).all()
        return dict(name=self.name, P=P, g=E.grid_layout(P, self.delta, REGIMES[self.name][3]), delta=self.delta,
                    T34=self.T34, queries=self.queries, pairs=self.pairs)


@functools.lru_cache(maxsize=None)
def scene(name):
    b = Builder(name)
    for T in (False, True):
        b.family_a(T)
        b.family_b(T)
        b.family_e(T)
    b.family_d()
    b.family_fg()
    return b.finish()


# ---- the k-nearest descent on the host ----------------------------------------------------------------------------------
def emulate_knn(g, P, y, k, sq_radius, exclude=-1, bound_from="kth", **variant):
    """the row k_knn returns for the query y, its descent replayed (boxes halved on the longest axis, the nearer half
    first; rows in a block by z then y, points by x cell then index).  bound_from='first' takes the running bound from
    the first held entry instead of the k-th (a wrong form)"""
    cs = g["cshift"]
    cells = [point_cell(g, p) for p in P]
    blocks = {tuple(c >> cs for c in cell) for cell in cells}
    rows = {}
    for j in sorted(range(len(P)), key=lambda j: (cells[j][0], j)):
        rows.setdefault((cells[j][1], cells[j][2]), []).append((cells[j][0], j))
    u = query_u(g, y)
    held = []
    bound = f32(sq_radius)
    stack = [([0, 0, 0], [c - 1 for c in coarse_extent(g)])]
    while stack:
        lo, hi = stack.pop()
        box = block_cells(g, lo, hi)
        if any(c0 > c1 for c0, c1 in box):
            continue
        if cells_bound(g, y, box, **variant) > bound:
            continue
        if not any(all(lo[a] <= b[a] <= hi[a] for a in range(3)) for b in blocks):
            continue
        if lo != hi:
            a, mid = split(lo, hi)
            hi_lo, lo_hi = list(hi), list(lo)
            hi_lo[a], lo_hi[a] = mid, mid + 1
            low, high = (lo, hi_lo), (lo_hi, hi)
            lo_near = u[a] < float((mid + 1) << cs)
            stack.append(high if lo_near else low)
            stack.append(low if lo_near else high)
            continue
        (cx0, cx1), (cy0, cy1), (cz0, cz1) = box
        for cz in range(cz0, cz1 + 1):
            for cy in range(cy0, cy1 + 1):
                if cells_bound(g, y, ((cx0, cx1), (cy, cy), (cz, cz)), **variant) > bound:
                    continue
                for cx, j in rows.get((cy, cz), ()):
                    if not cx0 <= cx <= cx1:
                        continue
                    d2 = d2_f32(y, P[j])
                    if not d2 <= f32(sq_radius) or j == exclude:
                        continue
                    key = (int(d2.view(np.uint32)), j)
                    if len(held) == k and key >= held[-1]:
                        continue
                    held = sorted(held + [key])[:k]
                    if len(held) == k:
                        src = held[-1] if bound_from == "kth" else held[0]
                        bound = np.uint32(src[0]).view(f32)
    index = [j for _, j in held] + [-1] * (k - len(held))
    sq = [np.uint32(b).view(f32) for b, _ in held] + [f32(np.inf)] * (k - len(held))
    return np.array(index, np.int32), np.array(sq, f32)


# ---- family C: the grid s4g_set_cloud_p would need -----------------------------------------------------------------------
def field_reach_voxels(P, delta):
    """reach / v of the delta-field that s4g_set_cloud_p builds with the grid (context.cu): the field's slack and margin
    carry absolute terms 8 (1 + |p|) 2^-20 and (1 + |p|) 2^-40, so on a cloud at scale 2^-60 the reach is ~2^54 voxels:
    the voxel radius R = ceil(1 + reach / v) does not fit an int and the field cannot be built"""
    P = np.asarray(P, f32)
    g = E.grid_layout(P, delta)
    v = 1.0 / float(f32(4.0) * g["inv_h"])
    pabs = float(np.abs(P).max())
    slack = max(0.02 * v, math.ldexp(8.0 * (1.0 + pabs), -20))
    md = 1e-5 * float(f32(delta)) + math.ldexp(1.0 + pabs, -40)
    return (float(f32(delta)) + md + slack) / v
