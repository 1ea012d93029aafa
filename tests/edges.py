"""Decision-edge cases for Verify and the pair query, and an fp32 oracle that shares no code with oracle/port.cc.

Verify's count is exact only if every shortcut in front of the fp32 point test (the tile cull, the delta-field, the 2x2x2
probe block) is conservative.  Random clouds almost never put a decision within a few ulps of its boundary, so this module
builds such cases on purpose:

* `fp32_tq`, `fp32_d2`, `fp32_inlier`: the reference's decision with every operation in float32 and in its order
  (T q = ((m0 x + m1 y) + m2 z) + m3, d^2 = dx^2 + (dy^2 + dz^2), d^2 <= fl(delta * delta)).  numpy rounds every
  float32 operation and never fuses two, so this is the reference's arithmetic, not an approximation of it.
* `walk_targets`: targets t near a P point p in a direction u whose fl(d^2) lies k ulps from fl(delta^2), found by a
  search over float neighbours (nextafter steps) of p + delta u.
* `grid_layout`: the grid of s4g_set_cloud_p recomputed on the host from its formulas, so that points can be put within
  ulps of voxel, sub-voxel, cell, brick, coarse-block and outer faces.
* `regime_cloud`: a sparse P (every target has one P point within 3 delta) with anchors on those faces, and the targets.
* `verify_record` / `tile_live`: the candidate record (fast or robust path) and the tile cull of verify.cu, emulated
  exactly, to show that the off-centre cases reach the cull: a fixed 0.52-cell pad culls some of their inliers.
* `pair_cloud` / `pair_set`: point pairs at the edges of the pair query's distance band, and its predicate in float32.
"""
import math
from fractions import Fraction

import numpy as np

f32 = np.float32
KS = (-2, -1, 0, 1, 2)


# ---- float32 ordering helpers -----------------------------------------------------------------------------------------
def ordinal(x):
    """monotone integer image of float32 values (adjacent floats differ by 1)"""
    i = np.asarray(x, f32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7FFFFFFF), i)


def from_ordinal(o):
    o = np.asarray(o, np.int64)
    i = np.where(o < 0, (-o) | 0x80000000, o).astype(np.uint32)
    return i.view(f32)


def step(x, n):
    """x moved by n float32 steps (n may be an array)"""
    return from_ordinal(ordinal(x) + np.asarray(n, np.int64))


def round_f32(fr):
    """nearest float32 (ties to even) of an exact Fraction"""
    c = f32(float(fr))
    best = None
    for cand in (step(c, -1), c, step(c, 1)):
        cand = f32(cand)
        err = abs(Fraction(float(cand)) - fr)
        key = (err, int(cand.view(np.uint32)) & 1)
        if best is None or key < best[0]:
            best = (key, cand)
    return best[1]


def fma_f32(a, b, c):
    """fmaf: a * b + c rounded once"""
    return round_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


# ---- the decision, in float32 -----------------------------------------------------------------------------------------
def sq_eps(delta):
    return f32(delta) * f32(delta)


def fp32_d2(t, P):
    """(N, M) fl(d^2) of targets t (N, 3) against P (M, 3), as dx^2 + (dy^2 + dz^2)"""
    t, P = np.asarray(t, f32).reshape(-1, 3), np.asarray(P, f32).reshape(-1, 3)
    d = t[:, None, :] - P[None, :, :]
    return d[..., 0] * d[..., 0] + (d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2])


def fp32_inlier(P, t, delta):
    """does some P point lie within delta of each target (the reference's test, brute force)"""
    t = np.asarray(t, f32).reshape(-1, 3)
    out = np.zeros(len(t), bool)
    for s in range(0, len(t), 4096):
        out[s:s + 4096] = (fp32_d2(t[s:s + 4096], P) <= sq_eps(delta)).any(1)
    return out


def fp32_tq(T, q):
    """fl(T q) of row-major (K, 3, 4) transforms T for one point q, in the reference's order"""
    T, q = np.asarray(T, f32).reshape(-1, 3, 4), np.asarray(q, f32).reshape(3)
    return ((T[:, :, 0] * q[0] + T[:, :, 1] * q[1]) + T[:, :, 2] * q[2]) + T[:, :, 3]


def fp32_tq_all(T, Q):
    """(K, N, 3) fl(T q) of every candidate and every point of Q"""
    T, Q = np.asarray(T, f32).reshape(-1, 3, 4), np.asarray(Q, f32).reshape(-1, 3)
    a = T[:, None, :, 0] * Q[None, :, None, 0] + T[:, None, :, 1] * Q[None, :, None, 1]
    return (a + T[:, None, :, 2] * Q[None, :, None, 2]) + T[:, None, :, 3]


def margin_ulps(P, t, delta):
    """(ulps, dist): each target's min fl(d^2) over P minus fl(delta^2) in float32 steps (<= 0: inlier), and its exact
    float64 distance to the nearest P point"""
    d2 = fp32_d2(t, P).min(1)
    exact = np.sqrt(((np.asarray(t, np.float64)[:, None, :] - np.asarray(P, np.float64)[None]) ** 2).sum(-1)).min(1)
    return ordinal(d2) - ordinal(sq_eps(delta)), exact


def colmajor(T34):
    """row-major (K, 3, 4) -> the API's column-major (K, 16)"""
    T34 = np.asarray(T34, f32).reshape(-1, 3, 4)
    M = np.zeros((len(T34), 4, 4), f32)
    M[:, :3, :] = T34
    M[:, 3, 3] = 1
    return np.ascontiguousarray(M.transpose(0, 2, 1)).reshape(-1, 16)


def rotations(n, rng):
    """n random proper rotations (float32)"""
    A = rng.standard_normal((n, 3, 3))
    Qm, Rm = np.linalg.qr(A)
    Qm = Qm * np.sign(np.diagonal(Rm, axis1=1, axis2=2))[:, None, :]
    Qm[np.linalg.det(Qm) < 0, :, 0] *= -1
    return Qm.astype(f32)


# ---- targets at k ulps ------------------------------------------------------------------------------------------------
def directions(rng, n_random=3):
    """the axes, face diagonals and body diagonals (random signs) and random unit directions"""
    out = [np.eye(3)[i] for i in range(3)]
    out += [np.array(v, float) / math.sqrt(2) for v in ((1, 1, 0), (1, 0, 1), (0, 1, 1))]
    out += [np.array(v, float) / math.sqrt(3) for v in ((1, 1, 1), (1, -1, 1))]
    out = [u * rng.choice([-1, 1], 3) for u in out]
    for _ in range(n_random):
        u = rng.standard_normal(3)
        out.append(u / np.linalg.norm(u))
    return out


def walk_targets(p, u, delta, main=4, side=24):
    """targets near the ray p + s u, s ~ delta: {k: t} with fl(d^2(t, p)) exactly k float steps from fl(delta^2) for
    every k of KS that the float neighbours of p + delta u reach, and under 'in' / 'out' the reached target closest to
    the boundary on either side.  Among equal k the one closest to the ray wins."""
    p = np.asarray(p, f32)
    t0 = (p.astype(np.float64) + float(delta) * np.asarray(u)).astype(f32)
    ax = int(np.argmax(np.abs(u)))
    o = [np.arange(-side, side + 1)] * 3
    o[ax] = np.arange(-main, main + 1)
    g = np.meshgrid(*o, indexing="ij")
    T = np.stack([step(t0[i], g[i].ravel()) for i in range(3)], 1).astype(f32)
    k = (ordinal(fp32_d2(T, p[None])[:, 0]) - ordinal(sq_eps(delta)))
    dev = np.abs(g[0].ravel()) + np.abs(g[1].ravel()) + np.abs(g[2].ravel())
    out = {}
    for kk in KS:
        idx = np.nonzero(k == kk)[0]
        if len(idx):
            out[kk] = T[idx[np.argmin(dev[idx])]]
    for name, sel in (("in", k <= 0), ("out", k > 0)):
        idx = np.nonzero(sel)[0]
        if len(idx):
            best = idx[np.lexsort((dev[idx], np.abs(k[idx])))[0]]
            out[name] = T[best]
    return out


# ---- the grid of s4g_set_cloud_p, on the host ---------------------------------------------------------------------------
def cell_of(g, x, axis):
    """cell index of world coordinates x on one axis, as k_mark_* compute it: floor(fl(fl(x - o) * inv_h)), clamped"""
    c = np.floor((np.asarray(x, f32) - g["o"][axis]) * g["inv_h"]).astype(np.int64)
    return np.clip(c, 0, g["n"][axis] - 1)


def grid_layout(P, delta, cshift_min=1):
    P = np.asarray(P, f32)
    mn, mx = P.min(0), P.max(0)
    h = 2.0 * float(f32(delta)) * 1.01
    ext = max(float(mx[k]) - float(mn[k]) for k in range(3))
    widened = ext / h > 2000.0
    if widened:
        h = ext / 2000.0
    while True:
        o = np.array([f32(float(mn[k]) - 1.5 * h) for k in range(3)], f32)
        inv_h = f32(1.0 / h)
        n = [int(math.ceil((float(mx[k]) - float(o[k])) / h)) + 2 for k in range(3)]
        for bs in range(2, 7):
            B = 1 << bs
            tb = [(n[k] + B - 1) // B for k in range(3)]
            ntop = tb[0] * tb[1] * tb[2]
            if ntop <= 1 << 24:
                break
        if ntop <= 1 << 24:
            break
        h *= 1.5
    g = dict(h=h, o=o, inv_h=inv_h, n=n, bshift=bs, widened=widened)
    g["inv_v"] = f32(4.0) * inv_h
    v = 1.0 / float(g["inv_v"])
    pabs = max(max(abs(float(mn[k])), abs(float(mx[k]))) for k in range(3))
    g["v"] = v
    g["slack"] = max(0.02 * v, math.ldexp(8.0 * (1.0 + pabs), -20))
    g["md"] = 1e-5 * float(f32(delta)) + math.ldexp(1.0 + pabs, -40)
    g["vslack"] = f32(g["slack"] * 0.999)
    cs = max(1, min(11, cshift_min))
    while cs < 12:
        cn = [(n[k] >> cs) + 1 for k in range(3)]
        if (cn[0] + 1) * (cn[1] + 1) * (cn[2] + 1) <= 1 << 20:
            break
        cs += 1
    g["cshift"] = cs
    c = np.stack([cell_of(g, P[:, k], k) for k in range(3)], 1)
    g["bricks"] = len(np.unique(c >> bs, axis=0))
    g["cells"] = g["bricks"] << (3 * bs)
    g["occupied_blocks"] = {tuple(b) for b in (c >> cs).tolist()}
    return g


def face_coord(g, kind, axis, index):
    """world coordinate (float64) of face `index` of a lattice kind along an axis"""
    width = {"voxel": 0.25, "subvoxel": 0.125, "cell": 1.0, "brick": float(1 << g["bshift"]),
             "coarse": float(1 << g["cshift"])}[kind]
    return float(g["o"][axis]) + index * width * g["h"]


def first_in_cell(g, axis, cell, near):
    """smallest float32 x >= near - a few cells' worth of steps with cell_of(x) >= cell (the lowest point of that cell)"""
    x = f32(near)
    lo = step(x, -4096)
    hi = step(x, 4096)
    cand = step(lo, np.arange(0, int(ordinal(hi) - ordinal(lo)) + 1))
    ok = cell_of(g, cand, axis) >= cell
    return f32(cand[np.argmax(ok)])


# ---- regimes ----------------------------------------------------------------------------------------------------------
# name -> (delta, box centre, box half extents): the box corners fix the grid before the anchors are placed
REGIMES = {
    "centred": (0.01, (0.0, 0.0, 0.0), (0.25, 0.22, 0.2)),            # 4-cell bricks: k_verify<false, 2>
    "brick8": (0.0008, (0.0, 0.0, 0.0), (1.16, 1.16, 0.75)),          # > 2^24 four-cell bricks: k_verify<false, 0>
    "widened": (0.0004, (0.0, 0.0, 0.0), (1.2, 0.3, 0.3)),            # > 2000 cells of 2.02 delta: wider cells
    "offcentre1e3": (0.0078125, (1000.1, 999.7, 1000.3), (0.25, 0.22, 0.2)),   # slack = 2 % of a voxel still
    "offcentre1e4": (0.0078125, (12000.3, 11999.6, 12000.1), (0.25, 0.22, 0.2)),  # slack from the coordinates' size
}
FACE_KINDS = ("voxel", "subvoxel", "cell", "brick", "coarse")


def _corners(centre, half):
    c, hw = np.asarray(centre, np.float64), np.asarray(half, np.float64)
    return np.array([c + hw * np.array([sx, sy, sz]) for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)]).astype(f32)


def regime_cloud(name, seed=0, n_generic=8, n_face=4, cshift_min=1):
    """(P, cases, g): a sparse P whose bounding box is fixed by 8 corners, and a list of cases
    dict(t, anchor, kind, k) with kind in {'generic', 'outer', 'p_on_<face>', 't_on_<face>'}"""
    delta, centre, half = REGIMES[name]
    rng = np.random.RandomState(seed)
    corners = _corners(centre, half)
    g = grid_layout(corners, delta, cshift_min)
    lo, hi = corners.min(0).astype(np.float64), corners.max(0).astype(np.float64)
    anchors, kinds, axes = [], [], []

    def far_enough(p):
        return all(np.abs(np.asarray(a, np.float64) - p).max() > 7 * delta for a in anchors + list(corners))

    def add(p, kind, axis=0):
        p = np.asarray(p, f32)
        if far_enough(p.astype(np.float64)):
            anchors.append(p)
            kinds.append(kind)
            axes.append(axis)

    margin = 6 * delta
    while sum(k == "generic" for k in kinds) < n_generic:
        add(rng.uniform(lo + margin, hi - margin), "generic")
    for kind in FACE_KINDS:
        for _ in range(n_face):
            for _try in range(400):
                axis = rng.randint(3)
                p = rng.uniform(lo + margin, hi - margin)
                width = {"voxel": 0.25, "subvoxel": 0.125, "cell": 1, "brick": 1 << g["bshift"], "coarse": 1 << g["cshift"]}[kind]
                idx = int(round((p[axis] - float(g["o"][axis])) / (width * g["h"])))
                xf = face_coord(g, kind, axis, idx)
                if not (lo[axis] + margin < xf < hi[axis] - margin):
                    continue
                if kind in ("cell", "brick", "coarse"):
                    # the P point as close above the face as cell_of allows (it is then in the upper cell / block)
                    q = p.astype(f32)
                    q[axis] = step(first_in_cell(g, axis, int(round(idx * width)), xf), rng.randint(0, 3))
                else:
                    q = p.astype(f32)
                    q[axis] = step(f32(xf), rng.randint(-2, 3))
                # a target on the face: an anchor delta above it, whose walk towards -axis lands within ulps of it
                q2 = p.astype(np.float64)
                q2[(axis + 1) % 3] += 10 * delta if q2[(axis + 1) % 3] < 0 else -10 * delta
                q2 = q2.astype(f32)
                q2[axis] = step(f32(f32(xf) + f32(delta)), rng.randint(-2, 3))
                if far_enough(q.astype(np.float64)) and far_enough(q2.astype(np.float64)):
                    add(q, "p_on_" + kind, axis)
                    add(q2, "t_on_" + kind, axis)
                    break
    P = np.concatenate([corners, np.array(anchors, f32)]).astype(f32)
    cases = []
    for i, (p, kind, axis) in enumerate(list(zip(corners, ["outer"] * 8, [0] * 8)) + list(zip(anchors, kinds, axes))):
        if kind == "outer":
            # a query delta beyond the bounding box extremes, outward along each axis
            dirs = [np.eye(3)[a] * np.sign(float(p[a]) - float(centre[a])) for a in range(3)]
        elif kind.startswith("t_on_"):
            dirs = [-np.eye(3)[axis]]
        else:
            dirs = directions(rng)
        for u in dirs:
            for key, t in walk_targets(p, u, delta).items():
                cases.append(dict(t=np.asarray(t, f32), anchor=i, kind=kind, k=key))
    g = grid_layout(P, delta, cshift_min)
    return P, cases, g


def coverage(P, cases, delta, lattice_only=False):
    """(ulps, inlier) of the cases, asserted to hold exact ties, +-1 and +-2 ulps (unless the coordinates' lattice is
    coarser than an ulp of delta^2) and both outcomes"""
    t = np.array([c["t"] for c in cases], f32)
    ulps, dist = margin_ulps(P, t, delta)
    inl = fp32_inlier(P, t, delta)
    assert inl.any() and (~inl).any()
    assert (ulps == 0).any(), "no exact tie"
    if not lattice_only:
        for k in KS:
            assert (ulps == k).any(), "no case at %d ulps" % k
    # every target has exactly one P point within 3 delta (the decision is about that point)
    D = np.sqrt(((t.astype(np.float64)[:, None, :] - P.astype(np.float64)[None]) ** 2).sum(-1))
    assert ((D <= 3 * delta).sum(1) == 1).all()
    return ulps, inl


# ---- Verify's candidate record and the tile cull, emulated --------------------------------------------------------------
def verify_record(T34, g, qabs):
    """(V (3, 4), E, scale, fast) of s4g_verify_record for one row-major candidate, in float32 and its order"""
    m = np.asarray(T34, f32).reshape(12)
    o = g["o"]
    V = np.array([m[i] * g["inv_v"] if (i & 3) < 3 else (m[i] - o[i >> 2]) * g["inv_v"] for i in range(12)], f32)
    qa = np.asarray(qabs, f32)
    w = [((((abs(m[4 * r]) * qa[0] + abs(m[4 * r + 1]) * qa[1]) + abs(m[4 * r + 2]) * qa[2]) + abs(m[4 * r + 3]))
          + abs(o[r])) for r in range(3)]
    E = f32(max(w)) * f32(9.5367431640625e-7)
    M = m.reshape(3, 4)[:, :3]
    gd = [((M[0, i] * M[0, i] + M[1, i] * M[1, i]) + M[2, i] * M[2, i]) for i in range(3)]

    def off(i, j):
        return abs((M[0, i] * M[0, j] + M[1, i] * M[1, j]) + M[2, i] * M[2, j])
    g01, g02, g12 = off(0, 1), off(0, 2), off(1, 2)
    n2 = max((gd[0] + g01) + g02, max((g01 + gd[1]) + g12, (g02 + g12) + gd[2]))
    s = f32(np.sqrt(f32(n2))) * f32(1.00001)
    fast = bool(E <= g["vslack"]) and bool(s <= f32(1.0e6))
    return V.reshape(3, 4), E, s, fast


def tile_live(g, V, c, radius, scale, pad):
    """the tile cull of verify.cu (tile_live) with a given pad in cells: can a query in the sphere (c, radius) come within
    delta of a P point under the candidate of voxel-space matrix V?  (coarse occupancy from g['occupied_blocks'])"""
    cc = []
    for r in range(3):
        x = fma_f32(V[r, 0], c[0], fma_f32(V[r, 1], c[1], fma_f32(V[r, 2], c[2], V[r, 3])))
        cc.append(f32(0.25) * x)
    R = ((f32(radius) * g["inv_h"]) * f32(scale)) * f32(1.0001) + f32(pad)
    lo = [int(math.floor(float(f32(x - R)))) for x in cc]
    hi = [int(math.floor(float(f32(x + R)))) for x in cc]
    if any(hi[k] < 0 or lo[k] >= g["n"][k] for k in range(3)):
        return False
    cs = g["cshift"]
    rng = [range(max(0, lo[k]) >> cs, (min(g["n"][k] - 1, hi[k]) >> cs) + 1) for k in range(3)]
    return any((x, y, z) in g["occupied_blocks"] for x in rng[0] for y in rng[1] for z in rng[2])


# ---- the pair predicate, in float32 / float64 ---------------------------------------------------------------------------
def pair_params(Q, d, eps):
    """gcenter, ratio, nRadius, eps_round^2 of s4g_set_cloud_q / make_pair_args for the pair query"""
    Q = np.asarray(Q, f32)
    mn, mx = Q.min(0), Q.max(0)
    gc = (mn + mx) / f32(2)
    mc = (mx - mn).max()
    ratio = f32(float(mc) + 0.001)
    eps_norm = f32(eps) / ratio
    lvl = int(-np.log2(eps_norm))
    eps_round = f32(1.0 / 2.0 ** lvl)
    return gc, ratio, f32(d) / ratio, eps_round * eps_round


def pair_set(Q, d, eps):
    """every ordered pair (i, j), i != j, that the pair query accepts without filters: the unit-cube point test
    (|u_j - u_i| - nRadius)^2 < eps_round^2, then |fl(|q_i - q_j|) - d| <= eps in double; sorted"""
    Q = np.asarray(Q, f32)
    gc, ratio, nR, er2 = pair_params(Q, d, eps)
    U = ((Q - gc) / ratio) + f32(0.5)
    n = len(Q)
    out = []
    for s in range(0, n, 1024):
        du = U[None, :, :] - U[s:s + 1024, None, :]
        un = np.sqrt(du[..., 0] * du[..., 0] + (du[..., 1] * du[..., 1] + du[..., 2] * du[..., 2])) - nR
        dq = Q[None, :, :] - Q[s:s + 1024, None, :]
        dist = np.sqrt(dq[..., 0] * dq[..., 0] + (dq[..., 1] * dq[..., 1] + dq[..., 2] * dq[..., 2]))
        ok = (un * un < er2) & (np.abs(dist.astype(np.float64) - float(f32(d))) <= float(f32(eps)))
        i, j = np.nonzero(ok)
        i = i + s
        keep = i != j
        out.append(np.stack([i[keep], j[keep]], 1))
    p = np.concatenate(out).astype(np.int32) if out else np.zeros((0, 2), np.int32)
    return p[np.lexsort((p[:, 1], p[:, 0]))]


def prefilter_bounds(d, eps):
    """lo_sq, hi_sq of make_pair_args (the squared pre-filter band of k_pairs)"""
    lo = max(0.0, float(f32(d)) - float(f32(eps)))
    hi = float(f32(d)) + float(f32(eps))
    return f32(lo * lo * (1.0 - 4e-5)), f32(hi * hi * (1.0 + 4e-5)), lo, hi


# ---- point pairs at the edges of the distance band ----------------------------------------------------------------------
# (d, eps) of the pair queries run on PAIR_CLOUD; d - eps <= 0 for the last.  Every pair of the cloud is tuned to one of
# them; pairs of different sites are further apart than any band.
PAIR_QUERIES = ((1.0, 0.25), (1.0, 0.3), (0.9, 0.2), (1.1, 0.15), (0.1, 0.25))


def pair_cloud(unit_binding=False):
    """(Q, queries, kinds): pairs (a, b) with |b - a| at the edges of |dist - d| <= eps, one pair per site of a lattice
    of spacing 3 (spread over many 64-point Morton groups).

    * 'tie'     : b - a on the x axis, exactly d -+ eps (dyadic for (1, 0.25)), and 1, 2 floats either side;
    * 'prefilter': b - a = (x, y, 0) with fl(x^2 + y^2) stepping through the floats around lo^2 and hi^2 (the squared
                   pre-filter band of k_pairs) while fl(sqrt(.)) sits at the band's edge;
    * 'zero'    : d - eps <= 0: coincident points, tiny separations, and the upper tie.
    unit_binding: a cloud whose _ratio is exactly 4, so that eps / ratio is a power of two and the unit-cube test
    (|u_j - u_i| - nRadius)^2 < eps_round^2 is the one that rejects the exact ties (queries ((0.25, 0.0625),))."""
    pts, kinds = [], []
    site = [0]

    def add(sep_vec, kind, spacing=3.0, per_row=10):
        s = site[0]
        site[0] += 1
        a = np.array([0.0, spacing * (s % per_row), spacing * (s // per_row)], f32)
        b = (a + np.asarray(sep_vec, f32)).astype(f32)
        assert np.array_equal(b - a, np.asarray(sep_vec, f32)), "separation not exact"
        pts.extend([a, b])
        kinds.extend([kind, kind])

    if unit_binding:
        d, eps = 0.25, 0.0625
        for edge in (d - eps, d + eps):
            for k in KS:
                add([step(f32(edge), k), 0, 0], "tie", spacing=0.75, per_row=4)
        # clearly inside and outside the band, beyond the rounding of the unit coordinates
        for sep in (d, d - eps + 2.0 ** -12, d + eps - 2.0 ** -12, d - eps - 2.0 ** -12, d + eps + 2.0 ** -12):
            add([sep, 0, 0], "unit", spacing=0.75, per_row=4)
        # the bounding box 3.999 wide on x with centre 0: ratio = float(3.999f + 0.001) = 4, unit = x / 4 + 0.5 exactly
        h = f32(f32(3.999) / f32(2))
        pts.extend([np.array([-h, 1.1, 0.4], f32), np.array([h, 1.1, 0.4], f32)])
        kinds.extend(["box", "box"])
        Q = np.array(pts, f32)
        assert float(f32(float(Q[:, 0].max() - Q[:, 0].min()) + 0.001)) == 4.0
        return Q, ((d, eps),), np.array(kinds)

    for d, eps in PAIR_QUERIES:
        lo = max(0.0, float(f32(d)) - float(f32(eps)))
        hi = float(f32(d)) + float(f32(eps))
        edges = (hi,) if lo == 0.0 else (lo, hi)
        for edge in edges:
            for k in KS:
                add([step(f32(edge), k), 0, 0], "tie")
        if lo == 0.0:
            for sep in (0.0, 1e-30, 2.0 ** -20, 0.0625):
                add([sep, 0, 0], "zero")
            continue
        # fl(sq) on the floats around the pre-filter's squared bounds; x a float just inside the band
        for edge, inward in ((lo, 1), (hi, -1)):
            base = f32(edge * edge)
            lo_sq, hi_sq, _, _ = prefilter_bounds(d, eps)
            wanted = set(int(v) for v in ordinal(base) + np.arange(-3, 4))
            wanted |= set(int(v) for v in ordinal(lo_sq if inward > 0 else hi_sq) + np.arange(-1, 2))
            for x in (step(f32(edge), -inward * 2), step(f32(edge), -inward * 40)):
                ys = (np.arange(0, 6000) * f32(2.0 ** -19)).astype(f32)
                sq = x * x + (ys * ys + f32(0))        # dx^2 + (dy^2 + dz^2)
                o = ordinal(sq)
                for w in sorted(wanted):
                    hit = np.nonzero(o == w)[0]
                    if len(hit):
                        add([x, ys[hit[0]], 0], "prefilter")
    Q = np.array(pts, f32)
    return Q, PAIR_QUERIES, np.array(kinds)


def cull_pad(g):
    """the tile cull's pad in cells beyond r / h (verify.cu, tile_live)"""
    return max(f32(0.52), f32(0.5) + (g["vslack"] * g["inv_h"]) * f32(1.0001))


def coarse_face_cull_cases(name="offcentre1e4", n_faces=6, n_rot=24, seed=3):
    """(P, q, T34, g): P points on both sides of coarse-block faces of an off-centre cloud, one query q near the cloud,
    and candidates [R | m3] with small random rotations R and fl(R q + m3) exactly on the target: the P point's
    coordinate -+ delta across the face (an exact tie, d^2 = delta^2 on the coordinates' lattice).  Only the tile cull
    stands between such a query and the exact test, and its centre rounds at millions of voxels."""
    delta, centre, half = REGIMES[name]
    rng = np.random.RandomState(seed)
    corners = _corners(centre, half)
    g = grid_layout(corners, delta)
    lo, hi = corners.min(0).astype(np.float64), corners.max(0).astype(np.float64)
    cs = 1 << g["cshift"]
    anchors, targets = [], []
    while len(anchors) < 2 * n_faces:
        axis = rng.randint(3)
        p = rng.uniform(lo + 6 * delta, hi - 6 * delta)
        F = int(round((p[axis] - float(g["o"][axis])) * float(g["inv_h"]) / cs)) * cs
        up = first_in_cell(g, axis, F, face_coord(g, "coarse", axis, F // cs))
        down = step(up, -1)                                     # the last float of the block below
        a1, a2 = p.astype(f32), p.astype(f32)
        a2[(axis + 1) % 3] = f32(p[(axis + 1) % 3] + (12 * delta if p[(axis + 1) % 3] < centre[(axis + 1) % 3] else -12 * delta))
        a1[axis], a2[axis] = up, down
        if not all(np.abs(a.astype(np.float64) - b).max() > 8 * delta for a in (a1, a2) for b in anchors + list(corners)):
            continue
        t1, t2 = a1.copy(), a2.copy()
        t1[axis] = f32(up - f32(delta))                         # below the face, delta from the point above it
        t2[axis] = f32(down + f32(delta))                       # above the face, delta from the point below it
        anchors += [a1, a2]
        targets += [t1, t2]
    P = np.concatenate([corners, np.array(anchors, f32)])
    q = np.asarray(centre, f32)
    T = []
    for t in targets:
        for _ in range(n_rot):
            w = rng.standard_normal(3) * rng.uniform(0, 2e-3)
            K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
            R = (np.eye(3) + K + K @ K / 2)
            R = np.linalg.qr(R)[0] * np.sign(np.diag(np.linalg.qr(R)[1]))
            R = R.astype(f32)
            s = fp32_tq(np.concatenate([R, np.zeros((3, 1), f32)], 1), q)[0]
            m3 = (t.astype(np.float64) - s.astype(np.float64)).astype(f32)
            M = np.concatenate([R, m3[:, None]], 1).astype(f32)
            if np.array_equal(fp32_tq(M, q)[0], t):
                T.append(M)
    return P, q, np.array(T, f32), grid_layout(P, delta)
