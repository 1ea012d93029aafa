"""The quad search (FindCongruentQuadrilaterals over IndexedNormalSet<Point,3,7,float>) restated in numpy, and fixtures
that put each of its decisions within ulps of its boundary.

`find_quads` shares no code with oracle/port.cc or csrc/quads.cu.  It follows the reference's operation order
(reference algorithms/super4pcs.cc:80-177, accelerators/normalset.hpp:57-210, accelerators/utils.h:139-148):

* unit-cube coordinates u = (q - gcenter) / ratio + 0.5;
* grid: gridDepth = (int)-log2f(thr2 / ratio), egSize = 2^gridDepth, epsilon = 1 / egSize;
* P-pair key: cell of p1 + inv1 (p2 - p1) from (int)(pos / epsilon) per axis, direction bin of normalized(p2 - p1) from
  (int)(((n / 2) + 0.5) / nepsilon), nepsilon = float(1/7 + 1e-5);
* Q-pair: the query point's cell, the cone of nbSample directions at angle alpha = acosf(alpha_cos) around the Q-pair
  direction (glibc's acosf, atanf, sinf, cosf, mixed with the double M_PI as the reference does; at most 56 samples,
  NaN -> 0), rotated by Eigen's setFromTwoVectors((0, 0, 1), n) with its nearly-opposite (Householder) branch;
* distance: sqnorm(queryQ - invPoint) <= thr2 in sampled-Q coordinates against the UN-squared threshold;
* output in (index in pairs1, index in pairs2) order.

numpy rounds every float32 operation once and never fuses two, so this is the reference's arithmetic.  `mutant=` switches
one decision to a plausible wrong form, so that the tests can show which fixture tells each wrong form apart.
`find_quads64` evaluates the same predicate in float64 with a rotation matrix instead of a quaternion, as a check that
the float32 restatement does not inherit a misreading, and says how far each decision lies from its boundary.
"""
import ctypes
import math

import numpy as np

from tests import edges as E
from tests import pair_filters as F

f32 = np.float32
KS = E.KS
NEPS = f32(float(f32(1) / f32(7)) + 0.00001)
OPPOSITE = f32(f32(-1) + f32(1e-5))
MUTANTS = ("dist_lt", "bin_round", "opposite_le", "query_fma", "no_cap")
CATCHABLE = ("dist_lt", "bin_round", "opposite_le", "query_fma")    # no_cap changes nothing: nbSample never exceeds 56

_libm = ctypes.CDLL("libm.so.6")
for _fn in ("acosf", "atanf", "sinf", "cosf", "log2f"):
    getattr(_libm, _fn).restype = ctypes.c_float
    getattr(_libm, _fn).argtypes = [ctypes.c_float]


def _lm(name, x):
    return f32(getattr(_libm, name)(float(x)))


# ---- the restatement --------------------------------------------------------------------------------------------------
def normalization(Q):
    """gcenter, ratio of the unit cube (AlignedBox center, max extent + 0.001 in double)"""
    Q = np.asarray(Q, f32)
    mn, mx = Q.min(0), Q.max(0)
    return (mn + mx) / f32(2), f32(float((mx - mn).max()) + 0.001)


def unit(Q, gc, ratio):
    return ((np.asarray(Q, f32) - f32(gc)) / f32(ratio)) + f32(0.5)


def grid(thr2, ratio):
    """(depth, egSize, epsilon); depth outside 0..18 is an argument error of s4g_find_quads"""
    eps = f32(thr2) / f32(ratio)
    depth = int(-float(_lm("log2f", eps)))
    eg = 2 ** depth if 0 <= depth <= 62 else 0
    return depth, eg, (f32(1) / f32(eg) if eg else f32(0))


def alpha_cos(base):
    b = np.asarray(base, f32).reshape(4, 3)
    return F.dot(F.normalized(b[1] - b[0]), F.normalized(b[3] - b[2]))[()]


def n_samples(ac, mutant=None):
    alpha = _lm("acosf", ac)
    perimeter = f32(2.0 * math.pi * float(_lm("atanf", alpha)))
    nbf = f32(2) * np.ceil((perimeter * f32(7)) / f32(2))
    if not (nbf == nbf and nbf > 0):
        return 0
    return int(nbf) if mutant == "no_cap" else min(56, int(nbf))


def ring(ac, mutant=None):
    """(nbSample, 3) sample directions around +z (normalset.hpp:174-190)"""
    ns = n_samples(ac, mutant)
    if ns == 0:
        return np.zeros((0, 3), f32)
    alpha = _lm("acosf", ac)
    step = f32(2.0 * math.pi / float(f32(ns)))
    s = _lm("sinf", alpha)
    th = [f32(f32(a) * step) for a in range(ns)]
    return np.array([[s * _lm("cosf", t), s * _lm("sinf", t), f32(ac)] for t in th], f32)


def cell_coords(pos, epsilon):
    return np.asarray(pos, f32) / f32(epsilon)


def cell_of(pos, eg, epsilon):
    c = np.trunc(cell_coords(pos, epsilon)).astype(np.int64)
    return (c[..., 2] * eg + c[..., 1]) * eg + c[..., 0]


def bin_coords(n):
    return ((np.asarray(n, f32) / f32(2)) + f32(0.5)) / NEPS


def bin_of(n, mutant=None):
    c = bin_coords(n)
    c = np.rint(c) if mutant == "bin_round" else np.trunc(c)
    c = c.astype(np.int64)
    return (c[..., 2] * 7 + c[..., 1]) * 7 + c[..., 0]


def cross(a, b):
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _householder(v):
    """(essential part, tau, beta) of Eigen's makeHouseholder of the float32 vector v"""
    tail = v[1] * v[1]
    for x in v[2:]:
        tail = tail + x * x
    c0 = v[0]
    if tail <= f32(1.17549435e-38):
        return [f32(0)] * (len(v) - 1), f32(0), c0
    b = np.sqrt(c0 * c0 + tail)
    if c0 >= 0:
        b = -b
    return [x / (c0 - b) for x in v[1:]], (b - c0) / b, b


def _apply_left(M, off, ld, rows, cols, ess, tau):
    """applyHouseholderOnTheLeft on the rows x cols block of the flat list M at offset off, leading dimension ld"""
    if rows == 1:
        for j in range(cols):
            M[off + j] = M[off + j] * (f32(1) - tau)
        return
    if tau == 0:
        return
    tmp = []
    for j in range(cols):
        acc = None
        for i in range(rows - 1):
            t = ess[i] * M[off + (i + 1) * ld + j]
            acc = t if acc is None else acc + t
        tmp.append(acc + M[off + j])
    for j in range(cols):
        M[off + j] = M[off + j] - tau * tmp[j]
    for i in range(rows - 1):
        for j in range(cols):
            M[off + (i + 1) * ld + j] = M[off + (i + 1) * ld + j] - (tau * ess[i]) * tmp[j]


def null_axis(v0, v1):
    """third column of the Householder Q of the column-pivoted QR of [v0 | v1] (Eigen's JacobiSVD<2x3> with ComputeFullV
    in setFromTwoVectors: the Jacobi sweeps and the sort only touch the first two columns of V)"""
    v0, v1 = [f32(x) for x in v0], [f32(x) for x in v1]
    sc = max(abs(x) for x in v0 + v1)
    if sc == 0:
        sc = f32(1)
    A = [[v0[r] / sc, v1[r] / sc] for r in range(3)]
    nrm = [np.sqrt(A[0][k] * A[0][k] + (A[1][k] * A[1][k] + A[2][k] * A[2][k])) for k in range(2)]
    ess, tau = [None, None], [f32(0), f32(0)]
    for k in range(2):
        if k == 0 and nrm[1] > nrm[0]:
            for r in range(3):
                A[r][0], A[r][1] = A[r][1], A[r][0]
            nrm[0], nrm[1] = nrm[1], nrm[0]
        ess[k], tau[k], beta = _householder([A[r][k] for r in range(k, 3)])
        A[k][k] = beta
        if k == 0:
            M = [A[0][1], A[1][1], A[2][1]]
            _apply_left(M, 0, 1, 3, 1, ess[0], tau[0])
            A[0][1], A[1][1], A[2][1] = M
    Qm = [f32(1), f32(0), f32(0), f32(0), f32(1), f32(0), f32(0), f32(0), f32(1)]
    _apply_left(Qm, 4, 3, 2, 2, ess[1], tau[1])
    _apply_left(Qm, 0, 3, 3, 3, ess[0], tau[0])
    return np.array([Qm[2], Qm[5], Qm[8]], f32)


def quaternion(n, mutant=None):
    """(x, y, z, w), opposite: Eigen's setFromTwoVectors((0, 0, 1), n) for each row of n"""
    v0 = np.array([0, 0, 1], f32)
    v1 = F.normalized(n)
    c = F.dot(v1, v0[None])
    q = np.zeros((len(v1), 4), f32)
    opp = (c <= OPPOSITE) if mutant == "opposite_le" else (c < OPPOSITE)
    axis = cross(v0[None], v1)
    sq = np.sqrt((f32(1) + c) * f32(2))
    invs = f32(1) / sq
    with np.errstate(divide="ignore", invalid="ignore"):
        q[:, :3] = axis * invs[:, None]
        q[:, 3] = sq * f32(0.5)
    for i in np.nonzero(opp)[0]:
        ci = max(c[i], f32(-1))
        ax = null_axis(v0, v1[i])
        w2 = (f32(1) + ci) * f32(0.5)
        k = np.sqrt(f32(1) - w2)
        q[i, :3] = ax * k
        q[i, 3] = np.sqrt(w2)
    return q, opp


def rotate(q, v):
    """Eigen's _transformVector: v + w uv + qv x uv, uv = 2 (qv x v); q (n, 4), v (m, 3) -> (n, m, 3)"""
    qv = np.broadcast_to(q[:, None, :3], (len(q), len(v), 3))
    vv = np.broadcast_to(np.asarray(v, f32)[None], qv.shape)
    uv = cross(qv, vv)
    uv = uv + uv
    return (vv + q[:, None, 3:4] * uv) + cross(qv, uv)


def _invariant(a, b, inv, mutant=None):
    d = b - a
    if mutant == "query_fma":
        return (a.astype(np.float64) + np.float64(f32(inv)) * d.astype(np.float64)).astype(f32)
    return a + f32(inv) * d


def find_quads(Q, gc, ratio, pairs1, pairs2, inv1, inv2, thr2, base, mutant=None, detail=False):
    """(K, 4) quads (pairs1[id], pairs2[i]) in (id, i) order"""
    Q = np.asarray(Q, f32)
    pairs1, pairs2 = np.asarray(pairs1, np.int64).reshape(-1, 2), np.asarray(pairs2, np.int64).reshape(-1, 2)
    U = unit(Q, gc, ratio)
    depth, eg, epsilon = grid(thr2, ratio)
    if not 0 <= depth <= 18:
        raise ValueError("thr2 / ratio outside the grid depths 0 .. 18")
    ac = alpha_cos(base)
    R = ring(ac, mutant)
    # P-pairs: key, invariant point in sampled-Q coordinates
    p1, p2 = U[pairs1[:, 0]], U[pairs1[:, 1]]
    d = p2 - p1
    cellP = cell_of(p1 + f32(inv1) * d, eg, epsilon)
    binP = bin_of(F.normalized(d), mutant)
    qa, qb = Q[pairs1[:, 0]], Q[pairs1[:, 1]]
    invP = qa + (qb - qa) * f32(inv1)
    # Q-pairs: cell, cone mask, query point in sampled-Q coordinates
    u1, u2 = U[pairs2[:, 0]], U[pairs2[:, 1]]
    cellQ = cell_of(_invariant(u1, u2, inv2, mutant), eg, epsilon)
    queryQ = _invariant(Q[pairs2[:, 0]], Q[pairs2[:, 1]], inv2, mutant)
    quat, opp = quaternion(F.normalized(u2 - u1), mutant)
    mask = np.zeros((len(pairs2), 344), bool)
    if len(R) and len(pairs2):
        dirs = F.normalized(rotate(quat, R))
        b = bin_of(dirs, mutant)
        b = np.where((b >= 0) & (b < 343), b, 343)
        mask[np.arange(len(pairs2))[:, None], b] = True
    mask[:, 343] = False
    if len(pairs1) == 0 or len(pairs2) == 0 or len(R) == 0:
        hit = np.zeros((len(pairs1), len(pairs2)), bool)
    else:
        diff = queryQ[None, :, :] - invP[:, None, :]
        sq = F.sqn(diff)
        close = (sq < f32(thr2)) if mutant == "dist_lt" else (sq <= f32(thr2))
        hit = (cellP[:, None] == cellQ[None, :]) & mask[:, np.where((binP >= 0) & (binP < 343), binP, 343)].T & close
    ids, iq = np.nonzero(hit)
    quads = np.concatenate([pairs1[ids], pairs2[iq]], 1).astype(np.int32).reshape(-1, 4)
    if detail:
        return quads, dict(depth=depth, alpha_cos=ac, n_samples=len(R), opposite=opp, cellP=cellP, cellQ=cellQ,
                           binP=binP, mask=mask[:, :343], hit=hit)
    return quads


# ---- the same predicate in float64 --------------------------------------------------------------------------------------
def _rot64(n):
    """rotation matrices taking +z to each unit row of n (about z x n)"""
    out = np.zeros((len(n), 3, 3))
    for k, v in enumerate(n):
        a = np.cross([0.0, 0.0, 1.0], v)
        s, c = np.linalg.norm(a), v[2]
        if s == 0:
            out[k] = np.diag([1.0, 1.0, 1.0]) if c > 0 else np.diag([1.0, -1.0, -1.0])
            continue
        a /= s
        K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
        out[k] = np.eye(3) + s * K + (1 - c) * K @ K
    return out


def find_quads64(Q, gc, ratio, pairs1, pairs2, inv1, inv2, thr2, base):
    """(hit (n1, n2), margins (n1, n2)): the quad predicate in float64, and the relative distance of the nearest decision
    that (id, i) depends on from its boundary"""
    Q = np.asarray(Q, np.float64)
    pairs1, pairs2 = np.asarray(pairs1, np.int64).reshape(-1, 2), np.asarray(pairs2, np.int64).reshape(-1, 2)
    U = (Q - np.asarray(gc, np.float64)) / float(ratio) + 0.5
    depth = int(-math.log2(float(thr2) / float(ratio)))
    eg = 2.0 ** depth
    b = np.asarray(base, np.float64).reshape(4, 3)
    u, v = b[1] - b[0], b[3] - b[2]
    ac = float(np.dot(u / np.linalg.norm(u), v / np.linalg.norm(v)))
    alpha = math.acos(max(-1.0, min(1.0, ac)))
    per = 2 * math.pi * math.atan(alpha) * 3.5
    ns = min(56, 2 * math.ceil(per))
    th = np.arange(ns) * (2 * math.pi / ns) if ns else np.zeros(0)
    R = np.stack([math.sin(alpha) * np.cos(th), math.sin(alpha) * np.sin(th), np.full(ns, ac)], 1)

    def frac_margin(x):
        return np.abs(x - np.round(x)).min(-1)

    def unit_rows(x):
        return x / np.maximum(np.linalg.norm(x, axis=-1, keepdims=True), 1e-300)

    nep = float(NEPS)
    posP = U[pairs1[:, 0]] + inv1 * (U[pairs1[:, 1]] - U[pairs1[:, 0]])
    nP = unit_rows(U[pairs1[:, 1]] - U[pairs1[:, 0]])
    cP, bP = np.floor(posP * eg), np.floor((nP / 2 + 0.5) / nep)
    mP = np.minimum(frac_margin(posP * eg), frac_margin((nP / 2 + 0.5) / nep))
    posQ = U[pairs2[:, 0]] + inv2 * (U[pairs2[:, 1]] - U[pairs2[:, 0]])
    nQ = unit_rows(U[pairs2[:, 1]] - U[pairs2[:, 0]])
    cQ = np.floor(posQ * eg)
    dirs = np.einsum("kij,sj->ksi", _rot64(nQ), R)
    bS = np.floor((dirs / 2 + 0.5) / nep)
    mQ = frac_margin(posQ * eg)
    if ns:
        mQ = np.minimum(mQ, frac_margin((dirs / 2 + 0.5) / nep).min(-1))
    mQ = np.minimum(mQ, np.abs(nQ[:, 2] + 1 - 1e-5))
    mQ = np.where(np.linalg.norm(U[pairs2[:, 1]] - U[pairs2[:, 0]], axis=1) > 0, mQ, 0.0)   # no direction: no cone
    mQ = np.minimum(mQ, abs(per - round(per)))
    invP = Q[pairs1[:, 0]] + (Q[pairs1[:, 1]] - Q[pairs1[:, 0]]) * inv1
    qQ = Q[pairs2[:, 0]] + inv2 * (Q[pairs2[:, 1]] - Q[pairs2[:, 0]])
    sq = ((qQ[None, :, :] - invP[:, None, :]) ** 2).sum(-1)
    same_cell = (cP[:, None, :] == cQ[None, :, :]).all(-1)
    in_cone = (bP[:, None, None, :] == bS[None, :, :, :]).all(-1).any(-1) if ns else np.zeros(same_cell.shape, bool)
    hit = same_cell & in_cone & (sq <= float(thr2))
    margin = np.minimum(np.minimum(mP[:, None], mQ[None, :]), np.abs(sq - float(thr2)) / float(thr2))
    return hit, margin


# ---- fixtures ---------------------------------------------------------------------------------------------------------
H = f32(f32(3.999) / f32(2))           # box corners at +-H: gcenter = 0, ratio = float(3.999f + 0.001) = 4 exactly
CORNERS = np.array([[-H, -H, -H], [H, H, H]], f32)


def _cloud(*pts):
    Q = np.concatenate([CORNERS, np.asarray(pts, f32).reshape(-1, 3)]).astype(f32)
    gc, ratio = normalization(Q)
    assert ratio == 4 and not gc.any()
    return Q


def _world(u):
    """a world coordinate whose unit coordinate is about u"""
    return f32((np.asarray(u, np.float64) - 0.5) * 4.0)


def _walk(Q, point, axes, quantity, boundary, span=48, side=None, prefer0=None):
    """{k: Q'}: Q with coordinates `axes` of `point` moved by nextafter steps (+-span on the first axis, +-side, default
    span / 8, on the others) so that quantity(X), evaluated on the (m, 3) candidate positions X of the point, lies
    exactly k floats from `boundary`, k in KS (the candidate closest to the start among equals; at k = 0 one for which
    prefer0(X) holds, if there is one)"""
    side = span // 8 if side is None else side
    grids = np.meshgrid(*[np.arange(-span, span + 1) if j == 0 else np.arange(-side, side + 1)
                          for j in range(len(axes))], indexing="ij")
    offs = np.stack([g.ravel() for g in grids], 1)
    offs = offs[np.argsort(np.abs(offs).sum(1), kind="stable")]
    X = np.repeat(Q[point][None], len(offs), 0)
    for j, ax in enumerate(axes):
        X[:, ax] = E.step(Q[point, ax], offs[:, j])
    k = E.ordinal(np.asarray(quantity(X), f32)) - E.ordinal(f32(boundary))
    out = {}
    for kk in KS:
        hit = np.nonzero(k == kk)[0]
        if kk == 0 and prefer0 is not None and len(hit):
            hit = hit[np.argsort(~np.asarray(prefer0(X[hit]), bool), kind="stable")]
        if len(hit):
            Qc = Q.copy()
            Qc[point] = X[hit[0]]
            out[kk] = Qc
    return out


def _cone_dir(nq, base):
    """a cone sample direction of the Q-pair direction nq (unit coordinates) whose bin coordinates are furthest from a
    bin face: a P-pair along it has its bin in the Q-pair's mask"""
    q, _ = quaternion(F.normalized(np.asarray(nq, f32))[None])
    dirs = F.normalized(rotate(q, ring(alpha_cos(base))))[0]
    c = bin_coords(dirs)
    return dirs[int(np.argmax(np.abs(c - np.floor(c) - 0.5).max(1) * -1))].astype(np.float64)


def _fixture(family, name, Q, pairs1, pairs2, inv1, inv2, thr2, base, k=None, probe=None, decide=None):
    return dict(family=family, name=name, Q=np.asarray(Q, f32), pairs1=np.asarray(pairs1, np.int32).reshape(-1, 2),
                pairs2=np.asarray(pairs2, np.int32).reshape(-1, 2), inv1=f32(inv1), inv2=f32(inv2), thr2=f32(thr2),
                base=np.asarray(base, f32).reshape(4, 3), k=k, probe=probe, decide=decide)


def run(fx, mutant=None, detail=False):
    gc, ratio = normalization(fx["Q"])
    return find_quads(fx["Q"], gc, ratio, fx["pairs1"], fx["pairs2"], fx["inv1"], fx["inv2"], fx["thr2"], fx["base"],
                      mutant=mutant, detail=detail)


def decision(fx, mutant=None):
    """the fixture's designed decision as the restatement takes it (its `decide` key, default: is the probe a quad)"""
    if fx["decide"] == "depth":
        return grid(fx["thr2"], normalization(fx["Q"])[1])[0]
    q, info = run(fx, mutant, detail=True)
    if fx["decide"] == "n_samples":
        return info["n_samples"]
    if fx["decide"] == "opposite":
        return bool(info["opposite"][fx["probe"][1]])
    return bool(info["hit"][fx["probe"][0], fx["probe"][1]])


def _base_alpha(ac):
    """base points whose alpha_cos is exactly the float ac (segment 1 along +x: alpha_cos = normalized(b3 - b2).x)"""
    b0, b1, b2 = np.zeros(3, f32), np.array([1, 0, 0], f32), np.array([0, 0.5, 0], f32)
    ac = f32(ac)
    if abs(float(ac)) == 1.0:
        return np.stack([b0, b1, b2, (b2 + np.array([ac, 0, 0], f32)).astype(f32)])
    if ac == 0:
        return np.stack([b0, b1, b2, (b2 + np.array([0, 1, 0], f32)).astype(f32)])
    b3 = F.search_b2(b2, np.array([1, 0, 0], f32), ac, 1.0, side=24)
    assert b3 is not None, ("alpha_cos not reached", float(ac))
    base = np.stack([b0, b1, b2, b3])
    assert alpha_cos(base) == ac
    return base


def _alpha_base(alpha):
    return np.array([[0, 0, 0], [1, 0, 0], [0, 0.5, 0], [math.cos(alpha), 0.5 + math.sin(alpha), 0]], f32)


def _two_pairs(qa, qb, pa, pb):
    """cloud corners + one Q-pair (2, 3) and one P-pair (4, 5)"""
    return _cloud(qa, qb, pa, pb), [[4, 5]], [[2, 3]]


def _U(X):
    return unit(X, np.zeros(3, f32), f32(4))


INV = f32(0.3)                          # the invariants of the cell-face fixtures (0.5 would make a fused p1 + inv d exact)


def cell_face_fixtures(depths=(2, 4, 6)):
    """the invariant point of the P-pair (side 'P') or of the Q-pair (side 'Q') at pos / epsilon = an integer on each
    axis, the other invariant point inside the upper cell; the P-pair along a sample direction of the Q-pair's cone"""
    out = []
    base = _alpha_base(0.3)
    u = F.normalized(np.array([0.3, 0.5, 0.8], f32)).astype(np.float64)
    v = _cone_dir(u, base)
    for depth in depths:
        thr2 = f32(4.0 * 0.75 * 2.0 ** -depth)                  # thr2 / ratio = 0.75 * 2^-depth
        eg = 2 ** depth
        cellw = 1.0 / eg
        assert grid(thr2, f32(4))[0] == depth
        for axis in range(3):
            for side in ("P", "Q"):
                m = eg // 2 + 1                                  # the face between cells m - 1 and m
                face = np.full(3, (m + 0.4) * cellw)
                face[axis] = m * cellw
                other = face.copy()
                other[axis] = (m + 0.3) * cellw
                L = 0.2 * cellw
                q_at, p_at = (other, face) if side == "P" else (face, other)
                Q, p1, p2 = _two_pairs(_world(q_at - 0.3 * L * u), _world(q_at + 0.7 * L * u),
                                       _world(p_at - 0.3 * L * v), _world(p_at + 0.7 * L * v))
                pt = 4 if side == "P" else 2

                def quantity(X, Q=Q, pt=pt, axis=axis, cellw=cellw):
                    a, b = _U(X), _U(Q[pt + 1])[None]
                    return cell_coords(a + INV * (b - a), f32(cellw))[:, axis]
                for k, Qk in _walk(Q, pt, [axis], quantity, f32(m), span=600).items():
                    out.append(_fixture("cell_face", "cell-d%d-%s-ax%d-k%+d" % (depth, side, axis, k), Qk, p1, p2,
                                        INV, INV, thr2, base, k=k, probe=(0, 0)))
    return out


def _bin_edges(nq, base):
    """(sample, axis, face, across, direction) candidates: a sample of the cone of nq, an axis, the bin face nearest to the
    sample's bin coordinate on it, whether the bin across the face is in the mask, the sample's direction"""
    q, _ = quaternion(F.normalized(np.asarray(nq, f32))[None])
    dirs = F.normalized(rotate(q, ring(alpha_cos(base))))[0]
    c = bin_coords(dirs)
    bins = bin_of(dirs)
    mask = set(bins.tolist())
    out = []
    for s in range(len(dirs)):
        for axis in range(3):
            rest = [j for j in range(3) if j != axis]
            if (np.abs(c[s, rest] - np.floor(c[s, rest]) - 0.5) > 0.35).any():
                continue
            face = int(np.round(c[s, axis]))
            if not 1 <= face <= 6:
                continue
            cc = np.trunc(c[s]).astype(int)
            cc[axis] = face - 1 if cc[axis] == face else face
            across = int((cc[2] * 7 + cc[1]) * 7 + cc[0])
            out.append((s, axis, face, across in mask, dirs[s].astype(np.float64)))
    return out


def bin_face_fixtures():
    """a P-pair direction component at a direction-bin face whose other side is outside the cone mask (side 'P'), and a
    cone sample's component at a bin face, reached by walking the Q-pair's direction, with the P-pair in the bin across
    the face, outside the mask otherwise (side 'S'); one cell (depth 0)"""
    out = []
    thr2 = f32(3.0)
    base = _alpha_base(0.1)
    centre = np.array([0.1, 0.05, -0.1])
    rng = np.random.RandomState(4)
    for j, nq in enumerate(rng.standard_normal((12, 3))):
        nq = F.normalized(np.array(nq, f32)).astype(np.float64)
        cands = _bin_edges(nq, base)
        used = set()
        for side in ("P", "S"):
            for (s, axis, face, across_in, d) in cands:
                if across_in or (side, axis) in used:
                    continue
                used.add((side, axis))
                qa, qb = centre - 0.25 * nq, centre + 0.25 * nq
                rest = [a for a in range(3) if a != axis]
                cross_bin = face - 1 if int(np.trunc(bin_coords(f32(d))[axis])) == face else face

                def towards(t, d=d, axis=axis, rest=rest):
                    """d with its `axis` component t after normalization"""
                    p = d.copy()
                    p[axis] = t
                    p[rest] *= math.sqrt(1 - t * t) / np.linalg.norm(d[rest])
                    return p
                if side == "P":                                  # P along the sample, its component at the face
                    pdir = towards(face * float(NEPS) * 2 - 1)
                    Q, p1, p2 = _two_pairs(qa, qb, centre - 0.25 * pdir, centre + 0.25 * pdir)

                    def quantity(X, Q=Q, axis=axis):
                        return bin_coords(F.normalized(_U(X) - _U(Q[4])[None]))[:, axis]
                    walked = _walk(Q, 5, [axis] + rest, quantity, f32(face), span=48, side=32)
                else:                                            # P in the bin across, the sample walked to the face
                    t_face = face * float(NEPS) * 2 - 1
                    n2 = nq.copy()
                    for _ in range(8):                           # turn the Q-pair until the sample is at the face
                        qq, _o = quaternion(F.normalized(f32(n2))[None])
                        ds = F.normalized(rotate(qq, ring(alpha_cos(base))[s:s + 1]))[0, 0].astype(np.float64)
                        n2[axis] += t_face - ds[axis]
                        n2 /= np.linalg.norm(n2)
                    qa, qb = centre - 0.25 * n2, centre + 0.25 * n2
                    pdir = ds.copy()
                    pdir[axis] = (cross_bin + 0.5) * float(NEPS) * 2 - 1
                    pdir[rest] *= math.sqrt(1 - pdir[axis] ** 2) / np.linalg.norm(ds[rest])
                    Q, p1, p2 = _two_pairs(qa, qb, centre - 0.25 * pdir, centre + 0.25 * pdir)
                    R = ring(alpha_cos(base))[s:s + 1]

                    def quantity(X, Q=Q, axis=axis, R=R):
                        q, _ = quaternion(F.normalized(_U(X) - _U(Q[2])[None]))
                        return bin_coords(F.normalized(rotate(q, R))[:, 0])[:, axis]
                    walked = _walk(Q, 3, [axis] + rest, quantity, f32(face), span=48, side=32)
                for k, Qk in walked.items():
                    out.append(_fixture("bin_face", "bin-%s-%d-ax%d-k%+d" % (side, j, axis, k), Qk, p1, p2, 0.5, 0.5,
                                        thr2, base, k=k, probe=(0, 0)))
    return out


def distance_fixtures():
    """sqnorm(queryQ - invPoint) at thr2 and 1, 2 floats either side, at depths 0 and 1"""
    out = []
    base = _alpha_base(0.3)
    u = F.normalized(np.array([0.2, 0.9, 0.4], f32)).astype(np.float64)
    v = _cone_dir(u, base)
    for thr2 in (f32(3.0), f32(1.5), f32(2.7182817)):
        r = math.sqrt(float(thr2))
        c = np.array([0.2, 0.15, 0.1])
        off = np.array([0.8, 0.4, 0.45]) / np.linalg.norm([0.8, 0.4, 0.45])
        Q, p1, p2 = _two_pairs(c - 0.1 * u, c + 0.1 * u, c + r * off - 0.1 * v, c + r * off + 0.1 * v)

        def quantity(X, Q=Q):
            qQ = Q[2] + f32(0.5) * (Q[3] - Q[2])
            iP = Q[4][None] + (X - Q[4][None]) * f32(0.5)
            return F.sqn(qQ[None] - iP)
        for k, Qk in _walk(Q, 5, [0, 1, 2], quantity, thr2, span=64).items():
            out.append(_fixture("distance", "dist-%g-k%+d" % (thr2, k), Qk, p1, p2, 0.5, 0.5, thr2, base, k=k,
                                probe=(0, 0)))
    return out


def fused_fixtures():
    """a long Q-pair whose query point p1 + 0.3 (p2 - p1) is at a cell face on x (depth 2), where the product 0.3 (p2 - p1)
    is large enough that fmaf(0.3, p2 - p1, p1) rounds differently from the reference's two roundings: at k = 0 the
    walk takes such a position if there is one"""
    out = []
    base = _alpha_base(0.3)
    thr2 = f32(4.0 * 0.75 * 2.0 ** -2)
    for j, (dy, dz) in enumerate(((0.1, 0.05), (-0.07, 0.12), (0.15, -0.1))):
        a = np.array([0.29, 0.4, 0.45])
        b = a + np.array([0.7, dy, dz])
        u = F.normalized(f32(b - a)).astype(np.float64)
        v = _cone_dir(u, base)
        pc = np.array([0.55, 0.4 + 0.3 * dy, 0.45 + 0.3 * dz])           # the P invariant in the same cell, x > 0.5
        Q, p1, p2 = _two_pairs(_world(a), _world(b), _world(pc - 0.3 * 0.05 * v), _world(pc + 0.7 * 0.05 * v))

        def quantity(X, Q=Q):
            x, y = _U(X), _U(Q[3])[None]
            return cell_coords(x + INV * (y - x), f32(0.25))[:, 0]

        def fused_below(X, Q=Q):
            x, y = _U(X), _U(Q[3])[None]
            return cell_coords(_invariant(x, y, INV, "query_fma"), f32(0.25))[:, 0] < f32(2)
        for k, Qk in _walk(Q, 2, [0], quantity, f32(2), span=3000, prefer0=fused_below).items():
            out.append(_fixture("fused", "fused-%d-k%+d" % (j, k), Qk, p1, p2, INV, INV, thr2, base, k=k, probe=(0, 0)))
    return out


def crowd(n=24, seed=0, spread=1.6):
    """n random points in the box (with its corners): every ordered pair is a P-pair and a Q-pair"""
    rng = np.random.RandomState(seed)
    Q = _cloud(rng.uniform(-spread, spread, (n - 2, 3)))
    i, j = np.meshgrid(np.arange(len(Q)), np.arange(len(Q)), indexing="ij")
    pairs = np.stack([i.ravel(), j.ravel()], 1)
    return Q, pairs[pairs[:, 0] != pairs[:, 1]]


def _sample_steps():
    """{n: (x_lo, x_hi)}: alpha_cos floats with n_samples(x_lo) == n and n_samples(x_hi) == n - 2, x_hi the next float,
    for n = 2 .. 56 (n_samples falls as alpha_cos rises)"""
    out = {}
    lo_o, hi_o = int(E.ordinal(f32(-1))), int(E.ordinal(f32(1)))
    for n in range(2, 57, 2):
        lo, hi = lo_o, hi_o                              # n_samples(lo) >= n > n_samples(hi)
        if n_samples(f32(E.from_ordinal(lo))) < n:
            continue
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if n_samples(f32(E.from_ordinal(mid))) >= n:
                lo = mid
            else:
                hi = mid
        out[n] = (f32(E.from_ordinal(lo)), f32(E.from_ordinal(hi)))
    return out


def cone_fixtures():
    """every step of nbSample (0 .. 56) at -2 .. +2 floats of alpha_cos around it; alpha_cos = 1, 1 - ulp, above 1 (NaN),
    -1 and 0; on the crowded cloud at depth 0"""
    Q, pairs = crowd()
    thr2 = f32(3.0)
    out = []
    steps = _sample_steps()
    for n, (x_lo, x_hi) in steps.items():
        for k in KS:
            x = E.step(x_lo if k <= 0 else x_hi, k if k <= 0 else k - 1)   # k <= 0: at or below x_lo, k > 0: from x_hi on
            if abs(float(x)) > 1:
                continue
            out.append(_fixture("cone", "cone-n%d-k%+d" % (n, k), Q, pairs, pairs, 0.5, 0.5, thr2, _base_alpha(x), k=k,
                                decide="n_samples"))
    rng = np.random.RandomState(7)
    above = None
    while above is None:                                    # fl(normalized(w) . normalized(w)) > 1
        w = rng.standard_normal(3).astype(f32)
        if F.dot(F.normalized(w), F.normalized(w)) > 1:
            above = w
    specials = {"ac_one": _base_alpha(1), "ac_below_one": _base_alpha(E.step(f32(1), -1)),
                "ac_above_one": np.stack([np.zeros(3, f32), above, np.zeros(3, f32), above]),
                "ac_minus_one": _base_alpha(-1), "ac_zero": _base_alpha(0)}
    for name, base in specials.items():
        out.append(_fixture("cone", name, Q, pairs, pairs, 0.5, 0.5, thr2, base, decide="n_samples"))
    return out


def opposite_fixtures():
    """Q-pair directions whose z component c is at -1 + 1e-5 and 1, 2 floats either side (Eigen's nearly-opposite
    branch of setFromTwoVectors), against the crowded cloud's P-pairs"""
    Qc, pairs = crowd(n=40, seed=3)
    thr2 = f32(3.0)
    out = []
    # at c = -1 + 1e-5 the regular branch loses most of 1 + c to cancellation: its rotation takes +z about 0.07 rad away
    # from the nearly-opposite branch's, which moves the samples of a narrow cone across bin faces in some directions
    for j, (phi, alpha) in enumerate(((0.0, 0.15), (0.93, 0.15), (1.88, 0.15), (2.5, 0.4), (3.6, 0.4), (4.4, 0.15),
                                      (5.3, 0.4), (6.0, 0.15))):
        base = _alpha_base(alpha)
        sx, sy = math.cos(phi), math.sin(phi)
        s = math.sqrt(1 - (1 - 1e-5) ** 2)
        n = np.array([sx * s, sy * s, -(1 - 1e-5)])
        a = np.array([0.2, -0.1, 0.9])
        Q = np.concatenate([Qc, np.array([a, a + 1.5 * n], f32)]).astype(f32)
        qi = len(Q) - 2

        def quantity(X, Q=Q, qi=qi):
            return F.normalized(F.normalized(_U(X) - _U(Q[qi])[None]))[:, 2]      # setFromTwoVectors normalizes again
        for k, Qk in _walk(Q, qi + 1, [0], quantity, OPPOSITE, span=6000).items():
            p2 = np.array([[qi, qi + 1]], np.int32)
            out.append(_fixture("opposite", "opp-%d-k%+d" % (j, k), Qk, pairs, p2, 0.5, 0.5, thr2, base, k=k,
                                probe=(0, 0), decide="opposite"))
    return out


def _depth_step(d):
    """the smallest float e = thr2 / ratio whose grid depth is <= d (the next float below has depth d + 1)"""
    lo, hi = int(E.ordinal(f32(2.0 ** -(d + 3)))), int(E.ordinal(f32(2.0 ** -(d - 2))))
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if grid(f32(4) * E.from_ordinal(mid), f32(4))[0] <= d:
            hi = mid
        else:
            lo = mid
    return f32(E.from_ordinal(hi))


def depth_fixtures():
    """grid depths 0, 1, 14, 15, 18 on the crowded cloud (beyond 14 the batched keys fall back), and thr2 / ratio at the
    steps from depth 0 to the error below it (near 2: the depth is truncated towards zero), 14 to 15 and 18 to the error
    beyond it (log2f rounds, so a step lies a few floats above its power of two)"""
    Q, pairs = crowd(n=20, seed=5)
    base = _alpha_base(0.7)
    out = []
    for depth in (0, 1, 14, 15, 18):
        thr2 = f32(4.0 * 0.75 * 2.0 ** -depth)
        assert grid(thr2, f32(4))[0] == depth
        out.append(_fixture("depth", "depth-%d" % depth, Q, pairs, pairs, 0.5, 0.5, thr2, base))
    for d in (-1, 14, 18):
        e = _depth_step(d)
        for k in KS:
            thr2 = f32(4) * E.step(e, k)                         # k >= 0: depth d, k < 0: depth d + 1
            out.append(_fixture("depth_edge", "depth-edge-%d-k%+d" % (d, k), Q, pairs, pairs, 0.5, 0.5, thr2, base,
                                k=k, decide="depth"))
    return out


def crowded_fixtures():
    """several entries per cell and bin, duplicate and zero-length pairs, coincident points, clouds of 2 to 40 points,
    invariants other than 0.5"""
    out = []
    rng = np.random.RandomState(11)
    for n in (2, 3, 5, 9, 17, 40):
        Q, pairs = crowd(n=n, seed=n, spread=0.3)
        out.append(_fixture("crowd", "crowd-%d" % n, Q, pairs, pairs, 0.5, 0.5, f32(0.9), _alpha_base(0.5)))
    Q, pairs = crowd(n=16, seed=2, spread=0.6)
    Q = np.concatenate([Q, Q[2:6]]).astype(f32)                 # coincident points
    extra = np.array([[2, 2], [3, 3], [2, len(Q) - 4], [len(Q) - 4, 2]], np.int32)  # zero-length pairs
    p = np.concatenate([pairs, extra, pairs[:40]])              # and duplicates
    for inv1, inv2 in ((0.5, 0.5), (0.2, 0.7), (0.0, 1.0), (0.93, 0.11)):
        out.append(_fixture("crowd", "dup-%g-%g" % (inv1, inv2), Q, p, p[rng.permutation(len(p))], inv1, inv2, f32(0.6),
                            _alpha_base(0.9)))
    return out


FAMILIES = {"cell_face": cell_face_fixtures, "bin_face": bin_face_fixtures, "distance": distance_fixtures,
            "cone": cone_fixtures, "opposite": opposite_fixtures, "fused": fused_fixtures, "depth": depth_fixtures,
            "crowd": crowded_fixtures}
_cache = {}


def fixtures(family):
    if family not in _cache:
        _cache[family] = FAMILIES[family]()
    return _cache[family]


def all_fixtures():
    return [fx for fam in FAMILIES for fx in fixtures(fam)]


# ---- the batched quad keys and offsets, emulated on the host -----------------------------------------------------------
ID_BITS = 26


def pack_quad_key(base, pid, qid):
    """k_bquad_query's key base << 52 | id << 26 | i in 64 bits"""
    return ((np.uint64(base) << np.uint64(2 * ID_BITS)) | (np.uint64(pid) << np.uint64(ID_BITS)) | np.uint64(qid))


def unpack_quad_key(k):
    """k_bquad_emit's reading: (base, id, i)"""
    k = np.uint64(k)
    m = np.uint64((1 << ID_BITS) - 1)
    return int(k >> np.uint64(2 * ID_BITS)), int((k >> np.uint64(ID_BITS)) & m), int(k & m)


def scan32(counts):
    """the uint32 exclusive scan of the per-entry quad counts and its last element (the batch total it reports)"""
    c = np.asarray(counts, np.uint64)
    off = (np.concatenate([np.zeros(1, np.uint64), np.cumsum(c, dtype=np.uint64)]) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return off, int(off[-1])
