"""Builds and runs tests/cpp/fpfh_main.cc, the test program of Utils::ComputeFPFH and Utils::MatchFPFH, for
tests/test_fpfh_cpu.py (on the oracle stand-in) and tests/test_fpfh_gpu.py (on the real library).  Also restatements that
share no code with the port: Open3D's formulas in numpy float64 (atan2, acos, hist_incr added per pair, S_h interleaved
with the sums), the s4g_fpfh contract in plain Python doubles, and the match in numpy float32 column by column."""
import math

import numpy as np

from tests import cpp_main

_f = np.float32

# c_i, s_i of beta_i = -pi + 2 pi i / 11, i = 1..5 (include/s4g.h), as the contract tabulates them
FACE_C = [float.fromhex(h) for h in ("-0x1.aeb8c8764f0bap-1", "-0x1.a9628d9c712b6p-2", "0x1.2375f640f44dbp-3",
                                     "0x1.4f49e7f775887p-1", "0x1.eb42a9bcd5057p-1")]
FACE_S = [float.fromhex(h) for h in ("-0x1.14cedf8bb580bp-1", "-0x1.d1bb48eee2c13p-1", "-0x1.fac9e043842efp-1",
                                     "-0x1.82f19bb3a28a1p-1", "-0x1.207e7fd768dbfp-2")]


def face(i):
    """(c_i, s_i) for i = 1..10"""
    return (FACE_C[i - 1], FACE_S[i - 1]) if i <= 5 else (FACE_C[10 - i], -FACE_S[10 - i])


def build(outdir):
    return cpp_main.build("fpfh_main", outdir)


def run_compute(exe, workdir, xyz, normals, k, max_distance=np.inf, preload=None):
    """-> None when ComputeFPFH threw, else its descriptors [n, 33] float32"""
    xyz = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    payload = np.int32(len(xyz)).tobytes() + xyz.tobytes() + np.ascontiguousarray(normals, _f).tobytes()
    r = cpp_main.Reader(cpp_main.run(exe, workdir, payload, ["compute", str(int(k)), repr(float(max_distance))], preload))
    if r.take(np.int32, 1)[0]:
        return None
    return r.take(_f, 33 * len(xyz)).reshape(-1, 33)


def run_match(exe, workdir, source, target, mutual=True, preload=None):
    """-> None when MatchFPFH threw, else its indices [n_source] int32"""
    S = np.ascontiguousarray(source, _f).reshape(-1, 33)
    T = np.ascontiguousarray(target, _f).reshape(-1, 33)
    payload = np.int32(len(S)).tobytes() + np.int32(len(T)).tobytes() + S.tobytes() + T.tobytes()
    r = cpp_main.Reader(cpp_main.run(exe, workdir, payload, ["match", str(int(bool(mutual)))], preload))
    if r.take(np.int32, 1)[0]:
        return None
    return r.take(np.int32, len(S))


# ---- surfaces

def surface(n, seed=0, bumps=4):
    """n points of a smooth random height field over [-1, 1]^2 (a sum of a few sinusoids), in random order"""
    rng = np.random.RandomState(seed)
    uv = rng.uniform(-1, 1, (n, 2))
    z = np.zeros(n)
    for _ in range(bumps):
        f, ph, a = rng.uniform(1, 4, 2), rng.uniform(0, 2 * np.pi, 2), rng.uniform(0.05, 0.2)
        z += a * np.sin(f[0] * uv[:, 0] + ph[0]) * np.cos(f[1] * uv[:, 1] + ph[1])
    return np.concatenate([uv, z[:, None]], 1).astype(_f)


# ---- Open3D's formulas in numpy float64

def _unit(N):
    N = np.asarray(N, np.float64)
    has = np.isfinite(N).all(1) & (N != 0).any(1)
    out = np.zeros_like(N)
    out[has] = N[has] / np.sqrt((N[has] ** 2).sum(1))[:, None]
    return out, has


def open3d_pairs(P, N, rows):
    """-> (bins [n, k, 3], valid [n, k], margin [n, k]): Open3D's ComputePairFeatures and bins for every row entry, and
    each pair's distance to the nearest decision face (the swap |a1| = |a2|, an f1 face in radians, an f2 or f3 face)"""
    P = np.asarray(P, _f).astype(np.float64)
    U, has = _unit(N)
    n, k = rows.shape
    r = np.where(rows >= 0, rows, 0)
    valid = (rows >= 0) & has[r] & has[:, None]
    p1, n1 = P[:, None, :], np.broadcast_to(U[:, None, :], (n, k, 3))
    p2, n2 = P[r], U[r]
    dp = p2 - p1
    d = np.sqrt((dp * dp).sum(-1))
    with np.errstate(all="ignore"):
        a1 = (n1 * dp).sum(-1) / d
        a2 = (n2 * dp).sum(-1) / d
        swap = np.arccos(np.abs(a1)) > np.arccos(np.abs(a2))
        u = np.where(swap[..., None], n2, n1)
        m = np.where(swap[..., None], n1, n2)
        dp = np.where(swap[..., None], -dp, dp)
        f3 = np.where(swap, -a2, a1)
        v = np.cross(dp, u)
        vn = np.sqrt((v * v).sum(-1))
        v = v / vn[..., None]
        w = np.cross(u, v)
        f2 = (v * m).sum(-1)
        f1 = np.arctan2((w * m).sum(-1), (u * m).sum(-1))
        zero = (d == 0) | (vn == 0)
        f1, f2, f3 = np.where(zero, 0.0, f1), np.where(zero, 0.0, f2), np.where(zero, 0.0, f3)
        t1 = 11 * (f1 + np.pi) / (2 * np.pi)
        t2, t3 = 11 * (f2 + 1.0) * 0.5, 11 * (f3 + 1.0) * 0.5
        b = np.stack([np.clip(np.floor(t), 0, 10) for t in (t1, t2, t3)], -1).astype(np.int64)
        b[..., 1] += 11
        b[..., 2] += 22
        edge = lambda t: np.abs(t - np.round(t))  # noqa: E731
        gap = np.abs(np.abs(a1) - np.abs(a2))
        gap = np.where(gap == 0, np.inf, gap)              # equal: neither form swaps (e.g. two equal normals)
        margin = np.minimum.reduce([gap, edge(t1) * 2 * np.pi / 11, edge(t2) / 5.5,
                                    edge(t3) / 5.5])
    margin = np.where(zero, np.inf, margin)
    return b, valid, np.where(valid, margin, np.inf)


def open3d_fpfh(P, N, rows, sq):
    """-> (fpfh [n, 33] float64, spfh [n, 33] float64, margin [n, k]) in Open3D's order: hist_incr = 100 / m added per
    pair, the FPFH sums with S_h accumulated interleaved with them, then acc * (100 / S_h) + spfh"""
    bins, valid, margin = open3d_pairs(P, N, rows)
    n, k = rows.shape
    m = valid.sum(1)
    incr = np.where(m > 0, 100.0 / np.maximum(m, 1), 0.0)
    spfh = np.zeros((n, 33))
    idx = np.arange(n)
    for e in range(k):
        for c in range(3):
            np.add.at(spfh, (idx[valid[:, e]], bins[valid[:, e], e, c]), incr[valid[:, e]])
    acc, S = np.zeros((n, 33)), np.zeros((n, 3))
    r = np.where(rows >= 0, rows, 0)
    sq = np.asarray(sq, _f).astype(np.float64)
    for e in range(k):
        use = valid[:, e] & (sq[:, e] > 0)
        for b in range(33):
            val = np.where(use, spfh[r[:, e], b] / np.where(use, sq[:, e], 1.0), 0.0)
            S[:, b // 11] += val
            acc[:, b] += val
    with np.errstate(divide="ignore"):
        scale = np.where(S != 0, 100.0 / S, 0.0)
    return acc * np.repeat(scale, 11, 1) + spfh, spfh, margin


# ---- the s4g_fpfh contract in plain Python doubles

def contract_f1_bin(x, y):
    if y == 0.0:
        return 10 if x < 0.0 else 5
    if y > 0.0:
        return 5 + sum(1 for i in range(6, 11) if face(i)[0] * y - face(i)[1] * x >= 0.0)
    return sum(1 for i in range(1, 6) if face(i)[0] * y - face(i)[1] * x >= 0.0)


def contract_bin(f):
    return int(min(max(math.floor(11 * (f + 1.0) * 0.5), 0), 10))


def _dot(a, b):
    return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]


def _cross(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def contract_normal(nv):
    x, y, z = (float(c) for c in nv)
    if not all(math.isfinite(c) for c in (x, y, z)) or (x == 0.0 and y == 0.0 and z == 0.0):
        return None
    n = (x, y, z)
    ln = math.sqrt(_dot(n, n))
    return (x / ln, y / ln, z / ln)


def contract_pair(p1, n1, p2, n2):
    """the three bins of a pair under the contract (unit normals in double, points as floats)"""
    dp = tuple(float(b) - float(a) for a, b in zip(p1, p2))
    d = math.sqrt(_dot(dp, dp))
    if d == 0.0:
        return 5, 16, 27
    a1, a2 = _dot(n1, dp) / d, _dot(n2, dp) / d
    if abs(a1) < abs(a2):
        u, m, dp, f3 = n2, n1, tuple(-c for c in dp), -a2
    else:
        u, m, f3 = n1, n2, a1
    v = _cross(dp, u)
    vn = math.sqrt(_dot(v, v))
    if vn == 0.0:
        return 5, 16, 27
    v = tuple(c / vn for c in v)
    w = _cross(u, v)
    return contract_f1_bin(_dot(u, m), _dot(w, m)), 11 + contract_bin(_dot(v, m)), 22 + contract_bin(f3)


def contract_fpfh(P, N, rows, sq):
    """-> [n, 33] float32: the s4g_fpfh contract in Python doubles, for small clouds"""
    P = np.asarray(P, _f)
    n, k = rows.shape
    U = [contract_normal(v) for v in np.asarray(N, _f)]
    spfh = [[0.0] * 33 for _ in range(n)]
    for j in range(n):
        if U[j] is None:
            continue
        cnt, m = [0] * 33, 0
        for e in range(k):
            i = int(rows[j, e])
            if i < 0:
                break
            if U[i] is None:
                continue
            for b in contract_pair(P[j], U[j], P[i], U[i]):
                cnt[b] += 1
            m += 1
        if m:
            spfh[j] = [(100.0 * c) / m for c in cnt]
    out = np.zeros((n, 33), _f)
    for j in range(n):
        if U[j] is None:
            continue
        acc = [0.0] * 33
        for e in range(k):
            i = int(rows[j, e])
            if i < 0:
                break
            d2 = float(sq[j, e])
            if U[i] is None or not d2 > 0.0:
                continue
            acc = [a + s / d2 for a, s in zip(acc, spfh[i])]
        for h in range(3):
            S = 0.0
            for b in range(11 * h, 11 * h + 11):
                S = S + acc[b]
            for b in range(11 * h, 11 * h + 11):
                out[j, b] = acc[b] * (100.0 / S) + spfh[j][b] if S != 0.0 else spfh[j][b]
    return out


# ---- the match in numpy float32

def match_numpy(a, b, mutual=False):
    """-> (index, sq_dist): d^2 summed column by column in float32 (no FMA), the first smallest finite d^2"""
    A, B = np.asarray(a, _f).reshape(-1, 33), np.asarray(b, _f).reshape(-1, 33)
    s = np.zeros((len(A), len(B)), _f)
    for c in range(33):
        d = A[:, c, None] - B[None, :, c]
        s = s + d * d
    fin = np.where(np.isfinite(s), s, np.inf)

    def nearest(M):
        if M.shape[1] == 0:
            return np.full(M.shape[0], -1, np.int32), np.full(M.shape[0], np.inf, _f)
        j = np.argmin(M, 1)
        d = M[np.arange(len(M)), j]
        return np.where(np.isinf(d), -1, j).astype(np.int32), d.astype(_f)

    idx, d = nearest(fin)
    if mutual and len(B):
        back, _ = nearest(fin.T)
        ok = idx >= 0
        ok[ok] = back[idx[ok]] == np.nonzero(ok)[0]
        idx = np.where(ok, idx, -1).astype(np.int32)
    return idx, d


# ---- the pair feature of the contract, vectorised in its operation order, and pairs built on its decision faces

def _vdot(a, b, right=False):
    """(a0 b0 + a1 b1) + a2 b2 in float64, one rounding per operation; right: a0 b0 + (a1 b1 + a2 b2)"""
    p0, p1, p2 = a[..., 0] * b[..., 0], a[..., 1] * b[..., 1], a[..., 2] * b[..., 2]
    return p0 + (p1 + p2) if right else (p0 + p1) + p2


def _vcross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _h(f):
    return 11 * (f + 1.0) * 0.5


def contract_pairs_np(p1, n1, p2, n2, f1_atan2=False, dot_right=False, swap_le=False):
    """-> (bins [m, 3], margin dict): the contract's pair feature of m pairs of float32 points and normals (every normal
    a normal), evaluated in float64 in the contract's operation order, numpy applying one rounding per operation.  The
    margins are the decision quantities themselves: 'swap' = | |a1| - |a2| |, 'f1' = min over the faces of
    |c_i y - s_i x| / |(x, y)| (radians), 'f2' and 'f3' = the distance of 11 (f + 1) 0.5 from the nearest integer, in f.
    The flags evaluate a wrong form instead: f1 by atan2, every dot product reassociated, or a swap on |a1| <= |a2|."""
    dot = lambda a, b: _vdot(a, b, dot_right)  # noqa: E731
    p1, p2 = np.asarray(p1, _f).astype(np.float64), np.asarray(p2, _f).astype(np.float64)

    def unit(n):
        n = np.asarray(n, _f).astype(np.float64)
        return n / np.sqrt(dot(n, n))[:, None]

    n1, n2 = unit(n1), unit(n2)
    dp = p2 - p1
    d = np.sqrt(dot(dp, dp))
    with np.errstate(all="ignore"):
        a1, a2 = dot(n1, dp) / d, dot(n2, dp) / d
        swap = (np.abs(a1) <= np.abs(a2)) if swap_le else (np.abs(a1) < np.abs(a2))
        u = np.where(swap[:, None], n2, n1)
        m = np.where(swap[:, None], n1, n2)
        dp = np.where(swap[:, None], -dp, dp)
        f3 = np.where(swap, -a2, a1)
        v = _vcross(dp, u)
        vn = np.sqrt(dot(v, v))
        v = v / vn[:, None]
        w = _vcross(u, v)
        x, y, f2 = dot(u, m), dot(w, m), dot(v, m)
        C = np.array([face(i)[0] for i in range(1, 11)])
        S = np.array([face(i)[1] for i in range(1, 11)])
        side = C[None, :] * y[:, None] - S[None, :] * x[:, None]
        if f1_atan2:
            b1 = np.clip(np.floor(11 * (np.arctan2(y, x) + np.pi) / (2 * np.pi)), 0, 10)
        else:
            b1 = np.where(y > 0, 5 + (side[:, 5:] >= 0).sum(1), (side[:, :5] >= 0).sum(1))
            b1 = np.where(y == 0, np.where(x < 0, 10, 5), b1)
        near = C[None, :] * x[:, None] + S[None, :] * y[:, None] > 0        # the face's own half, not its opposite ray
        f1m = np.where(near, np.abs(side), np.inf).min(1) / np.hypot(x, y)
        bins = np.stack([b1, 11 + np.clip(np.floor(_h(f2)), 0, 10), 22 + np.clip(np.floor(_h(f3)), 0, 10)], 1)
        degenerate = (d == 0) | (vn == 0)
    bins = np.where(degenerate[:, None], [5, 16, 27], bins).astype(np.int64)
    dist = lambda f: np.abs(_h(f) - np.round(_h(f))) / 5.5  # noqa: E731
    inf = np.where(degenerate, np.inf, 0.0)
    return bins, dict(swap=np.abs(np.abs(a1) - np.abs(a2)) + inf, f1=f1m + inf, f2=dist(f2) + inf, f3=dist(f3) + inf)


def _convergents(r, limit=1 << 24):
    """the continued-fraction convergents (p, q) of the non-negative Fraction r with p, q < limit, last = best"""
    from fractions import Fraction
    out, h0, h1, k0, k1, x = [], 0, 1, 1, 0, Fraction(r)
    while True:
        a = x.numerator // x.denominator
        h0, h1, k0, k1 = h1, a * h1 + h0, k1, a * k1 + k0
        if h1 >= limit or k1 >= limit:
            return out
        out.append((h1, k1))
        if x == a:
            return out
        x = 1 / (x - a)


def _sqrt_ratio(o):
    """sqrt(121 - o^2) / |o| as a Fraction good to about 1e-45"""
    from decimal import Decimal, getcontext
    from fractions import Fraction
    getcontext().prec = 60
    return Fraction((Decimal(121 - o * o).sqrt() / Decimal(abs(o))))


def _int_vectors(L):
    """every integer vector of length exactly L"""
    r = np.arange(-L, L + 1)
    g = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 3)
    return g[(g * g).sum(1) == L * L]


def exact_face_pairs(cap=20, seed=0):
    """integer offsets dp (p2 = p1 + dp, lengths 3 to 15) and integer normals of length 11 whose exact feature lies ON
    a face, so that only the rounding of the contract's double arithmetic decides the bin -> (n1 [m, 3], dp [m, 3],
    n2 [m, 3], kind [m]): 2: f2 = o / 11, 3: f3 = a1 = o / 11 (o odd, |o| <= 9), 4: |a1| = |a2| exactly (the swap's
    tie), each without a swap unless it is a tie.  At most `cap` per (kind, o)."""
    rng = np.random.RandomState(seed)
    V = _int_vectors(11)
    out = []
    for D in (3, 5, 7, 9, 13, 15):
        for dp in _int_vectors(D):
            t1 = V @ dp                                              # 11 D a1
            c = np.cross(dp, V)                                      # |c| |v| direction of each n1
            cc = (c * c).sum(1)
            Q = np.rint(np.sqrt(cc)).astype(np.int64)
            for j in range(len(V)):
                n1 = V[j]
                if t1[j] % D == 0 and (t1[j] // D) % 2 == 1 and abs(t1[j] // D) <= 9:
                    out.append((3, int(t1[j] // D), n1, dp, np.cross(dp, n1)))   # n2 . dp = 0: no swap
                t2 = V @ dp
                ok = np.abs(t2) <= abs(t1[j])
                if Q[j] > 0 and Q[j] * Q[j] == cc[j]:
                    f = V @ c[j]                                     # 11 |c| f2 = 11 (c . n2)
                    hit = ok & (f % Q[j] == 0) & ((f // Q[j]) % 2 == 1) & (np.abs(f // Q[j]) <= 9)
                    for n2 in V[hit]:
                        out.append((2, int((c[j] @ n2) // Q[j]), n1, dp, n2))
                if t1[j] != 0:
                    for n2 in V[(t2 == t1[j]) & ~(V == n1).all(1)]:
                        out.append((4, 0, n1, dp, n2))
    picked = []
    keys = sorted({(k, o) for k, o, *_ in out})
    for key in keys:
        group = [r for r in out if (r[0], r[1]) == key]
        for i in rng.permutation(len(group))[:cap if key[0] != 4 else 4 * cap]:
            picked.append(group[i])
    kind = np.array([r[0] for r in picked])
    n1, dp, n2 = (np.array([r[i] for r in picked], np.float64) for i in (2, 3, 4))
    return n1, dp, n2, kind


def face_pairs(seed=0, per_face=3):
    """isolated pairs (p1, p2) of float32 points and normals whose row p1 -> p2 lands, in the contract's double
    arithmetic, within rounding of a decision face -> (P [2m, 3], N [2m, 3], kind [m]: 1, 2, 3 for the f1, f2 and f3
    faces, 4 for the swap's tie |a1| = |a2|).  p1 lies on a lattice of spacing 32, so each point's nearest other point is
    its partner.
      f1: dp = (1, 0, 0) and n1 = (alpha, 0, gamma), so that u = n1 / |n1|, v = (0, -1, 0) and w = (gamma, 0, -alpha) / |n1|
          up to rounding; n2 = (X, Y, Z) with X (c_i w_x - s_i u_x) + Z (c_i w_z - s_i u_z) = 0 up to the approximation of
          Z / X by a continued-fraction convergent (integers below 2^24, floats exactly) of that exact rational ratio of
          doubles: the face test c_i y - s_i x is zero up to the rounding of x and y.  Y is large, so |a2| < |a1|.
      f2, f3 and the tie: exact_face_pairs, integer inputs whose exact feature lies on the face."""
    from fractions import Fraction
    rng = np.random.RandomState(seed)
    n1s, dps, n2s, kinds = [], [], [], []
    C = [face(i)[0] for i in range(1, 11)]
    S = [face(i)[1] for i in range(1, 11)]
    for alpha, gamma in zip(np.ones(24, _f), rng.uniform(0.05, 0.85, 24).astype(_f)):   # u_x >= 0.76: no swap below
        a, g = float(alpha), float(gamma)
        ln = math.sqrt(a * a + g * g)
        ux, uz = a / ln, g / ln
        vy = -uz / math.sqrt(uz * uz)
        wx, wz = -(uz * vy), ux * vy
        for i in range(10):
            A = C[i] * Fraction(wx) - S[i] * Fraction(ux)
            B = C[i] * Fraction(wz) - S[i] * Fraction(uz)
            r = -A / B if abs(B) >= abs(A) else -B / A                      # Z / X, or X / Z
            for p, q in _convergents(abs(r))[-per_face:]:
                num = -p if r < 0 else p
                X, Z = (q, num) if abs(B) >= abs(A) else (num, q)
                if C[i] * (ux * X + uz * Z) + S[i] * (wx * X + wz * Z) < 0:  # the face's ray, not its opposite
                    X, Z = -X, -Z
                Y = float(2 ** (math.ceil(math.log2(max(abs(X), abs(Z), 1))) + 2))
                n1s.append((a, 0.0, g))
                dps.append((1.0, 0.0, 0.0))
                n2s.append((X, Y, Z))
                kinds.append(1)
    e1, edp, e2, ek = exact_face_pairs(seed=seed)
    n1 = np.concatenate([np.array(n1s), e1])
    dp = np.concatenate([np.array(dps), edp])
    n2 = np.concatenate([np.array(n2s), e2])
    kind = np.concatenate([np.array(kinds), ek])
    m = len(kind)
    side = int(math.ceil(m ** (1 / 3)))
    p1 = 32.0 * np.stack(np.unravel_index(np.arange(m), (side, side, side)), 1)
    P = np.concatenate([p1, p1 + dp]).astype(_f)
    N = np.concatenate([n1, n2]).astype(_f)
    assert np.array_equal(P.astype(np.float64), np.concatenate([p1, p1 + dp])), "points are floats exactly"
    assert np.array_equal(N.astype(np.float64), np.concatenate([n1, n2])), "normals are floats exactly"
    return P, N, kind
