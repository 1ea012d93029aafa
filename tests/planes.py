"""Helpers of the plane segmentation tests (tests/test_planes_cpu.py, tests/test_planes_gpu.py):

* scenes whose planes are known: a room (a floor and two walls) and a table scene (a table top and separated objects made
  of synth's bumpy-sphere surface, standing on it), with noise along the normals and uniform outliers;
* a numpy restatement of the draws, the hypothesis planes and every hypothesis count of one round (float32 operations in
  numpy are IEEE, one rounding each, no contraction), independent of the C++ port;
* the build and run of tests/cpp/planes_main.cc, the test program of Utils::SegmentPlanes."""
import numpy as np

from super4pcs_b200 import synth
from tests import cpp_main

_f = np.float32
M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


# ---- scenes ---------------------------------------------------------------------------------------------------------

def _rotation(seed):
    a = np.random.RandomState(seed).standard_normal(3)
    a /= np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    ang = 0.4
    return np.eye(3) + np.sin(ang) * K + (1 - np.cos(ang)) * (K @ K)


def room(n, noise=0.002, outliers=0.0, seed=0, offset=(0.0, 0.0, 0.0)):
    """-> (P [n, 3] float32, label [n] int (0 floor, 1 and 2 the walls, -1 outliers), planes [3, 4] float64 (unit
    normal, d)).  Floor z = 0 over [-1, 1]^2 (area 4), wall x = -1 (y in [-1, 1], z in [0, 1.5]: area 3), wall y = 1 (x in
    [-0.9, 1], z in [0, 1.2]: area 2.28), points in proportion to area, noise along the normal, then a fixed rotation,
    the offset, and `outliers` of the points uniform in the bounding box; shuffled."""
    rng = np.random.RandomState(seed)
    n_out = int(round(outliers * n))
    n_in = n - n_out
    areas = np.array([4.0, 3.0, 2.28])
    k = np.floor(n_in * areas / areas.sum()).astype(int)
    k[0] += n_in - k.sum()
    u = lambda lo, hi, m: rng.uniform(lo, hi, m)  # noqa: E731
    floor = np.stack([u(-1, 1, k[0]), u(-1, 1, k[0]), rng.normal(0, noise, k[0])], 1)
    wall1 = np.stack([-1 + rng.normal(0, noise, k[1]), u(-1, 1, k[1]), u(0, 1.5, k[1])], 1)
    wall2 = np.stack([u(-0.9, 1, k[2]), 1 + rng.normal(0, noise, k[2]), u(0, 1.2, k[2])], 1)
    X = np.concatenate([floor, wall1, wall2])
    lab = np.repeat([0, 1, 2], k)
    normals = np.array([[0, 0, 1.0], [1.0, 0, 0], [0, 1.0, 0]])
    points = np.array([[0, 0, 0], [-1.0, 0, 0], [0, 1.0, 0]])
    R = _rotation(seed + 11)
    X = X @ R.T + np.asarray(offset)
    N = normals @ R.T
    Pt = points @ R.T + np.asarray(offset)
    planes = np.concatenate([N, -(N * Pt).sum(1, keepdims=True)], 1)
    if n_out:
        lo, hi = X.min(0), X.max(0)
        X = np.concatenate([X, lo + rng.random_sample((n_out, 3)) * (hi - lo)])
        lab = np.concatenate([lab, -np.ones(n_out, int)])
    perm = rng.permutation(len(X))
    return X[perm].astype(_f), lab[perm], planes


def table(n_plane=40000, n_object=5000, centres=((-0.5, -0.5), (0.5, -0.4), (-0.4, 0.5), (0.45, 0.5)), scale=0.12,
          noise=0.001, seed=0):
    """-> (P float32, label int: 0 the table top, k >= 1 object k).  The top z = 0 over [-1, 1]^2 as a 200 x 200 grid of
    spacing 0.01 jittered by at most 0.002 (neighbours closer than 0.015, so the top alone is one radius-0.02
    component), noise along z; each object synth's bumpy-sphere surface scaled by `scale`, lifted so that its lowest point
    is at z = 0.004: it touches the top in the radius graph, and the objects are far apart."""
    rng = np.random.RandomState(seed)
    g = (np.arange(200) + 0.5) / 100.0 - 1.0
    X, Y = np.meshgrid(g, g, indexing="ij")
    top = np.stack([X.ravel() + rng.uniform(-0.002, 0.002, X.size), Y.ravel() + rng.uniform(-0.002, 0.002, X.size),
                    rng.normal(0, noise, X.size)], 1)[:n_plane]
    parts, labs = [top], [np.zeros(len(top), int)]
    for i, (cx, cy) in enumerate(centres):
        _, S = synth._surface(rng, n_object, lambda z: z > -2)
        S = S * scale
        S = S + np.array([cx, cy, 0.004 - S[:, 2].min()])
        parts.append(S)
        labs.append(np.full(n_object, i + 1))
    P, lab = np.concatenate(parts), np.concatenate(labs)
    perm = rng.permutation(len(P))
    return P[perm].astype(_f), lab[perm]


# ---- the numpy restatement ------------------------------------------------------------------------------------------

def splitmix64(seed, k):
    """the SplitMix64 outputs of indices k (uint64 array) of the stream seeded with seed (mod 2^64)"""
    with np.errstate(over="ignore"):
        z = np.uint64(int(seed) % 2 ** 64) + np.asarray(k, np.uint64) * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def draws(m, H, seed_r):
    """-> [H, 3] positions into the active list of length m"""
    k = (3 * np.arange(H, dtype=np.uint64)[:, None] + np.arange(3, dtype=np.uint64)[None, :] + np.uint64(1))
    z = splitmix64(seed_r, k)
    with np.errstate(over="ignore"):
        return (((z >> np.uint64(32)) * np.uint64(m)) >> np.uint64(32)).astype(np.int64)


def hypotheses(P, active, H, seed_r):
    """-> (sample [H, 3] int32 positions j, plane [H, 4] float32 (NaN: invalid), valid [H] bool)"""
    active = np.asarray(active, np.int64)
    sample = active[draws(len(active), H, seed_r)]
    p = P[sample].astype(np.float64)                                 # [H, 3 draws, 3]
    u, v = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    n = np.stack([u[:, 1] * v[:, 2] - u[:, 2] * v[:, 1], u[:, 2] * v[:, 0] - u[:, 0] * v[:, 2],
                  u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]], 1)
    length = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    valid = length != 0
    plane = np.full((H, 4), np.nan, _f)
    nv = n[valid] / length[valid, None]
    big = nv[np.arange(len(nv)), np.argmax(np.abs(nv), 1)]          # argmax: the lowest axis on a tie
    nv[big < 0] *= -1
    p0 = p[valid, 0]
    d = -((nv[:, 0] * p0[:, 0] + nv[:, 1] * p0[:, 1]) + nv[:, 2] * p0[:, 2])
    plane[valid] = np.concatenate([nv, d[:, None]], 1).astype(_f)
    return sample.astype(np.int32), plane, valid


def counts(P, active, plane, threshold, block=64):
    """-> [H] uint32: per plane (a, b, c, d) the points of P[active] with |((a x + b y) + c z) + d| < threshold, fp32"""
    X = P[np.asarray(active, np.int64)].astype(_f)
    x, y, z = X[:, 0][None], X[:, 1][None], X[:, 2][None]
    thr = _f(threshold)
    out = np.empty(len(plane), np.uint32)
    for b in range(0, len(plane), block):
        pl = plane[b:b + block].astype(_f)
        a, bb, c, d = (pl[:, i:i + 1] for i in range(4))
        with np.errstate(invalid="ignore", over="ignore"):
            r = ((a * x + bb * y) + c * z) + d
            out[b:b + block] = (np.abs(r) < thr).sum(1)
    return out


def angle_deg(n1, n2):
    """the angle between two plane normals, sign-free"""
    n1, n2 = np.asarray(n1, np.float64)[:3], np.asarray(n2, np.float64)[:3]
    c = abs(np.dot(n1, n2)) / (np.linalg.norm(n1) * np.linalg.norm(n2))
    return float(np.degrees(np.arccos(min(1.0, c))))


# ---- the C++ test program -------------------------------------------------------------------------------------------

def build(outdir):
    return cpp_main.build("planes_main", outdir)


def run(exe, workdir, xyz, threshold, max_planes=1, min_inliers=1, iterations=1000, seed=0, refine=True, preload=None):
    """-> None when the call threw, else the planes: a list of (coefficients [4] float32, inliers int32 array)"""
    xyz = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    args = [repr(float(threshold)), str(int(max_planes)), str(int(min_inliers)), str(int(iterations)), str(int(seed)),
            "1" if refine else "0"]
    b = cpp_main.run(exe, workdir, np.int32(len(xyz)).tobytes() + xyz.tobytes(), args, preload)
    buf = np.frombuffer(b, np.int32)
    if buf[0]:
        return None
    out, at = [], 2
    for _ in range(int(buf[1])):
        coef = buf[at:at + 4].view(_f).copy()
        s = int(buf[at + 4])
        out.append((coef, buf[at + 5:at + 5 + s].copy()))
        at += 5 + s
    return out
