"""Builds and runs tests/cpp/orient_normals_main.cc, the test program of Utils::OrientNormals, for
tests/test_orient_normals_cpu.py (on the oracle stand-in) and tests/test_orient_normals_gpu.py (on the real library).
Also two restatements of the s4g_orient_normals contract that share no code with the port (scipy's minimum spanning tree and a
plain-Python Kruskal), and the shapes with analytic normals the tests share."""
import numpy as np

from tests import cpp_main, normals as tnormals

_f = np.float32


def build(outdir):
    return cpp_main.build("orient_normals_main", outdir)


def run(exe, workdir, xyz, normals, k, max_distance=np.inf, viewpoint=None, preload=None):
    """-> (threw, returned count, normals [n, 3] float32 as the points hold them afterwards)"""
    xyz = np.ascontiguousarray(xyz, _f).reshape(-1, 3)
    args = [str(int(k)), repr(float(max_distance))]
    if viewpoint is not None:
        args += [repr(float(v)) for v in np.asarray(viewpoint, _f)]
    payload = np.int32(len(xyz)).tobytes() + xyz.tobytes() + np.ascontiguousarray(normals, _f).tobytes()
    r = cpp_main.Reader(cpp_main.run(exe, workdir, payload, args, preload))
    threw, count = r.take(np.int32, 2)
    return bool(threw), int(count), r.take(_f, 3 * len(xyz)).reshape(-1, 3)


def expected_held(normals, oriented):
    """what OrientNormals leaves in the points, from the normals they held (set_normal of the input) and the oriented
    normals of the same: a flipped normal goes through set_normal(-normal()) once more, the others stay as they were"""
    held = np.asarray(normals, _f)
    oriented = np.asarray(oriented, _f)
    flipped = (held.view(np.uint32) != oriented.view(np.uint32)).any(1)
    out = held.copy()
    out[flipped] = tnormals.set_normal(-held[flipped])
    return out


# ---- restatements of the contract, sharing no code with oracle/orient_normals_port.cc

def dots(N, lo, hi):
    """fp32 (xi xj + yi yj) + zi zj of the edges (lo, hi)"""
    a, b = np.asarray(N, _f)[lo], np.asarray(N, _f)[hi]
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def edges_from_rows(N, rows):
    """the undirected edges (lo, hi) [m, 2] of the symmetrised rows between vertices, unique, in ascending (lo, hi)"""
    N = np.asarray(N, _f)
    n, k = rows.shape
    u = np.repeat(np.arange(n), k)
    v = rows.reshape(-1).astype(np.int64)
    vert = (N != 0).any(1)
    ok = v >= 0
    u, v = u[ok], v[ok]
    ok = vert[u] & vert[v]
    u, v = u[ok], v[ok]
    E = np.unique(np.stack([np.minimum(u, v), np.maximum(u, v)], 1), axis=0)
    return E.reshape(-1, 2)


def anchor_rule(P, N, members, root, viewpoint):
    """-> (anchor, negated) of a component (members ascending)"""
    if viewpoint is None:
        return root, False
    v = np.asarray(viewpoint, _f)
    d = np.asarray(P, _f)[members] - v
    d2 = d[:, 0] * d[:, 0] + (d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
    a = int(members[np.argmin(d2)])     # argmin: the first of equal values, the smallest j
    pa, na = np.asarray(P, _f)[a].astype(np.float64), np.asarray(N, _f)[a].astype(np.float64)
    s = ((float(v[0]) - pa[0]) * na[0] + (float(v[1]) - pa[1]) * na[1]) + (float(v[2]) - pa[2]) * na[2]
    return a, bool(s < 0.0)


def finish(P, N, n, tree, viewpoint):
    """the outputs of the contract from a forest tree [m, 2] (lo, hi): (oriented, root, n_components, tree sorted)"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import breadth_first_order, connected_components
    N = np.asarray(N, _f)
    vert = (N != 0).any(1)
    tree = np.asarray(tree, np.int64).reshape(-1, 2)
    flip = (dots(N, tree[:, 0], tree[:, 1]) < 0).astype(np.int8)
    # weights flip + 1 so that a no-flip edge is not an absent entry
    G = coo_matrix((np.concatenate([flip, flip]) + 1, (np.concatenate([tree[:, 0], tree[:, 1]]),
                                                       np.concatenate([tree[:, 1], tree[:, 0]]))), shape=(n, n)).tocsr()
    _, lab = connected_components(G, directed=False)
    out, root = np.asarray(N, _f).copy(), np.full(n, -1, np.int32)
    n_comp = 0
    for c in np.unique(lab[vert]):
        members = np.nonzero((lab == c) & vert)[0]
        r = int(members[0])
        root[members] = r
        n_comp += 1
        a, neg = anchor_rule(P, N, members, r, viewpoint)
        order, pred = breadth_first_order(G, a, directed=False, return_predecessors=True)
        par = {a: int(neg)}
        for x in order[1:]:
            par[int(x)] = par[int(pred[x])] ^ (int(G[pred[x], x]) - 1)
        for x in members:
            if par[int(x)]:
                out[x] = -out[x]
    tree = tree[np.lexsort((tree[:, 1], tree[:, 0]))] if len(tree) else tree
    return out, root, n_comp, tree.astype(np.int32)


def scipy_orient(P, N, rows, viewpoint=None):
    """the contract through scipy.sparse.csgraph.minimum_spanning_tree: valid only when every edge weight is distinct
    (the caller asserts it with distinct_weights); rows: the knn rows with self-exclusion"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import minimum_spanning_tree
    N = np.asarray(N, _f)
    n = len(N)
    E = edges_from_rows(N, rows)
    w = weights(N, E)
    M = minimum_spanning_tree(coo_matrix((w, (E[:, 0], E[:, 1])), shape=(n, n)).tocsr()).tocoo()
    tree = np.stack([np.minimum(M.row, M.col), np.maximum(M.row, M.col)], 1)
    return finish(P, N, n, tree, viewpoint)


def weights(N, E):
    """positive float64 weights that order the edges as |dot| descending (1 + max |dot| - |dot|)"""
    a = np.abs(dots(N, E[:, 0], E[:, 1]).astype(np.float64))
    return 1.0 + (a.max() if len(a) else 0.0) - a


def distinct_weights(N, rows):
    E = edges_from_rows(N, rows)
    w = weights(N, E)
    return len(np.unique(w)) == len(w)


def kruskal_orient(P, N, rows, viewpoint=None):
    """the contract with a plain-Python Kruskal keyed on (-|dot|, lo, hi): exact under ties"""
    N = np.asarray(N, _f)
    n = len(N)
    E = edges_from_rows(N, rows)
    a = np.abs(dots(N, E[:, 0], E[:, 1]))
    order = sorted(range(len(E)), key=lambda i: (-float(a[i]), int(E[i, 0]), int(E[i, 1])))
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x

    tree = []
    for i in order:
        x, y = find(int(E[i, 0])), find(int(E[i, 1]))
        if x != y:
            parent[max(x, y)] = min(x, y)
            tree.append(E[i])
    return finish(P, N, n, np.asarray(tree, np.int64).reshape(-1, 2), viewpoint)


# ---- shapes with analytic normals

def sphere(n, seed=0, radius=1.0):
    """n points on a sphere (Fibonacci lattice, jittered) -> (xyz, outward unit normals)"""
    rng = np.random.RandomState(seed)
    i = np.arange(n) + 0.5
    z = 1 - 2 * i / n
    t = np.pi * (1 + 5 ** 0.5) * i + rng.uniform(-0.3, 0.3, n)
    r = np.sqrt(1 - z * z)
    U = np.stack([r * np.cos(t), r * np.sin(t), z], 1)
    U = U[rng.permutation(n)]
    return (U * radius).astype(_f), U.astype(_f)


def torus(n, seed=0, R=1.0, r=0.35):
    """n points on a torus around z, sampled with uniform area density -> (xyz, outward unit normals)"""
    rng = np.random.RandomState(seed)
    u, v = [], []
    while sum(len(x) for x in u) < n:
        uu, vv = rng.uniform(0, 2 * np.pi, 2 * n), rng.uniform(0, 2 * np.pi, 2 * n)
        keep = rng.uniform(0, 1, 2 * n) < (R + r * np.cos(vv)) / (R + r)
        u.append(uu[keep])
        v.append(vv[keep])
    u, v = np.concatenate(u)[:n], np.concatenate(v)[:n]
    Nrm = np.stack([np.cos(v) * np.cos(u), np.cos(v) * np.sin(u), np.sin(v)], 1)
    X = np.stack([(R + r * np.cos(v)) * np.cos(u), (R + r * np.cos(v)) * np.sin(u), r * np.sin(v)], 1)
    return X.astype(_f), Nrm.astype(_f)


def scramble(N, seed=0):
    """the normals with random signs"""
    s = np.where(np.random.RandomState(seed).rand(len(N)) < 0.5, -1, 1).astype(_f)
    return (np.asarray(N, _f) * s[:, None]).astype(_f)
