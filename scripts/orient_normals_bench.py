"""Timing of s4g_orient_normals on the cfg2 P (1M points, delta = 0.003), unbounded, k in {8, 16, 32}, on the unoriented
s4g_normals (k = 16) of the same cloud; one JSON line per k, with the card's name and power limit.

GPU, CUDA events around `reps` calls of s4g_orient_normals_dev (every output requested) after one warm-up call:
  dev_ms       the whole call
  knn_ms       s4g_knn_dev of the P points with self-exclusion: the rows alone, for comparison
and, from one torch.profiler pass over `reps` further calls (CUPTI kernel durations, mean per call):
  stage_ms     rows = k_normals_queries + k_knn + k_on_init; rounds = k_on_find + k_on_best + k_on_hook over every round
               enqueued (later rounds return at once); finish = k_on_roots + k_on_anchor + k_on_output + the radix sort of
               the forest + k_on_edges
  rounds_with_work  the Borůvka rounds that hooked something, from a numpy replay of the rounds on the same rows (each
               component's smallest edge in the contract's order, then the components they join)
CPU, wall clock: the port (oracle/orient_normals_port.cc, one thread, on the GPU's rows) and whether every output equals
the GPU's bit for bit; scipy (cKDTree.query with k + 1 in float64 and the point itself dropped, csgraph's
minimum_spanning_tree on 1 + max|dot| - |dot| and breadth_first_order), and the share of the points whose sign it gives as
ours (its rows and tie order differ where fp32 distances or |dot| tie).

usage: python scripts/orient_normals_bench.py [reps]
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from oracle import orient_normals as oon  # noqa: E402
from super4pcs_b200 import Context, synth  # noqa: E402

KS = [8, 16, 32]
STAGES = {"rows": ("k_normals_queries", "k_knn", "k_on_init"), "rounds": ("k_on_find", "k_on_best", "k_on_hook"),
          "finish": ("k_on_roots", "k_on_anchor", "k_on_output", "DeviceRadixSort", "k_on_edges")}


def stage_ms(prof, reps):
    out = {s: 0.0 for s in STAGES}
    for e in prof.key_averages():
        for s, names in STAGES.items():
            if any(nm in e.key for nm in names):
                out[s] += e.device_time_total / 1e3 / reps
                break
    return out


def edges(N, rows):
    n, k = rows.shape
    u = np.repeat(np.arange(n, dtype=np.int64), k)
    v = rows.reshape(-1).astype(np.int64)
    vert = (N != 0).any(1)
    ok = v >= 0
    u, v = u[ok], v[ok]
    ok = vert[u] & vert[v]
    lo, hi = np.minimum(u[ok], v[ok]), np.maximum(u[ok], v[ok])
    key = np.unique(lo * n + hi)
    lo, hi = key // n, key % n
    a, b = N[lo], N[hi]
    dot = (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]
    return lo, hi, dot


def boruvka_rounds(n, lo, hi, dot):
    """rounds of Borůvka that hook something, on the contract's total order"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    rank = np.empty(len(lo), np.int64)
    rank[np.lexsort((hi, lo, -np.abs(dot.astype(np.float64))))] = np.arange(len(lo))
    comp = np.arange(n)
    rounds = 0
    while True:
        cu, cv = comp[lo], comp[hi]
        x = cu != cv
        if not x.any():
            return rounds
        rounds += 1
        best = np.full(n, len(lo), np.int64)
        np.minimum.at(best, cu[x], rank[x])
        np.minimum.at(best, cv[x], rank[x])
        c = np.nonzero(best < len(lo))[0]
        order = np.argsort(rank)
        e = order[best[c]]
        g = coo_matrix((np.ones(len(c)), (comp[lo[e]], comp[hi[e]])), shape=(n, n))
        _, lab = connected_components(g, directed=False)
        comp = lab[comp]


def scipy_orient(P, N, k):
    """cKDTree rows + minimum_spanning_tree + breadth_first_order, anchors at each component's smallest index"""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import breadth_first_order, connected_components, minimum_spanning_tree
    from scipy.spatial import cKDTree
    n = len(P)
    _, idx = cKDTree(P.astype(np.float64)).query(P.astype(np.float64), k + 1, workers=-1)
    rows = np.where(idx[:, 1:] < n, idx[:, 1:], -1)
    lo, hi, dot = edges(N, rows)
    a = np.abs(dot.astype(np.float64))
    T = minimum_spanning_tree(coo_matrix((1.0 + a.max() - a, (lo, hi)), shape=(n, n)).tocsr()).tocoo()
    f = (((N[T.row] * N[T.col]).sum(1)) < 0).astype(np.int8)
    G = coo_matrix((np.ones(2 * len(f)), (np.concatenate([T.row, T.col]), np.concatenate([T.col, T.row]))),
                   shape=(n, n)).tocsr()
    _, lab = connected_components(G, directed=False)
    first = np.full(lab.max() + 1, n)
    np.minimum.at(first, lab, np.arange(n))
    # one walk from a virtual node n joined to every component's smallest index
    H = coo_matrix((np.ones(2 * len(f) + 2 * len(first)),
                    (np.concatenate([T.row, T.col, first, np.full(len(first), n)]),
                     np.concatenate([T.col, T.row, np.full(len(first), n), first]))), shape=(n + 1, n + 1)).tocsr()
    order, pred = breadth_first_order(H, n, directed=False, return_predecessors=True)
    fp = np.zeros(n + 1, np.int8)
    m = pred[T.col] == T.row
    fp[T.col[m]] = f[m]
    m = pred[T.row] == T.col
    fp[T.row[m]] = f[m]
    par, pl, fl = [0] * (n + 1), pred.tolist(), fp.tolist()
    for x in order[1:].tolist():
        par[x] = par[pl[x]] ^ fl[x]
    par = np.asarray(par[:n], np.int8)
    return np.where(par[:, None] == 1, -N, N)


def main(reps=5):
    import torch
    n, delta = 1_000_000, 0.003
    P, _ = synth.center(synth.make_pair(n, 0.3, seed=42)["P"])
    P = np.ascontiguousarray(P, np.float32)
    dev = bench.device_info(0, 0)
    stream = torch.cuda.Stream()
    dX = torch.from_numpy(P).cuda()
    excl = torch.arange(n, dtype=torch.int32, device="cuda")
    idx = torch.empty(n * max(KS), dtype=torch.int32, device="cuda")
    dN = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    dO = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    root = torch.empty(n, dtype=torch.int32, device="cuda")
    tree = torch.empty((n - 1, 2), dtype=torch.int32, device="cuda")
    out2 = torch.empty(2, dtype=torch.int64, device="cuda")

    def timed(call):
        call()
        stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            call()
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    with Context(0) as ctx, torch.cuda.stream(stream):
        ctx.set_stream(stream.cuda_stream)
        ctx.set_cloud_p(P, delta)
        ctx.normals_dev(16, dN.data_ptr())
        stream.synchronize()
        N = dN.cpu().numpy()
        for k in KS:
            call = lambda: ctx.orient_normals_dev(dN.data_ptr(), k, dO.data_ptr(), out2.data_ptr(),  # noqa: E731
                                                  root.data_ptr(), tree.data_ptr())
            dev_ms = timed(call)
            knn_ms = timed(lambda: ctx.knn_dev(dX.data_ptr(), n, k, idx.data_ptr(), None, d_exclude_ptr=excl.data_ptr()))
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    call()
                stream.synchronize()
            stages = stage_ms(prof, reps)
            nc, nt = [int(x) for x in out2.cpu()]
            got = (dO.cpu().numpy(), root.cpu().numpy(), nc, tree.cpu().numpy()[:nt])
            rows = idx[:n * k].cpu().numpy().reshape(n, k)
            t0 = time.perf_counter()
            want = oon.port(P, N, k, rows=rows)
            port_ms = (time.perf_counter() - t0) * 1e3
            equal = (got[2] == want[2] and np.array_equal(got[0].view(np.uint32), want[0].view(np.uint32)) and
                     np.array_equal(got[1], want[1]) and np.array_equal(got[3], want[3]))
            lo, hi, dot = edges(N, rows)
            row = dict(cfg="cfg2", stage="orient_normals", k=k, n_p=n, delta=delta, sq_radius="inf", reps=reps,
                       dev_ms=dev_ms, knn_ms=knn_ms, stage_ms=stages, n_components=nc, n_tree_edges=nt,
                       n_edges=int(len(lo)), rounds_enqueued=int(np.ceil(np.log2(n))) + 1,
                       rounds_with_work=boruvka_rounds(n, lo, hi, dot), port_ms_1_thread=port_ms,
                       dev_equals_port=bool(equal), device=dev)
            try:
                t0 = time.perf_counter()
                sp = scipy_orient(P, N, k)
                row.update(cpu_threads=os.cpu_count(), scipy_ms=(time.perf_counter() - t0) * 1e3,
                           scipy_same_sign_share=float((sp.view(np.uint32) == got[0].view(np.uint32)).all(1).mean()))
            except ImportError:
                pass
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main(int(sys.argv[1]) if len(sys.argv) > 1 else 5)
