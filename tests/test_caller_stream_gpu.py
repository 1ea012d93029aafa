"""The device-pointer entry points on a caller's stream (include/s4g.h, s4g_set_stream).

Every _dev entry point enqueues on the context's stream, which s4g_set_stream may point at a stream the caller owns, and
returns without synchronising.  bench.py's timed step relies on both: it binds the context to its own torch stream and
times s4g_verify_best_dev (k_verify, k_argmax, the key) there with no host wait.  The other GPU tests call each _dev
form between torch.cuda.synchronize() and ctx.synchronize(), so they check the arithmetic but not the order.  Here, on a
torch side stream S:

  ordered, input side    the device inputs hold poison (NaN transforms, queries and descriptors, zero normals, all-zero
                         quads); S runs a sleep, the copy of the true inputs from pinned memory, the call, and a copy of
                         the outputs into fresh buffers.  Work that runs anywhere but on S reads the poison.
  ordered, output side   S also fills every output with a sentinel after the sleep: work that runs early is overwritten.
  Both patterns run for every _dev entry point with every optional output given, after one warm-up call, and the copied
  outputs are bit-equal to the host form on a second context that keeps its own stream (the Verify counts: to the port,
  oracle/port.cc).
  no host wait           after a warm-up call with the same shapes (first launches load modules, scratch grows), a long
                         sleep on S, then the call: it returns while S is still busy.
  s4g_try_congruent_set_dev returns a host record, so it waits for S: quads produced on S after a sleep are read in
  order.  Then the chain bench.py times (two s4g_verify_best_dev back to back at three query patches, a permuted index
  array, the maximum tied across three chunks), s4g_set_stream itself (switching waits for the old stream, NULL restores
  the context's own stream, cudaStreamLegacy orders after torch's default stream, whose handle 0 means "own stream"),
  two contexts on one stream and one context moved between two streams.

Every delay is a torch.cuda._sleep spin of a bounded number of clock cycles, calibrated once per module with CUDA events.
No stream waits on a host flag or on an event that may never be recorded: a broken library fails a test, never hangs it.
"""
import collections
import time

import numpy as np
import pytest

from oracle import port as oport
from tests import common

pytestmark = pytest.mark.gpu

DELTA = 0.01
VIEW = np.float32([0.3, -2.0, 1.5])
ORDER_MS = 100                 # the sleep in front of an ordered chain
BUSY_MS = 150                  # the sleep a call that does not synchronise returns within
MAX_MS = 150                   # no sleep is longer
MAX_CYCLES_PER_MS = 1.98e6     # the H100's highest SM clock, 1980 MHz: a larger calibration is a measurement error
CUDA_STREAM_LEGACY = 1         # cudaStreamLegacy's handle

# one entry point (or, for the range query, the count + fill pair) with its device buffers:
#   inputs  [(device tensor, pinned host tensor, poison)]   outputs [(device tensor, sentinel)]
#   call()  enqueues it on the context's stream;  want: host-form arrays;  got(outputs as numpy) -> comparable arrays
Case = collections.namedtuple("Case", "inputs outputs call want got")


@pytest.fixture(scope="module")
def sleep_ms():
    """sleep_ms(ms): a spin of ms milliseconds on the current stream, the cycles per ms measured here with CUDA events"""
    import torch
    n = 20_000_000
    rates = []
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(1000)                                   # loads the spin kernel
        for _ in range(3):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            torch.cuda._sleep(n)
            b.record()
            b.synchronize()
            rates.append(n / a.elapsed_time(b))
    rate = min(float(np.median(rates)), MAX_CYCLES_PER_MS)
    print("\nsleep calibration: %.0f cycles per ms (runs %s)" % (rate, ", ".join("%.0f" % r for r in rates)))

    def sleep(ms):
        assert 0 < ms <= MAX_MS
        torch.cuda._sleep(int(ms * rate))
    return sleep


def pinned(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory()


def empty(shape, dtype):
    import torch
    return torch.empty(shape, dtype=dtype, device="cuda")


def same(got, want, what):
    assert len(got) == len(want), what
    for i, (g, w) in enumerate(zip(got, want)):
        g, w = np.ascontiguousarray(g).reshape(-1), np.ascontiguousarray(w).reshape(-1)
        assert g.nbytes == w.nbytes, (what, i, g.shape, w.shape)
        gb, wb = g.view(np.uint8), w.view(np.uint8)
        assert np.array_equal(gb, wb), (what, i, np.flatnonzero(gb != wb)[:8])


def warm_up(S, case):
    """one call with the true inputs: the first launch of a kernel can wait for the whole device while its module loads,
    which would order a misplaced launch by accident"""
    import torch
    for d, h, _ in case.inputs:
        d.copy_(h)
    torch.cuda.synchronize()
    with torch.cuda.stream(S):
        case.call()
    S.synchronize()


def run_ordered(S, case, sleep_ms):
    """poison the inputs, then on S: sleep, the true inputs, the sentinels, the call, the copies; -> case.got(copies)"""
    import torch
    warm_up(S, case)
    for d, _, poison in case.inputs:
        d.fill_(poison)
    torch.cuda.synchronize()
    with torch.cuda.stream(S):
        sleep_ms(ORDER_MS)
        for d, h, _ in case.inputs:
            d.copy_(h, non_blocking=True)
        for o, sentinel in case.outputs:
            o.fill_(sentinel)
        case.call()
        outs = [o.clone() for o, _ in case.outputs]
    S.synchronize()
    return case.got([o.cpu().numpy() for o in outs])


def with_ties(port, T, spots):
    """T with the best candidate copied to the first two of `spots` outside its chunk of 16 -> (T, the port's counts,
    the tied positions); the maximum then lies in three chunks"""
    good = port.verify_batch(T, 0.0, nthreads=oport.num_threads())[1]
    a = int(np.argmax(good))
    T = T.copy()
    T[[p for p in spots if p // 16 != a // 16][:2]] = T[a]
    good = port.verify_batch(T, 0.0, nthreads=oport.num_threads())[1]
    top = np.flatnonzero(good == good.max())
    assert len(set(top // 16)) >= 3 and good.max() > 0
    return T, good, top


def best_key(counts, index):
    """max_k (counts[k] << 32 | 0xFFFFFFFF - index[k]), the key of s4g_verify_best"""
    c, i = counts.astype(np.uint64), index.astype(np.uint64)
    return np.array([((c << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - i)).max()], np.uint64)


Env = collections.namedtuple("Env", "S ctx ref sc port T counts index X T1 ex N0 N1 cases")


@pytest.fixture(scope="module")
def env(s4g_lib):
    """one context bound to the side stream S and one on its own stream, both holding a 20 000-point P and Q"""
    import torch
    from super4pcs_b200 import Context
    sc = common.scenario(20000, 0.4, DELTA, seed=5)
    P, Q = sc["P"], sc["Q"]
    rng = np.random.RandomState(1)
    X = (Q[rng.randint(0, len(Q), 3000)] + rng.normal(0, 0.5 * DELTA, (3000, 3))).astype(np.float32)   # T1 X lies on P
    ex = rng.randint(-1, len(P), len(X)).astype(np.int32)
    T = common.candidates_colmajor(sc, 40, n_near=12)
    port = oport.Port(P, Q, DELTA)
    counts = port.verify_batch(T, 0.0, nthreads=oport.num_threads())[1]
    assert len(np.unique(counts)) > 8                              # counts differ: a misordered write cannot hide
    index = rng.choice(10 ** 6, len(T), replace=False).astype(np.uint32)
    S = torch.cuda.Stream()
    ctx, ref = Context(0), Context(0)
    for c in (ctx, ref):
        c.set_cloud_p(P, DELTA)
        c.set_cloud_q(Q)
    N0 = ref.normals(16)[0]
    N1 = ref.orient_normals(N0, 16, viewpoint=VIEW)[0]
    ctx.set_stream(S.cuda_stream)
    yield Env(S, ctx, ref, sc, port, T, counts, index, X, common.candidates_colmajor(sc, 1, n_near=1)[0], ex, N0, N1, {})
    ctx.set_stream(None)
    ctx.close()
    ref.close()
    port.close()


def bound(e):
    """e.ctx bound to e.S again (a test may have moved it)"""
    e.ctx.set_stream(e.S.cuda_stream)
    return e.ctx


# ---- the cases: one per entry point, every optional output given ------------------------------------------------------

def case_verify_dev(e):
    import torch
    K = len(e.T)
    dT, dc = empty((K, 16), torch.float32), empty(K, torch.int32)
    return Case([(dT, pinned(e.T), float("nan"))], [(dc, -1)],
                lambda: e.ctx.verify_dev(dT.data_ptr(), K, dc.data_ptr()),
                [e.counts], lambda o: o)


def case_verify_best_dev(e):
    import torch
    K = len(e.T)
    dT, dI = empty((K, 16), torch.float32), empty(K, torch.int32)
    dc, dk = empty(K, torch.int32), empty(1, torch.int64)
    return Case([(dT, pinned(e.T), float("nan")), (dI, pinned(e.index.view(np.int32)), 0)], [(dc, -1), (dk, -1)],
                lambda: e.ctx.verify_best_dev(dT.data_ptr(), K, dI.data_ptr(), dc.data_ptr(), dk.data_ptr()),
                [e.counts, best_key(e.counts, e.index)], lambda o: o)


def case_verify_nearest_dev(e):
    import torch
    T = e.T[:8]
    K, nQ = len(T), e.ctx.nQ
    dT = empty((K, 16), torch.float32)
    di, ds, dc = empty((K, nQ), torch.int32), empty((K, nQ), torch.float32), empty(K, torch.int32)
    want = list(e.ref.verify_nearest(T))
    assert np.array_equal(want[2], e.counts[:8])
    return Case([(dT, pinned(T), float("nan"))], [(di, 7), (ds, 7.0), (dc, -1)],
                lambda: e.ctx.verify_nearest_dev(dT.data_ptr(), K, di.data_ptr(), ds.data_ptr(), dc.data_ptr()),
                want, lambda o: o)


def case_nearest_dev(e):
    import torch
    n, r = len(e.X), 9 * DELTA * DELTA
    dX, dT, dE = empty((n, 3), torch.float32), empty(16, torch.float32), empty(n, torch.int32)
    di, ds = empty(n, torch.int32), empty(n, torch.float32)
    want = list(e.ref.nearest(e.X, r, e.T1, e.ex))
    assert (want[0] >= 0).mean() > 0.2
    return Case([(dX, pinned(e.X), float("nan")), (dT, pinned(e.T1), float("nan")), (dE, pinned(e.ex), 0)],
                [(di, 7), (ds, 7.0)],
                lambda: e.ctx.nearest_dev(dX.data_ptr(), n, di.data_ptr(), ds.data_ptr(), r, dT.data_ptr(), dE.data_ptr()),
                want, lambda o: o)


def case_knn_dev(e):
    import torch
    n, k = len(e.X), 9
    dX, dT, dE = empty((n, 3), torch.float32), empty(16, torch.float32), empty(n, torch.int32)
    di, ds = empty((n, k), torch.int32), empty((n, k), torch.float32)
    return Case([(dX, pinned(e.X), float("nan")), (dT, pinned(e.T1), float("nan")), (dE, pinned(e.ex), 0)],
                [(di, 7), (ds, 7.0)],
                lambda: e.ctx.knn_dev(dX.data_ptr(), n, k, di.data_ptr(), ds.data_ptr(), np.inf, dT.data_ptr(),
                                      dE.data_ptr()),
                list(e.ref.knn(e.X, k, np.inf, e.T1, e.ex)), lambda o: o)


def case_range_dev(e):
    """count and fill chained on the stream, the total known from the host form (the offsets stay valid either way)"""
    import torch
    n, r = len(e.X), (3 * DELTA) ** 2
    want = list(e.ref.range_query(e.X, r, e.T1))
    total = int(want[0][-1])
    assert total > n // 3
    dX, dT = empty((n, 3), torch.float32), empty(16, torch.float32)
    do, di, ds = empty(n + 1, torch.int64), empty(total, torch.int32), empty(total, torch.float32)

    def call():
        e.ctx.range_count_dev(dX.data_ptr(), n, do.data_ptr(), r, dT.data_ptr())
        e.ctx.range_fill_dev(dX.data_ptr(), n, do.data_ptr(), total, di.data_ptr(), ds.data_ptr(), r, dT.data_ptr())
    return Case([(dX, pinned(e.X), float("nan")), (dT, pinned(e.T1), float("nan"))], [(do, 0), (di, -7), (ds, 7.0)],
                call, want, lambda o: o)


def case_normals_dev(e):
    import torch
    n = e.ctx.nP
    dn, dv = empty((n, 3), torch.float32), empty((n, 3), torch.float32)
    return Case([], [(dn, 7.0), (dv, 7.0)],
                lambda: e.ctx.normals_dev(16, dn.data_ptr(), dv.data_ptr(), np.inf, VIEW),
                list(e.ref.normals(16, np.inf, VIEW)), lambda o: o)


def case_orient_normals_dev(e):
    import torch
    n = e.ctx.nP
    dN, do = empty((n, 3), torch.float32), empty((n, 3), torch.float32)
    droot, d2, dtree = empty(n, torch.int32), empty(2, torch.int64), empty(2 * (n - 1), torch.int32)
    out, root, nc, tree = e.ref.orient_normals(e.N0, 16, viewpoint=VIEW)
    assert len(tree) > n // 2
    return Case([(dN, pinned(e.N0), 0.0)], [(do, 7.0), (droot, 7), (d2, 7), (dtree, 7)],
                lambda: e.ctx.orient_normals_dev(dN.data_ptr(), 16, do.data_ptr(), d2.data_ptr(), droot.data_ptr(),
                                                 dtree.data_ptr(), np.inf, VIEW),
                [out, root, np.array([nc, len(tree)], np.int64), tree],
                lambda o: [o[0], o[1], o[2], o[3][:2 * int(o[2][1])]])


def case_fpfh_dev(e):
    import torch
    n = e.ctx.nP
    dN, dF = empty((n, 3), torch.float32), empty((n, 33), torch.float32)
    return Case([(dN, pinned(e.N1), 0.0)], [(dF, 7.0)],
                lambda: e.ctx.fpfh_dev(dN.data_ptr(), 16, dF.data_ptr(), np.inf),
                [e.ref.fpfh(e.N1, 16)], lambda o: o)


def case_fpfh_match_dev(e):
    import torch
    rng = np.random.RandomState(3)
    A, B = rng.uniform(0, 60, (4000, 33)).astype(np.float32), rng.uniform(0, 60, (6000, 33)).astype(np.float32)
    B[:1500] = A[:1500] + 0.01
    dA, dB = empty(A.shape, torch.float32), empty(B.shape, torch.float32)
    di, ds = empty(len(A), torch.int32), empty(len(A), torch.float32)
    want = list(e.ref.fpfh_match(A, B, True))
    assert (want[0] >= 0).sum() >= 1500
    return Case([(dA, pinned(A), float("nan")), (dB, pinned(B), float("nan"))], [(di, 7), (ds, 7.0)],
                lambda: e.ctx.fpfh_match_dev(dA.data_ptr(), len(A), dB.data_ptr(), len(B), di.data_ptr(), ds.data_ptr(),
                                             mutual=True),
                want, lambda o: o)


def case_statistical_outliers_dev(e):
    import torch
    n = e.ctx.nP
    dk, dn, dm, d2 = empty(n, torch.int32), empty(1, torch.int64), empty(n, torch.float64), empty(2, torch.float64)
    keep, mean, mu, sigma = e.ref.statistical_outliers(8, 1.0)
    assert 0 < len(keep) < n
    return Case([], [(dk, 7), (dn, -7), (dm, 7.0), (d2, 7.0)],
                lambda: e.ctx.statistical_outliers_dev(8, 1.0, dk.data_ptr(), dn.data_ptr(), dm.data_ptr(), d2.data_ptr()),
                [keep, np.array([len(keep)], np.int64), mean, np.array([mu, sigma])],
                lambda o: [o[0][:int(o[1][0])], o[1], o[2], o[3]])


def case_radius_outliers_dev(e):
    import torch
    n, r = e.ctx.nP, (2 * DELTA) ** 2
    dk, dn, dc = empty(n, torch.int32), empty(1, torch.int64), empty(n, torch.int32)
    keep, counts = e.ref.radius_outliers(r, 4)
    assert 0 < len(keep) < n
    return Case([], [(dk, 7), (dn, -7), (dc, 7)],
                lambda: e.ctx.radius_outliers_dev(r, 4, dk.data_ptr(), dn.data_ptr(), dc.data_ptr()),
                [keep, np.array([len(keep)], np.int64), counts],
                lambda o: [o[0][:int(o[1][0])], o[1], o[2]])


def case_euclidean_clusters_dev(e):
    import torch
    n, r = e.ctx.nP, (2 * DELTA) ** 2
    dl, dn, dr = empty(n, torch.int32), empty(1, torch.int64), empty(n, torch.int32)
    do, dm = empty(n + 1, torch.int64), empty(n, torch.int32)
    labels, root, offsets, members = e.ref.euclidean_clusters(r, 2)
    assert len(offsets) > 100
    return Case([], [(dl, 7), (dn, -7), (dr, 7), (do, 7), (dm, 7)],
                lambda: e.ctx.euclidean_clusters_dev(r, dl.data_ptr(), dn.data_ptr(), dr.data_ptr(), do.data_ptr(),
                                                     dm.data_ptr(), min_size=2),
                [labels, np.array([len(offsets) - 1], np.int64), root, offsets, members],
                lambda o: [o[0], o[1], o[2], o[3][:int(o[1][0]) + 1], o[4][:int(o[3][int(o[1][0])])]])


def case_segment_planes_dev(e):
    import torch
    n, H, R = e.ctx.nP, 256, 3
    dl, dp, dn = empty(n, torch.int32), empty(R * 64, torch.uint8), empty(1, torch.int32)
    do, dm, dh = empty(R + 1, torch.int64), empty(n, torch.int32), empty((R, H), torch.int32)
    labels, planes, offsets, members, hyp = e.ref.segment_planes(DELTA, H, R, 1, 11, True, hyp_counts=True)
    k = len(planes)
    assert k == R
    return Case([], [(dl, 7), (dp, 7), (dn, 7), (do, 7), (dm, 7), (dh, 7)],
                lambda: e.ctx.segment_planes_dev(DELTA, dl.data_ptr(), dp.data_ptr(), dn.data_ptr(), do.data_ptr(),
                                                 dm.data_ptr(), dh.data_ptr(), H, R, 1, 11, True),
                [labels, planes, np.array([k], np.int32), offsets, members, hyp],
                lambda o: [o[0], o[1][:64 * int(o[2][0])], o[2], o[3][:int(o[2][0]) + 1],
                           o[4][:int(o[3][int(o[2][0])])], o[5]])


def case_voxel_grid_dev(e):
    import torch
    X = e.sc["P"]
    n, leaf = len(X), 4 * DELTA
    rng = np.random.RandomState(4)
    N, C = e.N1, rng.uniform(0, 1, (n, 3)).astype(np.float32)
    dx, dN, dC = (empty((n, 3), torch.float32) for _ in range(3))
    ox, oN, oC = (empty((n, 3), torch.float32) for _ in range(3))
    om, ocnt, ofst, ovof = empty(1, torch.int64), empty(n, torch.int32), empty(n, torch.int32), empty(n, torch.int32)
    xyz, nrm, rgb, counts, first, voxel_of = e.ref.voxel_grid(X, leaf, N, C, 2)
    assert 100 < len(xyz) < n // 2

    def got(o):
        m = int(o[1][0])
        return [o[0][:m], o[1], o[2][:m], o[3][:m], o[4][:m], o[5][:m], o[6]]
    return Case([(dx, pinned(X), float("nan")), (dN, pinned(N), 0.0), (dC, pinned(C), 0.0)],
                [(ox, 7.0), (om, 7), (oN, 7.0), (oC, 7.0), (ocnt, 7), (ofst, 7), (ovof, 7)],
                lambda: e.ctx.voxel_grid_dev(dx.data_ptr(), n, leaf, ox.data_ptr(), om.data_ptr(), dN.data_ptr(),
                                             dC.data_ptr(), oN.data_ptr(), oC.data_ptr(), ocnt.data_ptr(),
                                             ofst.data_ptr(), ovof.data_ptr(), min_points=2),
                [xyz, np.array([len(xyz)], np.int64), nrm, rgb, counts, first, voxel_of], got)


CASES = {name[len("case_"):]: f for name, f in sorted(globals().items()) if name.startswith("case_")}


def get_case(e, name):
    if name not in e.cases:
        e.cases[name] = CASES[name](e)
    return e.cases[name]


# ---- 1. every entry point ordered on the caller's stream --------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(CASES))
def test_ordered_on_the_callers_stream(env, sleep_ms, name):
    case = get_case(env, name)
    bound(env)
    same(run_ordered(env.S, case, sleep_ms), case.want, name)


# ---- 2. no host synchronisation --------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(CASES))
def test_returns_while_the_stream_is_busy(env, sleep_ms, name):
    """a warm-up call with the same shapes, then a long sleep on S and the call: S is still busy when it returns"""
    import torch
    case = get_case(env, name)
    bound(env)
    warm_up(env.S, case)
    with torch.cuda.stream(env.S):
        sleep_ms(BUSY_MS)
        t0 = time.perf_counter()
        case.call()
        host_ms = 1e3 * (time.perf_counter() - t0)
        busy = not env.S.query()
    env.S.synchronize()
    print("%s: %.2f ms on the host" % (name, host_ms))
    assert busy, "%s waited for the stream: the call took %.1f ms on the host behind a %d ms sleep" % (name, host_ms,
                                                                                                       BUSY_MS)


# ---- 3. s4g_try_congruent_set_dev: returns a host record, so it waits ----------------------------------------------

def test_try_congruent_set_dev_reads_its_quads_in_stream_order(s4g_lib, sleep_ms):
    """the quads reach the device on S after a sleep; the record the call returns (after waiting for S, which is then
    idle) equals the host form's field for field and the port's winner, gate count, LCP and transform bits"""
    import torch
    from super4pcs_b200 import Context
    delta = 0.05
    sc = common.scenario(3000, 0.4, delta)
    P, Q = sc["P"], sc["Q"]
    rng = np.random.RandomState(11)
    base = rng.choice(np.flatnonzero(np.abs((P + sc["cp"])[:, 2]) < 0.15), 4, replace=False).astype(np.int32)
    quads = common.congruent_like_quads(sc, base, 3000, 5)
    pt = oport.Port(P, Q, delta)
    want = pt.try_congruent_set(base, quads, best_lcp_in=0.0)
    pt.close()
    assert want["best_index"] >= 0 and want["n_gate"] > 16
    S = torch.cuda.Stream()
    with Context(0) as ctx, Context(0) as ref:
        for c in (ctx, ref):
            c.set_cloud_p(P, delta)
            c.set_cloud_q(Q)
        host = ref.try_congruent_set(P[base], quads, 2 * delta)
        ctx.set_stream(S.cuda_stream)
        dq = torch.zeros((len(quads), 4), dtype=torch.int32, device="cuda")   # poison: (0, 0, 0, 0), a degenerate quad
        hq = pinned(quads)
        torch.cuda.synchronize()
        with torch.cuda.stream(S):
            sleep_ms(ORDER_MS)
            dq.copy_(hq, non_blocking=True)
            got = ctx.try_congruent_set_dev(P[base], dq.data_ptr(), len(quads), 2 * delta)
            idle = S.query()
        S.synchronize()
        ctx.set_stream(None)
    assert idle                                                       # it waited for S to read the record back
    for k in ("key", "best_count", "best_index", "n_gate_pass", "n_q", "rms"):
        assert got[k] == host[k], k
    for k in ("T", "centroid1", "centroid2", "quad"):
        assert np.array_equal(common.bits(got[k]) if got[k].dtype == np.float32 else got[k],
                              common.bits(host[k]) if host[k].dtype == np.float32 else host[k]), k
    assert got["best_index"] == want["best_index"] and got["n_gate_pass"] == want["n_gate"]
    assert np.float32(got["best_count"]) / np.float32(got["n_q"]) == np.float32(want["best_lcp"])
    assert np.array_equal(common.bits(got["T"]), common.bits(want["T"]))


# ---- 4. the chain bench.py times -------------------------------------------------------------------------------------

def test_verify_best_dev_chain_at_three_patches(env, sleep_ms, monkeypatch):
    """two s4g_verify_best_dev on S back to back, no synchronisation between them, other candidates and a permuted,
    non-contiguous global index each, the maximum count tied across three chunks, Verify at three query patches (its
    candidate order per patch: a key kernel and a CUB radix sort on the stream): both keys and both count arrays equal
    those of the port's counts"""
    import torch
    from super4pcs_b200 import Context
    rng = np.random.RandomState(6)
    runs = []
    for K, seed, spots in ((96, 7, (5, 37, 90)), (80, 8, (20, 50, 75))):
        T, good, top = with_ties(env.port, common.candidates_colmajor(env.sc, K, seed=seed, n_near=K // 4), spots)
        index = rng.choice(10 ** 6, K, replace=False).astype(np.uint32)
        index[top] = np.sort(index[top])[::-1]                        # the last tied candidate has the smallest index
        want = best_key(good, index)
        assert int(want[0]) & 0xFFFFFFFF == 0xFFFFFFFF - int(index[top[-1]])
        runs.append((T, index, good, want))
    monkeypatch.setenv("S4G_VERIFY_PATCHES", "3")
    S = env.S
    with Context(0) as ctx:
        ctx.set_cloud_p(env.sc["P"], DELTA)
        ctx.set_cloud_q(env.sc["Q"])
        ctx.set_stream(S.cuda_stream)
        bufs = []
        for T, index, _, _ in runs:
            K = len(T)
            dT, dI, dc, dk = (empty((K, 16), torch.float32), empty(K, torch.int32), empty(K, torch.int32),
                              empty(1, torch.int64))
            dT.fill_(float("nan"))
            dI.zero_()
            bufs.append((dT, dI, dc, dk, pinned(T), pinned(index.view(np.int32))))
        torch.cuda.synchronize()
        launches = ctx.timings()["launches"]
        with torch.cuda.stream(S):
            sleep_ms(ORDER_MS)
            outs = []
            for dT, dI, dc, dk, hT, hI in bufs:
                dT.copy_(hT, non_blocking=True)
                dI.copy_(hI, non_blocking=True)
                dc.fill_(-1)
                dk.fill_(-1)
                ctx.verify_best_dev(dT.data_ptr(), len(dT), dI.data_ptr(), dc.data_ptr(), dk.data_ptr())
            for dT, dI, dc, dk, _, _ in bufs:
                outs.append((dc.clone(), dk.clone()))
        S.synchronize()
        # per call: k_pack_rec, the ordered path's key kernel and sort (5 launches), k_verify, k_argmax
        assert ctx.timings()["launches"] - launches >= 2 * 8
        ctx.set_stream(None)
    for (dc, dk), (_, _, good, want) in zip(outs, runs):
        assert np.array_equal(dc.cpu().numpy().view(np.uint32), good)
        assert np.array_equal(dk.cpu().numpy().view(np.uint64), want)


# ---- 5. s4g_set_stream itself ----------------------------------------------------------------------------------------

def test_switching_streams_waits_for_the_old_one(env, sleep_ms):
    """a delayed Verify on S1, then set_stream(S2): when it returns S1 has finished and the counts are final"""
    import torch
    ctx = bound(env)
    S1, S2 = env.S, torch.cuda.Stream()
    K = len(env.T)
    dT, dc, hT = empty((K, 16), torch.float32), empty(K, torch.int32), pinned(env.T)
    dT.fill_(float("nan"))
    torch.cuda.synchronize()
    with torch.cuda.stream(S1):
        sleep_ms(ORDER_MS)
        dT.copy_(hT, non_blocking=True)
        dc.fill_(-1)
        ctx.verify_dev(dT.data_ptr(), K, dc.data_ptr())
    t0 = time.perf_counter()
    ctx.set_stream(S2.cuda_stream)
    host_ms = 1e3 * (time.perf_counter() - t0)
    idle = S1.query()
    S1.synchronize()
    bound(env)
    assert idle, "set_stream returned after %.1f ms with the old stream still busy" % host_ms
    assert np.array_equal(dc.cpu().numpy().view(np.uint32), env.counts)


def test_null_restores_the_contexts_own_stream(env, sleep_ms):
    """after set_stream(NULL) the context runs on its own stream: ctx.synchronize() returns while a sleep on the
    stream it left is still running, with the counts final"""
    import torch
    ctx = bound(env)
    ctx.set_stream(None)
    K = len(env.T)
    dT, dc = torch.from_numpy(env.T).cuda(), empty(K, torch.int32)
    dc.fill_(-1)
    torch.cuda.synchronize()
    try:
        with torch.cuda.stream(env.S):
            sleep_ms(ORDER_MS)
        ctx.verify_dev(dT.data_ptr(), K, dc.data_ptr())
        ctx.synchronize()
        busy = not env.S.query()
        counts = dc.cpu().numpy().view(np.uint32)
    finally:
        env.S.synchronize()
        bound(env)
    assert busy
    assert np.array_equal(counts, env.counts)


def test_legacy_stream_orders_after_torchs_default_stream(env, sleep_ms):
    """torch's default stream has the handle 0, which s4g_set_stream reads as the context's own stream; a caller on it
    passes cudaStreamLegacy, and then the Verify runs after the default stream's sleep and copy and before its read"""
    import torch
    ctx = bound(env)
    default = torch.cuda.default_stream()
    assert default.cuda_stream == 0
    K = len(env.T)
    dT, dc, hT = empty((K, 16), torch.float32), empty(K, torch.int32), pinned(env.T)
    dT.fill_(float("nan"))
    torch.cuda.synchronize()
    ctx.set_stream(CUDA_STREAM_LEGACY)
    try:
        with torch.cuda.stream(default):
            sleep_ms(ORDER_MS)
            dT.copy_(hT, non_blocking=True)
            dc.fill_(-1)
            ctx.verify_dev(dT.data_ptr(), K, dc.data_ptr())
            out = dc.clone()
        torch.cuda.synchronize()
    finally:
        bound(env)
    assert np.array_equal(out.cpu().numpy().view(np.uint32), env.counts)


# ---- 6. contexts and streams -----------------------------------------------------------------------------------------

def test_two_contexts_on_one_stream(env, sleep_ms):
    """a second context with other clouds bound to the same stream, calls of both interleaved with no synchronisation:
    each result equals its own context's host form, so the contexts share no scratch"""
    import torch
    from super4pcs_b200 import Context
    scB = common.scenario(20000, 0.4, DELTA, seed=6)
    TB = common.candidates_colmajor(scB, len(env.T), seed=9, n_near=12)
    ptB = oport.Port(scB["P"], scB["Q"], DELTA)
    countsB = ptB.verify_batch(TB, 0.0, nthreads=oport.num_threads())[1]
    ptB.close()
    assert not np.array_equal(countsB, env.counts)
    ctx = bound(env)
    K, n, k = len(env.T), len(env.X), 16
    with Context(0) as ctxB, Context(0) as refB:
        for c in (ctxB, refB):
            c.set_cloud_p(scB["P"], DELTA)
            c.set_cloud_q(scB["Q"])
        wantA, wantB = env.ref.knn(env.X, k)[0], refB.knn(env.X, k)[0]
        assert not np.array_equal(wantA, wantB)
        ctxB.set_stream(env.S.cuda_stream)
        dTA, dTB, dX = empty((K, 16), torch.float32), empty((K, 16), torch.float32), empty((n, 3), torch.float32)
        for d in (dTA, dTB, dX):
            d.fill_(float("nan"))
        cA, cB, iA, iB = empty(K, torch.int32), empty(K, torch.int32), empty((n, k), torch.int32), empty((n, k), torch.int32)
        hTA, hTB, hX = pinned(env.T), pinned(TB), pinned(env.X)
        torch.cuda.synchronize()
        with torch.cuda.stream(env.S):
            sleep_ms(ORDER_MS)
            for d, h in ((dTA, hTA), (dTB, hTB), (dX, hX)):
                d.copy_(h, non_blocking=True)
            for o in (cA, cB, iA, iB):
                o.fill_(-7)
            ctx.verify_dev(dTA.data_ptr(), K, cA.data_ptr())
            ctxB.verify_dev(dTB.data_ptr(), K, cB.data_ptr())
            ctx.knn_dev(dX.data_ptr(), n, k, iA.data_ptr())
            ctxB.knn_dev(dX.data_ptr(), n, k, iB.data_ptr())
            outs = [o.clone() for o in (cA, cB, iA, iB)]
        env.S.synchronize()
        ctxB.set_stream(None)
    got = [o.cpu().numpy() for o in outs]
    assert np.array_equal(got[0].view(np.uint32), env.counts)
    assert np.array_equal(got[1].view(np.uint32), countsB)
    assert np.array_equal(got[2], wantA)
    assert np.array_equal(got[3], wantB)


def test_one_context_moved_between_two_streams(env, sleep_ms):
    """Verify on S1, k-nearest on S2, Verify again on S1, each behind a sleep on its stream and reading inputs copied
    there, the context switched between the calls: every result equals the host form"""
    import torch
    ctx = bound(env)
    S1, S2 = env.S, torch.cuda.Stream()
    K, n, k = len(env.T), len(env.X), 16
    T2 = env.T[::-1].copy()
    dT1, dT2, dX = empty((K, 16), torch.float32), empty((K, 16), torch.float32), empty((n, 3), torch.float32)
    for d in (dT1, dT2, dX):
        d.fill_(float("nan"))
    c1, c2, ix = empty(K, torch.int32), empty(K, torch.int32), empty((n, k), torch.int32)
    for o in (c1, c2, ix):
        o.fill_(-7)
    h1, h2, hX = pinned(env.T), pinned(T2), pinned(env.X)
    torch.cuda.synchronize()
    try:
        with torch.cuda.stream(S1):
            sleep_ms(ORDER_MS)
            dT1.copy_(h1, non_blocking=True)
            ctx.verify_dev(dT1.data_ptr(), K, c1.data_ptr())
        ctx.set_stream(S2.cuda_stream)
        with torch.cuda.stream(S2):
            sleep_ms(ORDER_MS)
            dX.copy_(hX, non_blocking=True)
            ctx.knn_dev(dX.data_ptr(), n, k, ix.data_ptr())
        ctx.set_stream(S1.cuda_stream)
        with torch.cuda.stream(S1):
            sleep_ms(ORDER_MS)
            dT2.copy_(h2, non_blocking=True)
            ctx.verify_dev(dT2.data_ptr(), K, c2.data_ptr())
    finally:
        S1.synchronize()
        S2.synchronize()
    assert np.array_equal(c1.cpu().numpy().view(np.uint32), env.counts)
    assert np.array_equal(c2.cpu().numpy().view(np.uint32), env.counts[::-1])
    assert np.array_equal(ix.cpu().numpy(), env.ref.knn(env.X, k)[0])
