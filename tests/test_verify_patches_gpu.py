"""Verify's query-patch schedule (k_verify, choose_patches; DESIGN.md section 3.1) at every patch count.

The Morton-ordered queries are cut into NP patches of `ptiles` consecutive super-tiles (1024 queries each).  With NP > 1
and more than one chunk of 16 candidates, every patch has its own candidate order (k_verify_keys + one CUB radix sort:
robust-path candidates in their own key bucket, candidates beyond a device-side count last), and each CTA adds into
counts[perm[...]].  The count derived from the L2 size only exceeds 1 at about a million queries, so these tests request
it through S4G_VERIFY_PATCHES (read when a context is created) at sizes where the CPU port is cheap, and compare integer
counts exactly with the port (pinned bit for bit to the unmodified reference) and with the reference when it is present.
One test runs the automatic schedule at the production size (1M x 1M).

Not covered: the slab loop of launches beyond 2^31 - 1 CTAs and the fall-back to one patch when NP * K > 2^31 - 1; neither
is reachable at a size a test can afford.
"""
import numpy as np
import pytest

from oracle import _build
from oracle import port as oport
from oracle import ref as oref
from super4pcs_b200 import synth
from tests import common
from tests.test_batch_gpu import _bases
from tests.test_host_logic_cpu import run_driver

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(_build.build_ref() is None, reason="oracle/_ref (compiled reference) not present")

SUPER_TILE = 1024          # queries per super-tile: 8 tiles of 128 (verify.cu kThreads * kTilesPerBlock)
MAX_PATCHES = 16           # kVerifyMaxPatches
KS = (1, 16, 17, 33, 96, 1000)   # one candidate, exactly one chunk, one chunk + 1, several and many chunks


def patch_layout(nQ, requested):
    """(NP, super-tiles per patch, super-tiles of the last patch) that choose_patches gives for a requested count > 0"""
    nst = -(-nQ // SUPER_TILE)
    np_ = max(1, min(requested, MAX_PATCHES, nst))
    ptiles = -(-nst // np_)
    NP = -(-nst // ptiles)
    return NP, ptiles, nst - (NP - 1) * ptiles


def auto_patches(nQ, grid_bytes, l2_bytes):
    """NP of the automatic schedule (choose_patches without a request)"""
    req = int(np.ceil(2.0 * (nQ * 16.0 + grid_bytes) / l2_bytes))
    return patch_layout(nQ, max(1, req))[0]


@pytest.fixture
def make_ctx(s4g_lib, monkeypatch):
    """make_ctx(patches) -> a fresh Context created with S4G_VERIFY_PATCHES = patches (None: unset)"""
    from super4pcs_b200 import Context
    made = []

    def make(patches):
        if patches is None:
            monkeypatch.delenv("S4G_VERIFY_PATCHES", raising=False)
        else:
            monkeypatch.setenv("S4G_VERIFY_PATCHES", str(patches))
        c = Context(0)
        made.append(c)
        return c
    yield make
    for c in made:
        c.close()


def verify_counted(ctx, T):
    """(counts, kernel launches that ctx.verify(T) enqueued)"""
    before = ctx.timings()["launches"]
    counts = ctx.verify(T)
    return counts, ctx.timings()["launches"] - before


def _colmajor(M):
    return np.ascontiguousarray(np.asarray(M, np.float32).transpose(0, 2, 1)).reshape(-1, 16)


def mixed_candidates(sc, K, seed=3):
    """K column-major candidates, every kind in the first chunks already:
      k % 8 == 3           robust path: NaN, 3x3 part scaled by 1e4, translation 1000 (in turn)
      k % 8 == 6           non-rigid near-ground-truth: shear or anisotropic scale (fast path, larger cull radius)
      k % 16 == 0, k > 0   exact duplicate of candidate k - 14 (a near-ground-truth one in another chunk)
      other even k         near-ground-truth motion with its own offset (<= 2 delta, <= 0.5 deg): counts that differ
      other odd k          random rigid motion"""
    near = synth.candidate_transforms(K, sc["delta"], seed=seed, n_near=K, centroid_p=sc["cp"], centroid_q=sc["cq"])
    rand = synth.candidate_transforms(K, sc["delta"], seed=seed + 1, n_near=0, centroid_p=sc["cp"], centroid_q=sc["cq"])
    rng = np.random.RandomState(seed)
    out = np.empty((K, 4, 4), np.float32)
    for k in range(K):
        if k % 8 == 3:
            kind = (k // 8) % 3
            if kind == 0:
                M = np.full((4, 4), np.nan, np.float32)
            elif kind == 1:
                M = near[k].copy()
                M[:3, :3] *= np.float32(1e4)
            else:
                M = np.eye(4, dtype=np.float32)
                M[:3, 3] = 1000.0
        elif k % 8 == 6:
            A = np.eye(4)
            if (k // 8) % 2 == 0:
                A[0, 1] = 0.05 + 0.25 * rng.random_sample()
            else:
                A[:3, :3] = np.diag([1.1, 0.9, 1.05])
            M = (near[k].astype(np.float64) @ A).astype(np.float32)
        elif k % 16 == 0 and k > 0:
            M = out[k - 14].copy()
        elif k % 2 == 0:
            M = near[k]
        else:
            M = rand[k]
        out[k] = M
    return _colmajor(out)


# ---- scenarios: 20 000 queries (20 super-tiles) and 33 816 (34 super-tiles, the last one 24 queries) -----------------

SCENARIOS = {20000: dict(n=20000, delta=0.01, seed=5), 33816: dict(n=33816, delta=0.01, seed=6)}
_oracle_cache = {}


def scenario_and_oracle(nq):
    """(scenario, candidates (1000), the port's counts [, the reference's counts when present]) -- computed once"""
    if nq not in _oracle_cache:
        s = SCENARIOS[nq]
        sc = common.scenario(s["n"], 0.4, s["delta"], seed=s["seed"])
        T = mixed_candidates(sc, max(KS))
        pt = oport.Port(sc["P"], sc["Q"], s["delta"])
        _, good, _ = pt.verify_batch(T, 0.0, nthreads=oport.num_threads())
        ref = None
        if oref.available():
            opt = oref.make_options(delta=s["delta"], sample_size=10 ** 8, overlap=0.4)
            m = oref.RefMatcher(sc["raw"]["P"], sc["raw"]["Q"], opt)
            ref, _ = m.verify_batch(T, 0.0, nthreads=oref.num_threads())
            m.close()
        _oracle_cache[nq] = (sc, T, good, ref)
    return _oracle_cache[nq]


LAYOUTS = [  # (queries, requested, NP, super-tiles per patch, super-tiles of the last patch)
    (20000, 1, 1, 20, 20), (20000, 2, 2, 10, 10), (20000, 3, 3, 7, 6), (20000, 7, 7, 3, 2), (20000, 16, 10, 2, 2),
    (33816, 1, 1, 34, 34), (33816, 2, 2, 17, 17), (33816, 3, 3, 12, 10), (33816, 7, 7, 5, 4), (33816, 16, 12, 3, 1),
]


@pytest.mark.parametrize("nq,req,NP,ptiles,last", LAYOUTS)
def test_counts_at_every_patch_count(make_ctx, nq, req, NP, ptiles, last):
    assert patch_layout(nq, req) == (NP, ptiles, last)
    sc, T, good, ref = scenario_and_oracle(nq)
    assert len(np.unique(good[good > 0])) > 20                       # counts differ: a permuted write cannot hide
    one = make_ctx(1)
    ctx = make_ctx(req)
    for c in (one, ctx):
        c.set_cloud_p(sc["P"], sc["delta"])
        c.set_cloud_q(sc["Q"])
    for K in KS:
        got, launches = verify_counted(ctx, T[:K])
        assert np.array_equal(got, good[:K]), K
        if ref is not None:
            assert np.array_equal(got.astype(np.float32) / np.float32(nq), ref[:K]), K
        _, launches1 = verify_counted(one, T[:K])
        if NP > 1 and K > 16:
            assert launches > launches1, K                           # the per-patch order (key kernel + sort) ran
        else:
            assert launches == launches1, K                          # one patch or one chunk: nothing to order


@pytest.mark.parametrize("nq,req", [(20000, 2), (20000, 3), (20000, 7), (20000, 16), (33816, 3), (33816, 16)])
def test_probe_statistics_do_not_depend_on_the_patch_count(make_ctx, nq, req):
    """every (query, candidate) pair is decided by one CTA from the same data whatever the order (DESIGN.md 3.1): the
    counts and all five probe statistics equal those of the one-patch schedule"""
    sc, T, good, _ = scenario_and_oracle(nq)
    one, ctx = make_ctx(1), make_ctx(req)
    for c in (one, ctx):
        c.set_cloud_p(sc["P"], sc["delta"])
        c.set_cloud_q(sc["Q"])
    for K in KS:
        assert np.array_equal(ctx.verify(T[:K]), one.verify(T[:K])), K
        assert ctx.verify_probe_stats(T[:K]) == one.verify_probe_stats(T[:K]), K
    assert one.verify_probe_stats(T)["tile_pairs_culled"] > 0


@pytest.mark.parametrize("nq,req", [(700, 7), (1, 16)])
def test_fewer_queries_than_one_super_tile(make_ctx, nq, req):
    """the request is clamped to the number of super-tiles: one patch, no sort"""
    assert patch_layout(nq, req)[0] == 1
    sc, T, _, _ = scenario_and_oracle(20000)
    Q = np.ascontiguousarray(sc["Q"][:nq])
    pt = oport.Port(sc["P"], Q, sc["delta"])
    _, good, _ = pt.verify_batch(T, 0.0, nthreads=oport.num_threads())
    one, ctx = make_ctx(1), make_ctx(req)
    for c in (one, ctx):
        c.set_cloud_p(sc["P"], sc["delta"])
        c.set_cloud_q(Q)
    got, launches = verify_counted(ctx, T)
    assert np.array_equal(got, good)
    assert launches == verify_counted(one, T)[1]
    if nq > 1:
        assert good.max() > 0


def test_context_reuse_rebuilds_what_the_clouds_change(make_ctx):
    """requested NP = 3 on one context: a new Q cloud of the same size (the cached patch centres are rebuilt), a new
    delta for P (grid and Morton scale of the keys change), a smaller K after a larger one (the grown sort buffer is
    reused): counts equal the port's after every step"""
    sc, T, good, _ = scenario_and_oracle(20000)
    P, delta = sc["P"], sc["delta"]
    Q2 = np.ascontiguousarray(common.scenario(20000, 0.4, delta, seed=9)["Q"])
    assert not np.array_equal(Q2, sc["Q"])
    ctx = make_ctx(3)
    ctx.set_cloud_p(P, delta)
    ctx.set_cloud_q(sc["Q"])
    assert np.array_equal(ctx.verify(T[:96]), good[:96])
    ctx.set_cloud_q(Q2)
    first, n_first = verify_counted(ctx, T[:96])
    again, n_again = verify_counted(ctx, T[:96])
    assert n_first == n_again + 1                                    # the new cloud's patch centres, once
    _, good2, _ = oport.Port(P, Q2, delta).verify_batch(T, 0.0, nthreads=oport.num_threads())
    assert np.array_equal(first, good2[:96]) and np.array_equal(again, good2[:96])
    ctx.set_cloud_p(P, 2 * delta)
    _, good3, _ = oport.Port(P, Q2, 2 * delta).verify_batch(T, 0.0, nthreads=oport.num_threads())
    assert not np.array_equal(good3, good2)
    for K in (33, 1000, 40, 17):
        got, launches = verify_counted(ctx, T[:K])
        assert np.array_equal(got, good3[:K]), K
        assert launches > 2, K                                       # still the ordered path


def test_verify_best_key_with_a_permuted_index(make_ctx):
    """s4g_verify_best at NP = 7: a permuted, non-contiguous index array and the maximum count tied between three
    candidates in different chunks -- the key is max_k (count_k << 32 | 0xFFFFFFFF - index_k) of the port's counts"""
    sc, T0, good0, _ = scenario_and_oracle(20000)
    T = T0[:96].copy()
    a = int(np.argmax(good0[:96]))
    ties = [p for p in (5, 37, 90) if p // 16 != a // 16][:2]        # copies of the best candidate in two other chunks
    T[ties] = T[a]
    _, good, _ = oport.Port(sc["P"], sc["Q"], sc["delta"]).verify_batch(T, 0.0, nthreads=oport.num_threads())
    top = np.nonzero(good == good.max())[0]
    assert set(top) >= {a, *ties} and len(set(top // 16)) >= 3
    rng = np.random.RandomState(4)
    index = rng.choice(10 ** 6, 96, replace=False).astype(np.uint32)
    index[top] = np.sort(index[top])[::-1]                           # the last of the tied candidates has the smallest index
    want = int(((good.astype(np.uint64) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - index.astype(np.uint64))).max())
    assert want & 0xFFFFFFFF == 0xFFFFFFFF - int(index[top[-1]])
    ctx = make_ctx(7)
    ctx.set_cloud_p(sc["P"], sc["delta"])
    ctx.set_cloud_q(sc["Q"])
    counts, key = ctx.verify_best(T, index)
    assert np.array_equal(counts, good)
    assert key == want
    counts, key = ctx.verify_best(T)                                 # no index array: the position is the index
    assert np.array_equal(counts, good)
    assert key == (int(good.max()) << 32 | (0xFFFFFFFF - int(top[0])))


@pytest.mark.parametrize("world", [1, 2])
def test_try_congruent_set_at_three_patches(make_ctx, world):
    """records written by k_rigid<1> for the gate-compacted list, verified at NP = 3 (3000 queries = 3 super-tiles, one
    each): gate count, winner index, LCP and transform bits equal the port's (and the reference's)"""
    assert patch_layout(3000, 3) == (3, 1, 1)
    delta = 0.05
    sc = common.scenario(3000, 0.4, delta)
    rng = np.random.RandomState(11)
    zP = (sc["P"] + sc["cp"])[:, 2]
    base = rng.choice(np.nonzero(np.abs(zP) < 0.15)[0], 4, replace=False).astype(np.int32)
    quads = common.congruent_like_quads(sc, base, 3000, 5)          # (near-congruent at even positions)
    quads = quads[np.random.RandomState(12).permutation(len(quads))]   # ... spread over both shards
    want = oport.Port(sc["P"], sc["Q"], delta).try_congruent_set(base, quads, best_lcp_in=0.0)
    assert want["best_index"] >= 0
    one, ctx = make_ctx(1), make_ctx(3)
    for c in (one, ctx):
        c.set_cloud_p(sc["P"], delta)
        c.set_cloud_q(sc["Q"])
    shards, shards1 = [], []
    for r in range(world):
        n0, n1 = ctx.timings()["launches"], one.timings()["launches"]
        shards.append(ctx.try_congruent_set(sc["P"][base], quads, 2 * delta, shard_rank=r, shard_world=world))
        shards1.append(one.try_congruent_set(sc["P"][base], quads, 2 * delta, shard_rank=r, shard_world=world))
        assert shards[-1]["n_gate_pass"] > 3 * 16                  # several chunks ...
        assert ctx.timings()["launches"] - n0 > one.timings()["launches"] - n1   # ... ordered per patch
    assert sum(s["n_gate_pass"] for s in shards) == want["n_gate"]
    key = max(s["key"] for s in shards)
    win = [s for s in shards if s["key"] == key][0]
    assert win["best_index"] == want["best_index"]
    lcp = np.float32(win["best_count"]) / np.float32(win["n_q"])
    assert lcp == np.float32(want["best_lcp"])
    assert np.array_equal(common.bits(win["T"]), common.bits(want["T"]))
    for s, s1 in zip(shards, shards1):                              # every shard's record equals the one-patch schedule's
        for k in ("key", "best_count", "best_index", "n_gate_pass", "n_q"):
            assert s[k] == s1[k], k
        assert np.array_equal(common.bits(s["T"]), common.bits(s1["T"]))
    if oref.available() and world == 1:
        opt = oref.make_options(delta=delta, sample_size=10 ** 8, overlap=0.4)
        m = oref.RefMatcher(sc["raw"]["P"], sc["raw"]["Q"], opt)
        m.set_best_lcp(0.0)
        r = m.try_congruent_set(base, quads)
        assert r["n_gate"] == win["n_gate_pass"]
        assert np.float32(r["best_lcp"]) == lcp
        assert np.array_equal(common.bits(r["T"]), common.bits(win["T"]))
        assert np.array_equal(r["congruent"], quads[win["best_index"]])


@pytest.mark.parametrize("n,ns,delta,normals,nb,req", [(50000, 3000, 0.01, False, 5, 3), (30000, 2000, 0.015, True, 9, 2)])
def test_try_bases_winners_equal_the_one_patch_schedule(make_ctx, n, ns, delta, normals, nb, req):
    """s4g_try_bases (records from k_brigid, candidate count on the device, candidates beyond it keyed last) at NP > 1:
    every base's winner record equals that of a context at NP = 1 -- key, count, index, gate passes, transform bits"""
    from super4pcs_b200 import PairFilters
    assert patch_layout(ns, req)[0] == req
    sc = common.scenario(n, 0.5, delta, seed=n % 97, normals=normals)
    rng = np.random.RandomState(ns)
    sel = rng.choice(n, ns, replace=False)
    Qs = np.ascontiguousarray(sc["Q"][sel])
    Qn = (sc["Qn"][sel] / np.linalg.norm(sc["Qn"][sel], axis=1, keepdims=True)).astype(np.float32) if normals else None
    filt = PairFilters(35.0, -1, -1, -1) if normals else PairFilters(-1, -1, -1, -1)
    diameter = float(np.linalg.norm(sc["P"].max(0) - sc["P"].min(0)))
    bases = _bases(sc["P"], sc["Pn"] if normals else None, rng, nb, diameter)
    eps = 2 * delta
    one, ctx = make_ctx(1), make_ctx(req)
    res, launches = [], []
    for c in (one, ctx):
        c.set_cloud_p(sc["P"], delta)
        c.set_cloud_q(Qs, normals=Qn)
        n0 = c.timings()["launches"]
        res.append(c.try_bases(bases, eps, eps, eps, filters=filt))
        launches.append(c.timings()["launches"] - n0)
    assert launches[1] > launches[0]                                 # the batch's Verify was ordered per patch
    assert sum(r["tcs"]["n_gate_pass"] for r in res[0]) > 16
    for a, b in zip(res[0], res[1]):
        assert a["n_pairs"] == b["n_pairs"] and a["n_quads"] == b["n_quads"]
        for k in ("key", "best_count", "best_index", "n_gate_pass", "n_q"):
            assert a["tcs"][k] == b["tcs"][k], k
        assert np.array_equal(common.bits(a["tcs"]["T"]), common.bits(b["tcs"]["T"]))
    assert any(r["tcs"]["best_index"] >= 0 for r in res[0])


def test_production_size_with_the_automatic_schedule(make_ctx):
    """1M x 1M, S4G_VERIFY_PATCHES unset: NP is what the card's L2 gives (5 on an H100).  Full counts of 32 mixed
    candidates against the port, probe statistics against a one-patch context, and the ordered path really ran."""
    import torch
    n, delta = 1_000_000, 0.003
    sc = common.scenario(n, 0.3, delta, seed=42)
    T = mixed_candidates(sc, 32, seed=8)
    auto, one = make_ctx(None), make_ctx(1)
    for c in (auto, one):
        c.set_cloud_p(sc["P"], delta)
        c.set_cloud_q(sc["Q"])
    NP = auto_patches(n, auto.grid_stats()["resident_bytes"], torch.cuda.get_device_properties(0).L2_cache_size)
    assert NP > 1
    got, launches = verify_counted(auto, T)
    _, launches1 = verify_counted(one, T)
    assert launches > launches1
    _, good, _ = oport.Port(sc["P"], sc["Q"], delta).verify_batch(T, 0.0, nthreads=oport.num_threads())
    assert np.array_equal(got, good)
    assert (good[0::2][good[0::2] > 0]).size >= 8                     # the near-ground-truth candidates see the overlap
    assert auto.verify_probe_stats(T) == one.verify_probe_stats(T)


# ---- the C++ layer: a synthetic pair whose sampled Q spans 4 super-tiles (s4g_try_bases on by default) ----------------

@pytest.fixture(scope="module")
def built(s4g_lib):
    from super4pcs_b200 import build_cpp
    if build_cpp.build_all()["lib"] is None or _build.build_dropin_harness() is None:
        pytest.skip("C++ layer not available")


@needs_ref
def test_cpp_layer_at_several_patches_matches_the_reference(built):
    """sampled-Q digest, then after every stepwise call the return value, best LCP, progress reports and the matrix bits
    equal the reference's at 1 and 4 patches, with the batched bases (s4g_try_bases) and with the per-base chain"""
    want = run_driver("patches", "reference")
    for patches in ("1", "4"):
        for batch in ("32", "1"):
            env = {"S4G_VERIFY_PATCHES": patches, "S4PCS_BATCH": batch}
            assert run_driver("patches", "dropin", extra_env=env, timeout=600) == want, env
