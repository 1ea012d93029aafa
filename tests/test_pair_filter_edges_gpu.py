"""k_pairs' normal, colour, translation and angle filters where their decisions flip, pair set by pair set against the
oracle of tests/pair_filters.py: for one base (s4g_extract_pairs), for a batch of 64 bases (s4g_try_bases, every base with
its own base points, rgb and normal angles), and at the shapes where the kernel's schedule changes -- a dense ball whose
survivors overflow the shared queue, group-boundary cloud sizes, and lists that outgrow the first slot / key buffer."""
import numpy as np
import pytest

from tests import pair_filters as F

pytestmark = pytest.mark.gpu

GROUPS = {"segments": F.segment_cases, "angle_sweep": F.angle_sweep_cases, "special": F.special_cases}


@pytest.fixture(scope="module")
def ctx(s4g_lib):
    from super4pcs_b200 import Context
    c = Context(0)
    yield c
    c.close()


def _set_q(ctx, cloud):
    if getattr(ctx, "_pf_cloud", None) != cloud["name"]:
        ctx.set_cloud_p(cloud["Q"], 0.01)
        ctx.set_cloud_q(cloud["Q"], normals=cloud["Qn"], rgb=cloud["Qrgb"])
        ctx._pf_cloud = cloud["name"]


def _extract(ctx, case):
    from super4pcs_b200 import PairFilters
    return ctx.extract_pairs(case["d"], float(case["na"]), case["eps"], case["b1"], case["b2"],
                             PairFilters(*case["filters"]), slot=0)


@pytest.mark.parametrize("group", list(GROUPS))
def test_one_base_equals_the_oracle(ctx, group):
    bad = []
    for case in GROUPS[group]():
        _set_q(ctx, case["cloud"])
        got, want = _extract(ctx, case), F.oracle_pairs(case)
        if not np.array_equal(got, want):
            bad.append((case["name"], len(got), len(want)))
    assert not bad, bad


def test_batch_of_64_bases_equals_the_oracle_and_the_per_base_chain(ctx):
    """128 segments (the segment cases, then again in a shifted pairing), all four filters on: every segment's pair count
    equals the oracle's, and n_quads and the TryCongruentSet record equal the per-base chain's"""
    from super4pcs_b200 import PairFilters
    segs = F.segment_cases()
    segs = (segs + segs[1:])[:128]
    cloud = segs[0]["cloud"]
    _set_q(ctx, cloud)
    bases = F.batch_bases(segs, cloud["Q"])
    assert len(bases) == 64
    filt = PairFilters(*F.FILTERS)
    got = ctx.try_bases(bases, F.EPS, F.EPS, F.EPS, filters=filt)
    assert len(got) == 64
    want = [[len(F.oracle_pairs(s)) for s in b["cases"]] for b in bases]
    assert [g["n_pairs"] for g in got] == want
    for b, g in zip(bases, got):
        s0, s1 = b["cases"]
        n1 = ctx.extract_pairs(b["d1"], b["na1"], F.EPS, s0["b1"], s0["b2"], filt, slot=0, fetch=False)
        n2 = ctx.extract_pairs(b["d2"], b["na2"], F.EPS, s1["b1"], s1["b2"], filt, slot=1, fetch=False)
        assert g["n_pairs"] == [n1, n2]
        nq = ctx.find_quads(b["inv1"], b["inv2"], F.EPS, b["b9"][:, :3], fetch=False) if n1 and n2 else 0
        assert g["n_quads"] == nq
        if nq == 0:
            assert g["tcs"]["best_index"] == -1 and g["tcs"]["n_gate_pass"] == 0
            continue
        w = ctx.try_congruent_set_resident(b["bxp"], F.EPS)
        t = g["tcs"]
        for k in ("key", "best_count", "best_index", "n_gate_pass", "n_q"):
            assert t[k] == w[k], k
        assert np.array_equal(t["T"].view(np.uint32), w["T"].view(np.uint32))
        assert np.array_equal(t["centroid1"].view(np.uint32), w["centroid1"].view(np.uint32))
        assert np.array_equal(t["centroid2"].view(np.uint32), w["centroid2"].view(np.uint32))


BALL = dict(n=640, d=0.05, eps=0.2)
BALL_FILTERS = {"angle": ((-1.0, -1.0, 90.0, -1.0), F.b9([0, 0, 0]), F.b9([0.3, 0.1, 0.2])),
                "colour": ((-1.0, -1.0, -1.0, 0.7), F.b9([0, 0, 0]), F.b9([0.3, 0.1, 0.2], (0.4, 0.6, 0.5)))}


@pytest.mark.parametrize("which", list(BALL_FILTERS))
def test_dense_ball_overflows_the_queue_and_the_first_slot_buffer(s4g_lib, which):
    """every pair passes the pre-filter (d - eps <= 0), so each test step has 16384 survivors for a 4096-entry queue;
    more than 131072 ordered pairs on a fresh context's first call (the slot buffer starts at 1 MiB)"""
    from super4pcs_b200 import Context
    cloud = F.dense_ball(BALL["n"])
    filters, b1, b2 = BALL_FILTERS[which]
    case = dict(cloud=cloud, d=BALL["d"], eps=BALL["eps"], na=np.float32(0), b1=b1, b2=b2, filters=filters)
    I, J, r = F.pair_bits(cloud["Q"], cloud["Qn"], cloud["Qrgb"], case["d"], 0, case["eps"], b1, b2, filters)
    assert len(F.band_pairs(cloud["Q"], case["d"], case["eps"])[0]) == BALL["n"] * (BALL["n"] - 1) // 2
    want = F.ordered(I, J, r)
    assert len(want) > 131072
    if which == "angle":
        assert (r != 3).mean() > 0.99                # one orientation per pair: the uneven append path
    with Context(0) as c:
        c.set_cloud_p(cloud["Q"], 0.01)
        c.set_cloud_q(cloud["Q"], normals=cloud["Qn"], rgb=cloud["Qrgb"])
        assert np.array_equal(_extract(c, case), want)


@pytest.mark.parametrize("n", [1, 63, 64, 65, 4095, 4096, 4097])
def test_group_boundary_sizes_with_every_filter(ctx, n):
    cloud = F.random_cloud(n)
    case = dict(cloud=cloud, d=0.3, eps=0.05, na=np.float32(0.3), b1=F.b9([0, 0, 0]),
                b2=F.b9([0.05, 0.01, 0], (0.6, 0.4, 0.5)), filters=(30.0, 0.6, 60.0, 0.5))
    _set_q(ctx, cloud)
    want = F.oracle_pairs(case)
    assert np.array_equal(_extract(ctx, case), want)
    if n >= 4095:
        assert len(want) > 1000


def test_batch_key_buffer_grows_on_a_fresh_context(s4g_lib):
    """more than 131072 keys in the first s4g_try_bases of a context (the key buffer starts at 1 MiB)"""
    from super4pcs_b200 import Context, PairFilters
    cloud = F.dense_ball(BALL["n"])
    filters = (-1.0, -1.0, -1.0, 0.7)
    b9s = [np.stack([F.b9([0, 0, 0], rgb), F.b9([0.3, 0.1, 0.2], rgb), F.b9([0, 0, 0]), F.b9([0, 0, 1])])
           for rgb in ((0.5, 0.5, 0.5), (0.3, 0.6, 0.5))]
    bases = [dict(d1=BALL["d"], d2=5.0, na1=0.0, na2=0.0, b9=b, bxp=cloud["Q"][:4], inv1=0.5, inv2=0.5) for b in b9s]
    want = [[len(F.oracle_pairs(dict(cloud=cloud, d=b["d1"], eps=BALL["eps"], na=0, b1=b["b9"][0], b2=b["b9"][1],
                                     filters=filters))), 0] for b in bases]
    assert sum(w[0] for w in want) > 131072
    with Context(0) as c:
        c.set_cloud_p(cloud["Q"], 0.01)
        c.set_cloud_q(cloud["Q"], normals=cloud["Qn"], rgb=cloud["Qrgb"])
        got = c.try_bases(bases, BALL["eps"], BALL["eps"], BALL["eps"], filters=PairFilters(*filters))
    assert [g["n_pairs"] for g in got] == want
    assert all(g["n_quads"] == 0 for g in got)
