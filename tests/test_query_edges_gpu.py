"""The point queries where the box descent's decisions flip (tests/query_edges.py builds the fixtures): every fixture
through knn (k = 1, at and around the k-th tie, 64), nearest, range_query (count and fill passes), radius_outliers
(counts and keep flags) and euclidean_clusters, each bit-equal to the brute force, in every regime, without T and under
a rigid T.  A wrong eps, a dropped (1 - 2^-20) factor or a wrong face offset in cells_bound drops a point the brute force
takes on some fixture here (tests/test_query_edges_cpu.py shows which)."""
import numpy as np
import pytest

from oracle import clusters as oclusters
from oracle import knn as oknn
from oracle import outliers as ooutliers
from oracle import range as orange
from tests import common
from tests import edges as E
from tests import query_edges as QE

pytestmark = pytest.mark.gpu

f32 = np.float32


@pytest.fixture
def make_ctx(s4g_lib, monkeypatch):
    from super4pcs_b200 import Context
    made = []

    def make(cshift_min=None):
        if cshift_min is None:
            monkeypatch.delenv("S4G_CSHIFT_MIN", raising=False)
        else:
            monkeypatch.setenv("S4G_CSHIFT_MIN", str(cshift_min))
        made.append(Context(0))
        return made[-1]
    yield make
    for c in made:
        c.close()


def bits_equal(a, b):
    return np.array_equal(common.bits(np.asarray(a, f32)), common.bits(np.asarray(b, f32)))


def loaded(make_ctx, name):
    sc = QE.scene(name)
    ctx = make_ctx(QE.env_cshift(name))
    ctx.set_cloud_p(sc["P"], sc["delta"])
    gs = ctx.grid_stats()
    assert gs["cell_edge"] == float(f32(sc["g"]["h"])) and gs["cells"] == sc["g"]["cells"]
    return sc, ctx


@pytest.mark.parametrize("name", list(QE.REGIMES))
def test_queries_bit_equal(make_ctx, name):
    sc, ctx = loaded(make_ctx, name)
    P = sc["P"]
    T16 = E.colmajor(sc["T34"])[0]
    for q in sc["queries"]:
        T = T16 if q["T"] else None
        x = q["x"][None]
        ex = np.array([q["exclude"]], np.int32)
        what = (q["family"], q["kind"], q["T"])
        for r in q["radii"]:
            want = oknn.bruteforce(P, x, 64, r, T, ex)
            for k in q["ks"]:
                got = ctx.knn(x, k, r, T=T, exclude=ex)
                assert np.array_equal(got[0], want[0][:, :k]), (what, k, r, got[0], want[0][:, :k])
                assert bits_equal(got[1], want[1][:, :k]), (what, k, r)
            idx, sq = ctx.nearest(x, r, T=T, exclude=ex)
            assert idx[0] == want[0][0, 0] and bits_equal(sq, want[1][:, 0]), (what, r)
            off, ind, sqd = ctx.range_query(x, r, T=T)
            woff, wind, wsq = orange.bruteforce(P, x, r, T)
            assert np.array_equal(off, woff) and np.array_equal(ind, wind) and bits_equal(sqd, wsq), (what, r)
        if q["family"] == "D" and not (np.abs(q["y"]) == 1e19).any():
            # every d^2 overflows: the k smallest indices at +inf, nothing within FLT_MAX, empty range lists
            got = ctx.knn(x, 3, np.inf)
            assert list(got[0][0]) == [0, 1, 2] and np.isinf(got[1]).all()
            assert (ctx.knn(x, 3, QE.FLT_MAX)[0] == -1).all()
            assert ctx.range_query(x, np.inf)[0][-1] == 0


@pytest.mark.parametrize("name", list(QE.REGIMES))
def test_radius_counts_and_cluster_links(make_ctx, name):
    sc, ctx = loaded(make_ctx, name)
    P = sc["P"]
    for pr in sc["pairs"]:
        for r in pr["radii"]:
            if pr["family"] == "F":
                _, _, raw = ooutliers.radius(P, r, len(P), raw=True)
                c = int(raw[pr["b"]])
                for m in (c, c + 1):
                    keep, counts = ctx.radius_outliers(r, m)
                    wkeep, wcounts = ooutliers.radius(P, r, m)
                    assert np.array_equal(keep, wkeep) and np.array_equal(counts, wcounts), (pr["kind"], r, m)
            else:
                labels, root, off, mem = ctx.euclidean_clusters(r)
                wl, wr, wo, wm = oclusters.clusters(P, r)
                assert np.array_equal(root, wr) and np.array_equal(labels, wl), (pr["kind"], r)
                assert np.array_equal(off, wo) and np.array_equal(mem, wm)
                assert (root[pr["a"]] == root[pr["b"]]) == bool(pr["d2"] < r)
