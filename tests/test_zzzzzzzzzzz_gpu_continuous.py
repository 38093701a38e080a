"""K2c site_continuous on the GPU: sx_cont_qscore[_dev] over the whole GQ grid equals the reference's frozen answers with no tie flag;
sx_site_continuous[_dev] equals the kernels' body compiled with g++ bit for bit (doubles included) on seeded multi-sample columns, deep
mitochondrial-like columns among them, and so the oracle's integers and the reference's strand bias within continuous_gen.SB_BOUND (both
checked against the body by tests/test_continuous.py); capacity, refusal and empty batches; and the DevWindow -> K2c route, with no host
step between the window pass and K2c, equals the host route on the bench's synthetic windows."""
import os
import sys

import numpy as np
import pytest

import continuous_gen as G
from strelka_b200 import _abi as A
from strelka_b200 import api
from strelka_b200 import batch as B

sys.path.insert(0, os.path.join(G.ROOT, "tools"))

pytestmark = pytest.mark.gpu

OPTS = [G.default_opts(), A.SxContOpts(0.2, 5.0, 10, 30)]


@pytest.fixture(scope="module")
def ctx():
    c = api.Context(0)
    yield c
    c.close()


def test_qscore_grid(ctx):
    g = np.load(G.GOLDEN)
    a, n = G.grid_pairs()
    gq, st = ctx.cont_qscore_dev(a, n)
    assert np.array_equal(gq, G.gq_from_thresholds(g["first"], a, n))
    assert not st.any(), "no tie flag on the grid"
    gq, st = ctx.cont_qscore(g["large_a"], g["large_n"])
    assert np.all(gq == 40) and not st.any()
    # other options: the host body's answers
    o = A.SxContOpts(0.01, 99.0, 10, 60)
    for f in (ctx.cont_qscore, ctx.cont_qscore_dev):
        assert [x.tobytes() for x in f(a[::97], n[::97], o)] == [x.tobytes() for x in G.core_qscore(a[::97], n[::97], o)]


@pytest.mark.parametrize("S", [1, 2, 3, 8])
@pytest.mark.parametrize("k", range(len(OPTS)))
def test_site_continuous_equals_body(ctx, S, k):
    b = G.case(100 * S + k, S)
    want = G.core_run(b, OPTS[k])
    G.same(ctx.site_continuous(b, OPTS[k]), want)
    G.same(ctx.site_continuous_dev(api.DevContBatch(ctx, b), OPTS[k]), want)


@pytest.mark.parametrize("S", [1, 3])
def test_deep_columns(ctx, S):
    b = G.case(7 + S, S, n_sites=300, kinds=("deep", "deep", "ordinary", "n_ref"))
    want = G.core_run(b, G.default_opts())
    G.same(ctx.site_continuous(b, G.default_opts()), want)
    G.same(ctx.site_continuous_dev(api.DevContBatch(ctx, b), G.default_opts()), want)
    # the same records run to run
    G.same(ctx.site_continuous(b, G.default_opts()), want)


def test_capacity_refusal_empty(ctx):
    b = G.case(5, 2)
    n = int(G.core_run(b, G.default_opts()).totals[0])
    with pytest.raises(api.SxError) as e:
        ctx.site_continuous(b, cap_loci=n - 1)
    assert e.value.code == A.SX_ERR_CAPACITY and int(e.value.totals[0]) == n
    with pytest.raises(api.SxError) as e:
        ctx.site_continuous_dev(api.DevContBatch(ctx, b), cap_loci=n - 1)
    assert e.value.code == A.SX_ERR_CAPACITY and int(e.value.totals[0]) == n
    for bad in (A.SxContOpts(0.5, 99.0, 17, 40), A.SxContOpts(0.0, 99.0, 17, 40), A.SxContOpts(0.01, -1.0, 17, 40), A.SxContOpts(0.01, 99.0, 71, 40),
                A.SxContOpts(0.01, 99.0, 17, -1)):
        with pytest.raises(api.SxError) as e:
            ctx.site_continuous(b, bad)
        assert e.value.code == A.SX_ERR_ARG
        with pytest.raises(api.SxError) as e:
            ctx.cont_qscore(np.ones(3), np.ones(3), bad)
        assert e.value.code == A.SX_ERR_ARG
    b.c.n_samples = 0
    with pytest.raises(api.SxError) as e:
        ctx.site_continuous(b)
    assert e.value.code == A.SX_ERR_ARG
    b.c.n_samples = 2
    b.c.sample[1].n_sites = b.n_sites - 1
    with pytest.raises(api.SxError) as e:
        ctx.site_continuous(b)
    assert e.value.code == A.SX_ERR_ARG
    empty = B.ContBatch([B.PileupBatch.from_sites([], "")])
    out = ctx.site_continuous(empty)
    assert int(out.totals[0]) == 0 and int(out.site_rec_off[0]) == 0
    assert ctx.cont_qscore(np.zeros(0), np.zeros(0))[0].size == 0


@pytest.mark.parametrize("cells,seed", [(200, 5), (400, 11)])
def test_window_route_equals_host_route(ctx, cells, seed):
    import window_workload as WW

    w = WW.make_window(WW.load_synth(), cells, seed)
    dws = [api.DevWindow(ctx, w), api.DevWindow(ctx, WW.make_window(WW.load_synth(), cells, seed))]
    for dw in dws:
        dw.run()
    got = ctx.site_continuous_dev(api.DevContBatch.from_windows(dws))
    ref = np.frombuffer(w.a["ref"].tobytes(), np.uint8)[w.report_begin - w.ref_begin: w.report_end - w.ref_begin]
    samples = []
    for dw in dws:
        d = dw.download()
        samples.append(B.PileupBatch(d["site_off"], d["calls"], ref))
    want = G.core_run(B.ContBatch(samples, w.report_begin), G.default_opts())
    assert int(want.totals[0]) > 0
    G.same(got, want)
    for dw in dws:
        dw.free()
