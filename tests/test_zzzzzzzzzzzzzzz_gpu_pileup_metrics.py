"""K4m (pile-up scoring metrics) on the GPU: sx_pileup_metrics[_dev] against the numpy host builder (batch.pileup_metrics, itself checked
against the g++-compiled k4m_core.cuh in tests/test_pileup_metrics.py) bit for bit -- seeded batches under every option set, the edge batch,
a site deeper than the reduce kernel's shared-memory tile, the rank-sum overflow status, full-read offsets --, argument errors, and the
window passes with metrics off (the existing entry, byte for byte) and on."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import pileup_metrics_gen as G
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import somatic_window_leg as SW  # noqa: E402
import window_workload as WW  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


def same_bits(a, b):
    return a.tobytes() == b.tobytes()


@pytest.mark.parametrize("mode", G.MODES)
@pytest.mark.parametrize("name", sorted(G.OPTION_SETS))
def test_random_batches(ctx, name, mode):
    for seed in (1, 2):
        pb = G.random_batch(seed, G.OPTION_SETS[name], qual_dict=seed == 2)
        want = B.pileup_metrics(pb, mode)
        assert same_bits(ctx.pileup_metrics(pb, mode), want)
        assert same_bits(ctx.pileup_metrics_dev(pb, mode), want)


@pytest.mark.parametrize("mode", G.MODES)
def test_edge_batch_and_full_reads(ctx, mode):
    pb = G.edge_batch()
    assert same_bits(ctx.pileup_metrics_dev(pb, mode), B.pileup_metrics(pb, mode))
    pb = G.random_batch(3, n_reads=200)
    fl, fo = G.full_read_arrays(pb, 3)
    assert same_bits(ctx.pileup_metrics(pb, mode, fl, fo), B.pileup_metrics(pb, mode, fl, fo))


def test_reference_goldens(ctx):
    """both entries equal the reference's own pileup_read_segment with the metrics on (tests/golden/pileup_metrics_ref.npz, frozen from
    oracle/ref_harness_pileup_metrics.cpp; the live harness where oracle/_ref is built)"""
    gold = G.golden()
    for key, pb, mode in G.golden_cases():
        got = ctx.pileup_metrics_dev(pb, mode)
        assert same_bits(got, gold[key]), key
        assert same_bits(ctx.pileup_metrics(pb, mode), gold[key]), key
        if G.have_ref():
            assert same_bits(G.ref_metrics(pb, mode), got), key


def test_sizes_across_scan_tiles(ctx):
    """more sites than one scan tile (4096) and many reads"""
    pb = G.random_batch(5, n_reads=4000, ref_len=12000)
    assert pb.n_sites > 2 * 4096
    for mode in G.MODES:
        assert same_bits(ctx.pileup_metrics_dev(pb, mode), B.pileup_metrics(pb, mode))


@pytest.mark.parametrize("mode", G.MODES)
def test_deep_site(ctx, mode):
    pb = G.deep_batch(5000)
    want = B.pileup_metrics(pb, mode)
    assert want["mapq_count"].max() > 4000
    got = ctx.pileup_metrics_dev(pb, mode)
    assert same_bits(got, want)
    assert same_bits(ctx.pileup_metrics_dev(pb, mode), got)  # two runs


def test_overflow_status(ctx):
    pb = G.overflow_batch()
    got = ctx.pileup_metrics_dev(pb, A.SX_PM_GERMLINE)
    assert got["status"][5] & A.SX_PM_ST_MQ_OVERFLOW and got["mq_ranksum"][5] == 0.0
    assert same_bits(got, B.pileup_metrics(pb, A.SX_PM_GERMLINE))


def test_bad_mode(ctx):
    from strelka_b200.api import SxError

    pb = G.random_batch(1, n_reads=20)
    for mode in (0, 4):
        with pytest.raises(SxError) as e:
            ctx.pileup_metrics(pb, mode)
        assert e.value.code == A.SX_ERR_ARG
        with pytest.raises(SxError) as e:
            ctx.pileup_metrics_dev(pb, mode)
        assert e.value.code == A.SX_ERR_ARG


@pytest.fixture(scope="module")
def window():
    return WW.make_window(WW.load_synth(), 400, 11)


def test_window_metrics(ctx, window):
    """sx_process_window_metrics_dev: NULL metrics is the existing entry (bytes and launches); with metrics the other outputs are unchanged,
    every base of the columns is counted, and two runs agree"""
    from strelka_b200.api import DevWindow

    plain = DevWindow(ctx, window)
    plain.run()
    l0 = ctx.timing().launches
    want = plain.download()
    null = DevWindow(ctx, window)
    ctx._chk(ctx.lib.sx_process_window_metrics_dev(ctx.h, C.byref(null.c), C.byref(null.out), null.totals.ctypes.data, None, None))
    assert ctx.timing().launches == l0
    got = null.download()
    assert all(np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes() for k in want)
    for mode in G.MODES:
        dw = DevWindow(ctx, window, metrics=mode)
        st = dw.run()
        assert "k4m_metrics" in st and ctx.timing().launches > l0
        out = dw.download()
        assert all(np.asarray(out[k]).tobytes() == np.asarray(want[k]).tobytes() for k in want)
        m = dw.metrics()
        # the pass's own pile-up batch, rebuilt on the host: the standalone entry (and the reference, where oracle/_ref is built) on it
        pb = G.window_pileup_batch(window, out, int(dw.c.enum_opts.max_indel_size))
        assert same_bits(ctx.pileup_metrics_dev(pb, mode), m)
        if G.have_ref():
            assert same_bits(G.ref_metrics(pb, mode), m)
        depth = np.diff(out["site_off"].astype(np.int64)) + np.diff(out["t2_off"].astype(np.int64))
        assert (m["mapq_count"] >= depth).all() and (m["mapq_count"] <= depth + out["n_submapped"]).all() and depth.sum() > 0
        dw.run()
        assert same_bits(dw.metrics(), m)
        if mode == A.SX_PM_GERMLINE:
            assert (m["read_pos_ranksum"] != 0).any() and (m["mean_edge_distance"] != 0).any()
        dw.free()
    plain.free()
    null.free()


def test_small_window_metrics_builder(ctx):
    """a small window: the pass's metrics equal the numpy host builder on the rebuilt pile-up batch, in every mode"""
    from strelka_b200.api import DevWindow

    w = WW.make_window(WW.load_synth(), 30, 5)
    for mode in G.MODES:
        dw = DevWindow(ctx, w, metrics=mode)
        dw.run()
        pb = G.window_pileup_batch(w, dw.download(), int(dw.c.enum_opts.max_indel_size))
        m = dw.metrics()
        dw.free()
        assert same_bits(B.pileup_metrics(pb, mode), m)
        assert m["mapq_count"].sum() > 0


def test_somatic_window_metrics(ctx, window):
    """sx_process_somatic_window_metrics_dev (normal SX_PM_MAPQ, tumor SX_PM_SOMATIC): its records equal sx_process_somatic_window_dev's, and
    each sample's metrics equal the germline window pass's on that sample alone"""
    from strelka_b200.api import DevSomaticWindow, DevWindow

    normal, tumor, loci, key_gid, forced = SW.two_sample_window(window, 11)
    o = A.default_sindel_opts()
    o.useTier2Evidence = 0
    plain = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced, opts=o)
    plain.run()
    want = plain.download()
    plain.free()
    sw = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced, opts=o, metrics=True)
    st = sw.run()
    assert "k4m_metrics" in st
    got = sw.download()
    for k in ("snv_calls", "indel_calls", "totals", "site_snv", "indel"):
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), k
    mn, mt = sw.metrics()
    for w, mode, m, part, dwin in ((normal, A.SX_PM_MAPQ, mn, "normal", sw.normal), (tumor, A.SX_PM_SOMATIC, mt, "tumor", sw.tumor)):
        pb = G.window_pileup_batch(w, got[part], int(dwin.c.enum_opts.max_indel_size))
        assert same_bits(ctx.pileup_metrics_dev(pb, mode), m)
        if G.have_ref():
            assert same_bits(G.ref_metrics(pb, mode), m)
    sw.free()
    assert (mt["n_alt_read_pos"] > 0).any() and (mn["mapq_count"] > 0).any()
    for w, mode, m in ((normal, A.SX_PM_MAPQ, mn), (tumor, A.SX_PM_SOMATIC, mt)):
        dw = DevWindow(ctx, w, metrics=mode)
        dw.run()
        assert same_bits(dw.metrics(), m)
        dw.free()
