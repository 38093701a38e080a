"""GPU: sx_process_window_dev -- the whole READ_BUFFER + POST_ALIGN pass of a window, device-resident -- against the reference run stage by
stage on the same window (tests/window_check.py): realignAndScoreRead, pileup_read_segment in read-buffer order, position_snp_call_pprob_digt.
Sorts last (it drives every kernel of the chain)."""
import numpy as np
import pytest

import reflib
import refgold
import window_check as W
from window_check import WW

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("block", range(20))
def test_window_equals_the_reference(ctx, block):
    """200 seeded batches (plain, clustered / conflicting, phased, dense windows, hard and soft clips, moved starts, over-long deletions,
    reads the gates turn away), each region a window: per read is_realigned / rseg.realignment segment for segment (hard clips included) and
    score_indels' records; per window the pile-up columns in read-buffer order and the germline site results -- against the reference where
    oracle/_ref is built, against its frozen digests elsewhere."""
    tot = {"reads": 0, "realigned": 0, "records": 0, "threw": 0, "calls": 0, "sites": 0}
    for case in range(10 * block, 10 * block + 10):
        for i, (eb1, gb1, flags, mapq) in enumerate(W.window_case(case)):
            s = W.check_window(ctx, eb1, gb1, f"{case}.{i}", read_flags=flags, mapq=mapq)
            for k in tot:
                tot[k] += s[k]
    assert tot["realigned"] > 0 and tot["records"] > 0 and tot["calls"] > 0, tot


@pytest.mark.parametrize("qual_bits,seed", [(4, 1), (8, 2), (4, 3)])
def test_synthetic_cfg2_window_equals_the_reference(ctx, qual_bits, seed):
    """bench.py's workload (tools/synth_window.cpp: a contig tiled by candidate loci at 30x, mapper-style alignments) through the one-call pass
    against the reference's realignAndScoreRead + pileup_read_segment + position_snp_call_pprob_digt on the same arrays: best alignments,
    score_indels records, columns (in read-buffer order across loci) and site results (or their frozen digests where oracle/_ref is not built)."""
    from strelka_b200.api import DevWindow

    w = WW.make_window(WW.load_synth(), 400, seed, tile=seed, qual_bits=qual_bits, ascii_reads=True)
    entry = refgold.golden()["synthetic"][f"{qual_bits}-{seed}"]
    assert entry["inputs"] == refgold.synthetic_inputs_digest(w), "the seeded inputs changed: regenerate tests/golden/window_ref_digests.json"
    dw = DevWindow(ctx, w)
    dw.run()
    d = dw.download()
    dw.run()  # a second pass over the same buffers (the region records were rewritten by the first)
    d2 = dw.download()
    dw.free()
    got = WW.window_items(w, d)
    refgold.compare(got, WW.reference_items(w, WW.reference_pass(w)[0]) if reflib.have_ref() else None, entry)
    stats = WW.window_stats(w, got)
    for k in d:
        assert np.asarray(d[k]).tobytes() == np.asarray(d2[k]).tobytes(), k
    assert stats["realigned"] > 5000 and stats["records"] > 10000 and stats["variant_sites"] > 50, stats


def test_regrouped_work_lists_change_no_output_byte(ctx, monkeypatch):
    """K7's active list and K6's list are regrouped by class before their kernels run (sx_regroup.cuh); which thread handles which read must not
    matter: the pass with the regrouping switched off (SX_K7_NO_CLASS_SORT / SX_K6_NO_CLASS_SORT, read at every call) gives the same bytes in
    every output array -- candidate-alignment CSR (through K9's best alignments and K6's records), columns, site results, variant records."""
    import os
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import window_workload as WW
    from strelka_b200.api import DevWindow

    w = WW.make_window(WW.load_synth(), 300, 11, tile=2, qual_bits=4, ascii_reads=True)
    dw = DevWindow(ctx, w)
    dw.run()
    d_on = dw.download()
    monkeypatch.setenv("SX_K7_NO_CLASS_SORT", "1")
    monkeypatch.setenv("SX_K6_NO_CLASS_SORT", "1")
    dw.run()
    d_off = dw.download()
    dw.free()
    assert set(d_on) == set(d_off) and len(d_on) > 5
    for k in d_on:
        assert np.asarray(d_on[k]).tobytes() == np.asarray(d_off[k]).tobytes(), k



def _keyless_window():
    """one region of 40 reads without a window entry (n_keys = 0): every fourth read has a single-base mismatch"""
    from strelka_b200 import batch as B

    rng = np.random.default_rng(5)
    ref = "".join(rng.choice(list("ACGT"), 700))
    rb = 10000
    reads, raw = [], []
    for i in range(40):
        pos = rb + 50 + 12 * i
        seq = list(ref[pos - rb : pos - rb + 100])
        if i % 4 == 0:
            seq[40] = "ACGT"[("ACGT".index(seq[40]) + 1) % 4]
        reads.append(B.EnumReadSpec("".join(seq), pos, [("M", 100)]))
        raw.append((pos, [("M", 100)]))
    eb = B.EnumBatch([(ref, rb, (rb, rb + 700), [], reads)])
    return B.WindowBatch.from_enum(eb, B.GateBatch(eb, raw), B.read_pools_of(eb))


def test_host_window_entry_takes_null_arrays(ctx):
    """sx_process_window (host arrays in and out) passes on what a caller may leave NULL: the key arrays of a window without window entries
    (n_keys = 0, key_ins_off / keys / key_ins / use_keys NULL) and the outputs it does not want.  Its outputs equal sx_process_window_dev's
    on the same window.  An empty window (no regions, no reads, every array NULL) runs and reports nothing."""
    import ctypes as C

    from strelka_b200 import _abi as A
    from strelka_b200 import batch as B
    from strelka_b200.api import DevWindow

    w = _keyless_window()
    assert w.n_keys == 0 and w.n_reads == 40
    dw = DevWindow(ctx, w)
    dw.run()
    d = dw.download()
    c = A.SxWindowBatch.from_buffer_copy(dw.c)
    host = {name: (None if w.a.get(name) is None or name in ("keys", "key_ins_off", "key_ins", "use_keys") else np.ascontiguousarray(w.a[name]))
            for name in B.WindowBatch.ARRAYS}
    for name, arr in host.items():
        setattr(c, name, None if arr is None else arr.ctypes.data)
    n, ns, cap = w.n_reads, w.n_sites, int(dw.out.cols.calls_capacity)
    h = {"gate": np.zeros(n, np.uint8), "best_pos": np.zeros(n, np.int32), "best_seg_off": np.zeros(n + 1, np.uint32), "best_n_seg": np.zeros(n, np.uint16),
         "best_segs": np.zeros(dw.cap_best, A.ALN_SEG_DT), "n_rec": np.zeros(n, np.uint32), "site_off": np.zeros(ns + 1, np.uint32), "t2_off": np.zeros(ns + 1, np.uint32),
         "n_spandel": np.zeros(ns, np.uint32), "n_submapped": np.zeros(ns, np.uint32), "calls": np.zeros(cap, np.uint16), "t2_calls": np.zeros(cap, np.uint16),
         "site_gl": np.zeros(ns, A.DIGT_RESULT_DT)}
    o = A.SxWindowOut()  # enum_status, realign_status, recs, totals and variant_sites stay NULL
    for k in ("gate", "best_pos", "best_seg_off", "best_n_seg", "best_segs", "n_rec", "site_gl"):
        setattr(o, k, h[k].ctypes.data)
    o.cap_best_segs = dw.cap_best
    o.cols = A.SxPileupColumns(h["site_off"].ctypes.data, h["calls"].ctypes.data, h["t2_off"].ctypes.data, h["t2_calls"].ctypes.data, h["n_spandel"].ctypes.data,
                               h["n_submapped"].ctypes.data, cap, cap)
    totals = np.zeros(A.SX_WIN_TOTALS, np.uint32)
    ctx._chk(ctx.lib.sx_process_window(ctx.h, C.byref(c), C.byref(o), totals.ctypes.data))
    dw.free()
    assert totals[6] > 0 and np.array_equal(totals[:8], d["totals"][:8]), (totals, d["totals"])
    h["best_segs"] = h["best_segs"][: int(h["best_seg_off"][n])]
    h["calls"], h["t2_calls"] = h["calls"][: int(totals[6])], h["t2_calls"][: int(totals[7])]
    for k, v in h.items():
        assert v.tobytes() == np.asarray(d[k]).tobytes(), k

    e = A.SxWindowBatch()
    ctx.lib.sx_default_window_opts(C.byref(e))
    e.ref_begin = e.report_begin = e.report_end = 1000
    site_off = np.full(1, 7, np.uint32)
    eo = A.SxWindowOut()
    eo.cols = A.SxPileupColumns(site_off.ctypes.data, None, None, None, None, None, 0, 0)
    totals[:] = 1
    ctx._chk(ctx.lib.sx_process_window(ctx.h, C.byref(e), C.byref(eo), totals.ctypes.data))
    assert not totals.any() and site_off[0] == 0, (totals, site_off)
