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

