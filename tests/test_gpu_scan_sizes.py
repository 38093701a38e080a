"""The shared prefix sum (sx_scan.cu) at the lengths where its tiling changes: one element, a tile less one, one tile, a tile and one, and
one element past what the tile-sum pass covers in one round -- driven through stages that own a scan, against their oracles: K4 (eight
inclusive scans of difference arrays, then two exclusive scans into the CSR offsets; every output array) and K6b (one- and two-array
exclusive scans with closing entries).  The tile and the round are read out of the sources, so the lengths follow them."""
import os
import re

import numpy as np
import pytest

import indel_reads_gen as G
import reflib
import specgen
from strelka_b200 import batch as B

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "strelka_b200", "csrc")


def _scan_constants():
    """(T, C): elements per tile, and tile sums the carry pass scans per round."""
    with open(os.path.join(CSRC, "sx_internal.h")) as f:
        m = re.search(r"constexpr uint32_t SX_SCAN_TILE = (\d+), SX_SCAN_THREADS = (\d+);", f.read())
    with open(os.path.join(CSRC, "sx_scan.cu")) as f:
        assert "for (uint32_t b = 0; b < nt; b += SX_SCAN_THREADS)" in f.read()  # the carry pass's round is SX_SCAN_THREADS tile sums
    return int(m[1]), int(m[2])


T, C = _scan_constants()
SIZES = [1, T - 1, T, T + 1, C * T + 1]


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


# K4's arrays hold n_sites and n_sites + 1 words: together these put both lengths on every size above (the longer ones on all but 1)
@pytest.mark.parametrize("n_sites", sorted({1, T - 2, T - 1, T, T + 1, C * T, C * T + 1}))
def test_k4_scans_at_tile_boundaries(ctx, n_sites):
    rng = np.random.default_rng(8100 + n_sites % 997)
    ref_len = n_sites + 250
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=max(30, n_sites // 250), ref_len=ref_len)
    pb = B.PileupReadsBatch(reads, ref, ref_begin, ref_begin + 100, ref_begin + 100 + n_sites, cand)
    want = reflib.ox_pileup_reads(pb)
    got = ctx.pileup_reads(pb)
    assert want[0].size == n_sites + 1 and int(want[0][-1]) > 0
    for w, g, name in zip(want, got, ("site_off", "calls", "t2_off", "t2_calls", "n_spandel", "n_submapped")):
        assert np.array_equal(w, g), name


@pytest.mark.parametrize("n_loci", SIZES)
def test_k6b_scans_at_tile_boundaries(ctx, n_loci):
    """The pair offsets scan 2 * n_loci counts; the output scans read_off (2 * n_loci) and alt_off (n_loci) side by side."""
    normal, tumor, full = G.synthetic_case(60 + n_loci % 89, n_gid=n_loci + 8, n_regions=max(8, n_loci // 50), depth=4.0, locus_frac=1.0)
    m = n_loci
    loci = B.IndelLoci(full.gid[:m], full.key[:m], full.is_forced_output[:m], full.err_idx[:m], full.gid_key, full.err_prob)
    rc, want = G.ox_link(normal, tumor, loci)
    assert rc == 0 and loci.n_loci == n_loci and int(want.totals[0]) > 0
    G.same(want, ctx.link_indel_reads(normal, tumor, loci))
