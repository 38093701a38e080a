"""K4's fill pass on inputs that steer it down its less common routes, each against the oracle (itself pinned to the reference's
pileup_read_segment): reads whose realigned start moved by the full shift across a window edge, tier-2 reads among tier-1 reads, windows
of hundreds of reads among shallow ones, and windows whose cand_snv slice is larger than the part a warp holds in shared memory, in the
same launch as windows whose slice fits."""
import numpy as np
import pytest

import reflib
import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

pytestmark = pytest.mark.gpu

COLUMNS = ("site_off", "calls", "t2_off", "t2_calls", "n_spandel", "n_submapped")
SOMATIC = A.SxPileupOpts(1, 0, 20, 3, 1, 10, 0, 0)  # tier-2 evidence on: the tier-2 filters decide


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


def _check(ctx, pb):
    want = reflib.ox_pileup_reads(pb)
    got = ctx.pileup_reads(pb)
    assert int(want[0][-1]) > 1000
    for w, g, name in zip(want, got, COLUMNS):
        assert np.array_equal(w, g), name
    return want


def _shifted(rng, reads, shift, share):
    """buffer positions: a `share` of the reads moved by exactly +-shift from their best alignment's start, the batch re-sorted by it"""
    bpos = []
    for r in reads:
        u = rng.random()
        bpos.append(int(r.pos) + (shift if u < share / 2 else -shift if u < share else 0))
    order = np.argsort(np.asarray(bpos), kind="stable")
    return [reads[i] for i in order], [bpos[i] for i in order]


@pytest.mark.parametrize("shift", [17, 40, 64])
@pytest.mark.parametrize("seed", range(2))
def test_k4_full_shift_across_window_edges(ctx, seed, shift):
    """Every moved read is moved by the batch's whole max_pos_shift D, half of them forward and half back: the window width is the
    span + D rounded to 32, so reads near every window edge reach D into the neighbouring window on either side."""
    rng = np.random.default_rng(7000 + 10 * seed + shift)
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=int(rng.integers(900, 1600)), ref_len=int(rng.integers(1500, 3000)))
    reads, bpos = _shifted(rng, reads, shift, 0.6)
    pb = B.PileupReadsBatch(reads, ref, ref_begin, ref_begin + 100, ref_begin + len(ref) - 150, cand, SOMATIC, buffer_pos=bpos)
    assert pb.c.max_pos_shift == shift
    _check(ctx, pb)


@pytest.mark.parametrize("t2_share", [0.3, 0.7])
def test_k4_tier2_reads_among_tier1(ctx, t2_share):
    """tier-1 and tier-2 reads interleaved in one window: each tier's column keeps its own read order"""
    rng = np.random.default_rng(7100 + int(10 * t2_share))
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=1400, ref_len=2500)
    for r in reads:
        if r.tier in (1, 2):
            r.tier = 2 if rng.random() < t2_share else 1
    reads, bpos = _shifted(rng, reads, 25, 0.4)
    pb = B.PileupReadsBatch(reads, ref, ref_begin, ref_begin + 100, ref_begin + len(ref) - 150, cand, SOMATIC, buffer_pos=bpos)
    want = _check(ctx, pb)
    assert int(want[2][-1]) > 1000  # the tier-2 columns are not empty


@pytest.mark.parametrize("seed", range(2))
def test_k4_deep_windows_among_shallow_ones(ctx, seed):
    """a ~250x tier-1 pile over 250 positions amid ~15x coverage: the warps of the windows over the pile walk hundreds of reads, loading
    their records 32 at a time, in the same launch as warps that walk a handful"""
    rng = np.random.default_rng(7300 + seed)
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=6000, ref_len=1500)
    deep = (ref_begin + 600, ref_begin + 850)
    reads = [r for r in reads if deep[0] <= r.pos < deep[1] or rng.random() < 0.05]
    reads, bpos = _shifted(rng, reads, 30, 0.4)
    pb = B.PileupReadsBatch(reads, ref, ref_begin, ref_begin + 100, ref_begin + len(ref) - 150, cand, SOMATIC, buffer_pos=bpos)
    want = _check(ctx, pb)
    depth = np.diff(want[0].astype(np.int64))
    assert depth.max() > 200 and np.median(depth) < 40


@pytest.mark.parametrize("seed", range(2))
def test_k4_cand_snv_slice_over_the_shared_memory_cap(ctx, seed):
    """every (position, base) of a 400-position stretch is a candidate SNV: the windows over it have slices of over a thousand keys, past
    what a warp stages in shared memory, and search them in place; the windows elsewhere hold their few keys in shared memory"""
    rng = np.random.default_rng(7200 + seed)
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=1500, ref_len=3000, snv_rate=0.03)
    dense = [(ref_begin + p, b) for p in range(1200, 1600) for b in range(4)]
    cand = sorted(set(cand) | set(dense))
    reads, bpos = _shifted(rng, reads, 20, 0.4)
    pb = B.PileupReadsBatch(reads, ref, ref_begin, ref_begin + 100, ref_begin + len(ref) - 150, cand, buffer_pos=bpos)
    assert pb.c.n_cand_snv > 1600
    _check(ctx, pb)
    # the same reads with the sparse list alone give different columns: the dense keys do change which mismatches count
    sparse = B.PileupReadsBatch(reads, ref, ref_begin, ref_begin + 100, ref_begin + len(ref) - 150, [k for k in cand if k not in set(dense)], buffer_pos=bpos)
    assert not np.array_equal(reflib.ox_pileup_reads(sparse)[1], reflib.ox_pileup_reads(pb)[1])
