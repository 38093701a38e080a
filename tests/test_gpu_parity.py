"""GPU parity: the CUDA path (through the C ABI) against oracle/liboracle.so on the same seeded inputs.
Bit-exact for every integer field and for the float/double likelihood sums the reference accumulates sequentially."""
import numpy as np
import pytest

import reflib
import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


@pytest.mark.parametrize("seed", range(6))
def test_k1_score_alignments_random_regions(ctx, seed):
    rng = np.random.default_rng(1000 + seed)
    regions = [specgen.random_region(rng, n_reads=int(rng.integers(1, 12))) for _ in range(40)]
    regions += [specgen.simple_region(rng, n_reads=int(rng.integers(5, 40))) for _ in range(10)]
    batch = B.build_align_batch(regions)
    want = reflib.ox_score(batch)
    got = ctx.score_alignments(batch)
    assert np.array_equal(_bits(got), _bits(want))
    t = ctx.timing()
    assert t.launches >= 1


def test_k1_device_resident_and_read_max(ctx):
    from strelka_b200.api import DevAlignBatch, DeviceArray

    rng = np.random.default_rng(5)
    regions = [specgen.simple_region(rng, n_reads=30) for _ in range(300)]
    batch = B.build_align_batch(regions)
    want = reflib.ox_score(batch)
    db = DevAlignBatch(ctx, batch)
    ctx.score_alignments_dev(db)
    got = db.out.download(np.float64, batch.n_alns)
    assert np.array_equal(_bits(got), _bits(want))
    mx = DeviceArray(ctx, batch.n_reads * 8)
    ma = DeviceArray(ctx, batch.n_reads * 4)
    ctx.read_max_dev(db, mx, ma)
    mlnp = mx.download(np.float64, batch.n_reads)
    maln = ma.download(np.uint32, batch.n_reads)
    reads = batch.alns["read"][:-1]
    for r in range(0, batch.n_reads, 97):
        idx = np.nonzero(reads == r)[0]
        assert mlnp[r] == want[idx].max()
        assert maln[r] == idx[np.argmax(want[idx])]


@pytest.mark.parametrize("qb,compact", [(8, True), (4, True), (2, False), (2, True)])
def test_k1_compact_wire_formats(ctx, qb, compact):
    """sx_aln8 / sx_aln_seg2 / 2-bit qualities: same doubles as the wide batch through the host entry (chunked copies), the device
    entry, and the per-read max epilogue; both kernels (a region too large for the fast path is in the batch)."""
    from strelka_b200.api import DevAlignBatch, DeviceArray

    rng = np.random.default_rng(41)
    regions = [specgen.random_region(rng, n_reads=int(rng.integers(1, 10))) for _ in range(40)]
    r_out = B.RegionSpec(
        "ACGTACGTAC", 100, [(B.codes_of("ACGTACGTACGT"), np.full(12, 37, np.uint8))],
        [B.CandidateAlignmentSpec(0, 95, [("M", 12)]), B.CandidateAlignmentSpec(0, 105, [("M", 12)]), B.CandidateAlignmentSpec(0, 5000, [("M", 12)]),
         B.CandidateAlignmentSpec(0, 100, [("S", 12)]), B.CandidateAlignmentSpec(0, 100, [("H", 5), ("S", 3), ("M", 9)])],
    )
    regions.append(r_out)
    regions.append(B.RegionSpec("ACGT" * 10, 100, [(B.codes_of("ACGT"), np.full(4, 37, np.uint8))], []))  # no alignments
    for r in regions:  # <= 4 distinct qualities so that the 2-bit format applies
        r.reads = [(codes, np.array([11, 25, 37, 2], np.uint8)[np.asarray(q) % 4]) for codes, q in r.reads]
    regions += [specgen.simple_region(rng, n_reads=int(rng.integers(3, 40))) for _ in range(30)]
    small = list(regions)
    for with_large in (False, True):
        regs = small + ([specgen.simple_region(rng, n_reads=330)] if with_large else [])
        wide = B.build_align_batch(regs)
        want = reflib.ox_score(wide)
        cb = B.build_align_batch(regs, qual_bits=qb, compact=compact)
        assert cb.fmt == (0 if not compact else 15 if qb == 2 else 11)  # ALN8 | SEG2 | REF4 (| BASEQ with the 2-bit dictionary)
        assert np.array_equal(_bits(ctx.score_alignments(cb)), _bits(want))
        if not with_large:
            # the chunk-pipelined host entry with chunk borders at arbitrary (odd) alignment indices
            from strelka_b200.api import Context

            p = A.default_params()
            p.pipeline_chunks = 7
            c7 = Context(0, p)
            assert np.array_equal(_bits(c7.score_alignments(cb)), _bits(want))
            c7.close()
        db = DevAlignBatch(ctx, cb)
        ctx.score_alignments_dev(db)
        assert np.array_equal(_bits(db.out.download(np.float64, cb.n_alns)), _bits(want))
        mx = DeviceArray(ctx, cb.n_reads * 8)
        ma = DeviceArray(ctx, cb.n_reads * 4)
        ctx.read_max_dev(db, mx, ma)
        mlnp = mx.download(np.float64, cb.n_reads)
        maln = ma.download(np.uint32, cb.n_reads)
        reads = wide.alns["read"][:-1]
        for r in range(0, cb.n_reads, 7):
            idx = np.nonzero(reads == r)[0]
            if idx.size == 0:
                assert maln[r] == 0xFFFFFFFF
            else:
                assert mlnp[r] == want[idx].max() and maln[r] == idx[np.argmax(want[idx])]


def test_k1_edge_cases(ctx):
    rng = np.random.default_rng(9)
    # a region without alignments, a region with one 1-base read, alignments far outside the held reference window
    r_empty = B.RegionSpec("ACGT" * 10, 100, [(B.codes_of("ACGT"), np.full(4, 30, np.uint8))], [])
    r_one = B.RegionSpec("ACGT" * 10, 100, [(B.codes_of("A"), np.array([40], np.uint8))], [B.CandidateAlignmentSpec(0, 100, [("M", 1)])])
    r_out = B.RegionSpec(
        "ACGTACGTAC", 100, [(B.codes_of("ACGTACGTACGT"), np.full(12, 37, np.uint8))],
        [B.CandidateAlignmentSpec(0, 95, [("M", 12)]), B.CandidateAlignmentSpec(0, 105, [("M", 12)]), B.CandidateAlignmentSpec(0, 5000, [("M", 12)]),
         B.CandidateAlignmentSpec(0, 100, [("S", 12)]), B.CandidateAlignmentSpec(0, 100, [("H", 5), ("S", 3), ("M", 9)])],
    )
    batch = B.build_align_batch([r_empty, r_one, r_out, specgen.random_region(rng)])
    want = reflib.ox_score(batch)
    got = ctx.score_alignments(batch)
    assert np.array_equal(_bits(got), _bits(want))
    # empty batch is a no-op
    empty = B.build_align_batch([])
    assert ctx.score_alignments(empty).size == 0


def test_k1_rejects_bad_input(ctx):
    from strelka_b200.api import SxError

    rng = np.random.default_rng(3)
    batch = B.build_align_batch([specgen.simple_region(rng, n_reads=4)])
    batch.qual[3] = 99  # qphred_cache::qscore_check throws above 70
    with pytest.raises(SxError) as e:
        ctx.score_alignments(batch)
    assert e.value.code == A.SX_ERR_RANGE
    batch = B.build_align_batch([specgen.simple_region(rng, n_reads=4), specgen.simple_region(rng, n_reads=4)])
    batch.regions["qual_off"][1] += 1
    with pytest.raises(SxError) as e:
        ctx.score_alignments(batch)
    assert e.value.code == A.SX_ERR_ALIGNMENT


def test_k1_four_bit_rejects_bad_quality_codes(ctx):
    """4-bit wire format: a dictionary quality above 70 used on a real base is a range error; the same quality on an N base is
    ignored, as the reference ignores it (score.cpp:125-126)."""
    from strelka_b200.api import SxError

    rng = np.random.default_rng(31)
    region = specgen.simple_region(rng, n_reads=6)
    batch = B.build_align_batch([region], qual_bits=4)
    want = ctx.score_alignments(batch)
    free = int(np.max(np.asarray(batch.qual[: batch.used["qual"]]) >> 4)) + 1  # first unused dictionary code
    assert free < 15
    # base 0 of read 0: quality code in the high nibble of byte 0
    keep = batch.qual[0]
    batch.c.qual_dict[free] = 99
    batch.qual[0] = (free << 4) | (keep & 15)
    with pytest.raises(SxError) as e:
        ctx.score_alignments(batch)
    assert e.value.code == A.SX_ERR_RANGE
    # ... but not when that base is an N: the read nibble 15 is skipped before its quality is looked at
    batch.qual[0] = (free << 4) | (keep & 15)
    seq0 = batch.seq4[0]
    batch.seq4[0] = (15 << 4) | (seq0 & 15)
    got = ctx.score_alignments(batch)
    assert got.shape == want.shape and np.all(np.isfinite(got))


def test_k1_four_bit_large_region_uses_general_kernel(ctx):
    """A region too large for the byte-entry kernel's 16-bit shared addresses is scored by the general kernel: same doubles."""
    rng = np.random.default_rng(32)
    regions = [specgen.simple_region(rng, n_reads=330), specgen.simple_region(rng, n_reads=5)]
    b4 = B.build_align_batch(regions, qual_bits=4)
    b8 = B.build_align_batch(regions, qual_bits=8)
    want = reflib.ox_score(b8)
    assert np.array_equal(_bits(ctx.score_alignments(b4)), _bits(want))


def _ga_scores(match, mismatch, open_, extend, off_edge, ins_del=0, allow_edge_ins=False, require_edge_del=False):
    return A.SxGaScores(match, mismatch, open_, extend, off_edge, ins_del, int(allow_edge_ins), int(require_edge_del))


@pytest.mark.parametrize("flags", [(False, False), (True, False), (False, True), (True, True)])
def test_k3_global_align_random(ctx, flags):
    rng = np.random.default_rng(77)
    qs, rs = specgen.random_ga_problems(rng, 400, n_frac=0.01)
    qs += ["A", "ACGT", "A" * 300, specgen.rand_seq(rng, 257)]
    rs += ["A", "T", "A" * 280, specgen.rand_seq(rng, 300)]
    gb = B.GaBatch(qs, rs, max_ops=700)
    for sc in (_ga_scores(1, -4, -5, -1, -100, -5, *flags), _ga_scores(2, -4, -5, -1, -1, 0, *flags)):
        o_res, o_cig = reflib.ox_global_align(sc, gb)
        g_res, g_cig = ctx.global_align(sc, gb)
        assert np.array_equal(o_res, g_res)
        assert np.array_equal(o_cig, g_cig)


@pytest.mark.parametrize("max_ops", [1, 2, 3, 5])
def test_k3_cigar_overflow_keeps_the_first_ops(ctx, max_ops):
    """More CIGAR operations than the caller's max_ops: status 1, n_ops = the true count, and the first max_ops operations are
    stored (both kernels: the group kernel builds the CIGAR backwards in a ring and must un-rotate it)."""
    rng = np.random.default_rng(78)
    qs, rs = specgen.random_ga_problems(rng, 300, n_frac=0.01)
    qs += ["A" * 300, specgen.rand_seq(rng, 257)]
    rs += ["A" * 280, specgen.rand_seq(rng, 300)]
    gb = B.GaBatch(qs, rs, max_ops=max_ops)
    sc = _ga_scores(1, -4, -5, -1, -100, -5, True, False)
    o_res, o_cig = reflib.ox_global_align(sc, gb)
    g_res, g_cig = ctx.global_align(sc, gb)
    assert (o_res["status"] == 1).any() and (o_res["status"] == 0).any() or max_ops == 1
    assert np.array_equal(o_res, g_res)
    assert np.array_equal(o_cig, g_cig)


def test_k3_reference_unit_test_goldens(ctx):
    import json
    import os

    gold = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "global_aligner_goldens.json")))
    for case in gold["cases"]:
        sc = _ga_scores(*case["scores"])
        gb = B.GaBatch([case["query"]], [case["ref"]], max_ops=64)
        res, cig = ctx.global_align(sc, gb)
        assert B.cigar_string(cig[0, : res["n_ops"][0]]) == case["cigar"], case["name"]
        assert int(res["beginPos"][0]) == case["beginPos"], case["name"]
        if "score" in case:
            assert int(res["score"][0]) == case["score"], case["name"]


def _same_germline(want, got):
    """every field of two sx_digt_result arrays: equal integers, the same bits for the floats and doubles"""
    for f in ("ref_gt", "is_computed", "n_used_calls", "phredLoghood"):
        assert np.array_equal(want[f], got[f]), f
    assert np.array_equal(_bits(want["lhood"]), _bits(got["lhood"]))
    assert np.array_equal(_bits(want["strand_bias"]), _bits(got["strand_bias"]))
    for rs in ("genome", "poly"):
        for f in ("max_gt", "snp_qphred", "max_gt_qphred"):
            assert np.array_equal(want[rs][f], got[rs][f]), (rs, f)
        assert np.array_equal(_bits(got[rs]["ref_pprob"]), _bits(want[rs]["ref_pprob"])), (rs, "ref_pprob")  # exp / log10 are the libm mirrors (sx_libm_mirror_d.h)


@pytest.mark.parametrize("seed,depth", [(0, 8.0), (1, 30.0), (2, 60.0), (3, 150.0)])
@pytest.mark.parametrize("always", [True, False])
def test_k2a_site_gl_germline(ctx, seed, depth, always):
    rng = np.random.default_rng(2000 + seed)
    pb = specgen.random_pileups(rng, 2000, depth=depth)
    p = A.default_params()
    _same_germline(reflib.ox_germline(p, pb, always), ctx.site_gl_germline(pb, always))
    o_off, o_de = reflib.ox_dependent_eprob(p, pb)
    g_off, g_de = ctx.dependent_eprob(pb)
    assert np.array_equal(o_off, g_off)
    assert np.array_equal(_bits(o_de), _bits(g_de))


@pytest.mark.parametrize("seed,depth", [(0, 50.0), (1, 20.0), (2, 33.0)])
def test_k2a_twelve_sites_per_warp(ctx, seed, depth):
    """the twelve-sites-per-warp kernel (every site <= 96 cleaned calls: one-ballot grouping up to 32 calls, chunked beyond; compacted
    (site, group) pairs; three sites per posterior block; strand sums for SNP sites only) on batches that exercise both grouping paths,
    haploid sites and is_always_test = False: every field against the oracle, bit for bit where the reference is float."""
    rng = np.random.default_rng(2100 + seed)
    pb0 = specgen.random_pileups(rng, 6000, depth=depth, max_depth=96)
    assert int(np.diff(pb0.site_off.astype(np.int64)).max()) <= 96 and int(np.diff(pb0.site_off.astype(np.int64)).max()) > (32 if depth > 25 else 0)
    pl = np.where(rng.random(pb0.n_sites) < 0.1, 1, 2).astype(np.uint8)
    pb = B.PileupBatch(pb0.site_off, pb0.calls, pb0.ref_base, pl)
    p = A.default_params()
    for always in (True, False):
        want = reflib.ox_germline(p, pb, always)
        got = ctx.site_gl_germline(pb, always)
        for f in ("ref_gt", "is_computed", "n_used_calls", "phredLoghood"):
            assert np.array_equal(want[f], got[f]), f
        assert np.array_equal(_bits(want["lhood"]), _bits(got["lhood"]))
        assert np.array_equal(_bits(want["strand_bias"]), _bits(got["strand_bias"]))
        assert int((want["strand_bias"] != 0).sum()) > 20
        for rs in ("genome", "poly"):
            for f in ("max_gt", "snp_qphred", "max_gt_qphred"):
                assert np.array_equal(want[rs][f], got[rs][f]), (rs, f)
            assert np.array_equal(_bits(got[rs]["ref_pprob"]), _bits(want[rs]["ref_pprob"])), (rs, "ref_pprob")  # exp / log10 are the libm mirrors (sx_libm_mirror_d.h)


def test_k2a_deep_and_empty_sites(ctx):
    rng = np.random.default_rng(31)
    deep = specgen.random_pileups(rng, 40, depth=900.0, max_depth=3000)  # beyond the shared-memory tile: global scratch path
    p = A.default_params()
    want = reflib.ox_germline(p, deep, True)
    got = ctx.site_gl_germline(deep, True)
    assert np.array_equal(want["phredLoghood"], got["phredLoghood"])
    assert np.array_equal(_bits(want["lhood"]), _bits(got["lhood"]))
    empty = B.PileupBatch.from_sites([[], [], [int(B.pack_call(30, 1, 1))]], "ANC")
    want = reflib.ox_germline(p, empty, True)
    got = ctx.site_gl_germline(empty, True)
    assert want.tobytes() == got.tobytes()
    # sites of <= 256 calls interleaved with sites of 257-3000 calls, more sites than the launch has warps: one launch (and one warp,
    # site after site) takes sites in its shared-memory tile and in its global-scratch region
    parts = [specgen.random_pileups(rng, 4400, depth=60.0), specgen.random_pileups(rng, 20, depth=250.0, max_depth=256),
             specgen.random_pileups(rng, 20, depth=300.0, max_depth=3000), specgen.random_pileups(rng, 20, depth=2000.0, max_depth=3000)]
    sites = [(pb.calls[pb.site_off[i]:pb.site_off[i + 1]].tolist(), chr(pb.ref_base[i])) for pb in parts for i in range(pb.n_sites)]
    sites += [([], "A"), ([], "C"), ([], "T")]
    sites = [sites[i] for i in rng.permutation(len(sites))]
    n_ref = next(i for i, (c, r) in enumerate(sites) if len(c) > 256 and r != "N")
    sites[n_ref] = (sites[n_ref][0], "N")
    ploidy = np.where(rng.random(len(sites)) < 0.1, 1, 2).astype(np.uint8)
    mixed = B.PileupBatch.from_sites([c for c, _ in sites], "".join(r for _, r in sites), ploidy)
    depth = np.diff(mixed.site_off.astype(np.int64))
    assert len(sites) % 16 != 0 and (depth == 0).sum() >= 3 and (depth > 256).sum() > 30 and depth.max() <= 3000
    assert np.count_nonzero(np.diff((depth > 256).astype(np.int8))) > 30  # interleaved
    from strelka_b200.api import Context

    p2 = A.SxParams(0.001, 0.0, 0.0, 0, 1, 0.0, 0.0, 1e-4, 5e-10, 0.0, 0.15, 0, 0)  # no dependent error model
    c2 = Context(0, p2)
    try:
        for params, c in ((p, ctx), (p2, c2)):
            for always in (True, False):
                _same_germline(reflib.ox_germline(params, mixed, always), c.site_gl_germline(mixed, always))
            o_off, o_de = reflib.ox_dependent_eprob(params, mixed)
            g_off, g_de = c.dependent_eprob(mixed)
            assert np.array_equal(o_off, g_off)
            assert np.array_equal(_bits(o_de), _bits(g_de))
    finally:
        c2.close()


def test_k2a_haploid_and_no_dependency(ctx):
    from strelka_b200.api import Context

    rng = np.random.default_rng(8)
    pb0 = specgen.random_pileups(rng, 1000, depth=25.0)
    pl = rng.integers(1, 3, pb0.n_sites).astype(np.uint8)
    pb = B.PileupBatch(pb0.site_off, pb0.calls, pb0.ref_base, pl)
    want = reflib.ox_germline(A.default_params(), pb, True)
    got = ctx.site_gl_germline(pb, True)
    assert np.array_equal(want["phredLoghood"], got["phredLoghood"])
    assert np.array_equal(_bits(want["lhood"]), _bits(got["lhood"]))
    p2 = A.SxParams(0.001, 0.0, 0.0, 0, 1, 0.0, 0.0, 1e-4, 5e-10, 0.0, 0.15, 0, 0)
    c2 = Context(0, p2)
    want = reflib.ox_germline(p2, pb, True)
    got = c2.site_gl_germline(pb, True)
    c2.close()
    assert np.array_equal(want["phredLoghood"], got["phredLoghood"])
    assert np.array_equal(_bits(want["lhood"]), _bits(got["lhood"]))


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("tier2", [False, True])
def test_k2b_site_gl_somatic(ctx, seed, tier2):
    rng = np.random.default_rng(3000 + seed)
    n = 2000
    npb = specgen.random_pileups(rng, n, depth=30.0, with_tier2=tier2, alt_frac_choices=(0.0, 0.0, 0.0, 0.0, 0.02, 0.5))
    tpb0 = specgen.random_pileups(rng, n, depth=60.0, with_tier2=tier2, alt_frac_choices=(0.0, 0.0, 0.05, 0.1, 0.2, 0.4))
    tpb = B.PileupBatch(tpb0.site_off, tpb0.calls, npb.ref_base, None, tpb0.t2_off, tpb0.t2_calls)
    forced = (rng.random(n) < 0.2).astype(np.uint8)
    p = A.default_params()
    want = reflib.ox_somatic(p, npb, tpb, forced)
    got = ctx.site_gl_somatic(npb, tpb, forced)
    assert np.array_equal(want["is_computed"], got["is_computed"])
    m = want["is_computed"] == 1
    assert m.sum() > 50
    for f in ("ref_gt", "snv_tier", "snv_from_ntype_tier", "ntype", "max_gt", "qphred", "from_ntype_qphred", "normal_alt_id", "tumor_alt_id"):
        assert np.array_equal(want[f][m], got[f][m]), f
    # the 21 grid likelihoods are float sums of table values: bit-exact
    assert np.array_equal(_bits(want["normal_lhood"][m][:, :21]), _bits(got["normal_lhood"][m][:, :21]))
    assert np.array_equal(_bits(want["tumor_lhood"][m][:, :21]), _bits(got["tumor_lhood"][m][:, :21]))
    # strand states end in a float log-sum through glibc's expf / log1p / logf: the device runs restatements of exactly those (sx_libm_mirror*.h)
    assert np.array_equal(_bits(got["tumor_lhood"][m][:, 21:30]), _bits(want["tumor_lhood"][m][:, 21:30]))
    assert np.array_equal(_bits(got["strandBias"][m]), _bits(want["strandBias"][m]))


def test_libm_mirrors_on_device(ctx):
    """de (powf mirror) and lhood (logf mirror) bit-equality above already exercise the mirrors; this adds a dense sweep of
    dependency exponents by driving single-group pileups with controlled neighbour-mismatch fractions."""
    rng = np.random.default_rng(123)
    sites = []
    for _ in range(3000):
        n = int(rng.integers(1, 40))
        q = rng.integers(3, 64, n)
        nbr = rng.random(n) < rng.random()
        sites.append(list(B.pack_call(q, 0, 1, nbr, 0, 0)))
    pb = B.PileupBatch.from_sites(sites, "A" * len(sites))
    p = A.default_params()
    o_off, o_de = reflib.ox_dependent_eprob(p, pb)
    g_off, g_de = ctx.dependent_eprob(pb)
    assert np.array_equal(_bits(o_de), _bits(g_de))


def test_cpp_host_mirror(tmp_path):
    """The C++ host mirror (strelka_b200/host/strelka_b200.hh, the layer a reference developer programs against): the reference's
    22 GlobalAligner goldens and reference-frozen scoreCandidateAlignment values, through sx::GlobalAligner<int>::align and
    sx::ReadAlignBatch::scoreCandidateAlignments."""
    import os
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = str(tmp_path / "test_host_mirror")
    lib = os.path.join(root, "strelka_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I" + os.path.join(root, "include"), "-I" + os.path.join(root, "strelka_b200", "host"),
                           os.path.join(root, "tests", "cpp", "test_host_mirror.cpp"), "-o", exe, "-L" + lib, "-lstrelka_b200", "-Wl,-rpath," + lib])
    out = subprocess.run([exe, os.path.join(root, "tests", "golden")], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "0 failures" in out.stdout


@pytest.mark.parametrize("seed", range(3))
def test_k5_indel_gl(ctx, seed):
    rng = np.random.default_rng(5000 + seed)
    ib = B.IndelBatch(specgen.random_indel_loci(rng, 1500))
    p = A.default_params()
    want = reflib.ox_indel_gl(p, ib)
    got = ctx.indel_gl(ib)
    assert np.array_equal(want["n_gt"], got["n_gt"])
    assert np.array_equal(want["support"], got["support"])
    assert np.array_equal(_bits(got["gt_lhood"]), _bits(want["gt_lhood"]))  # log / log1p / exp are the libm mirrors (sx_libm_mirror_d.h)


@pytest.mark.parametrize("seed", range(3))
def test_k1_four_bit_quality_wire_format(ctx, seed):
    """qual_bits=4 (dictionary-coded qualities, two per byte) is lossless: same doubles as the 8-bit format and as the oracle."""
    rng = np.random.default_rng(7000 + seed)
    regions = [specgen.random_region(rng, n_reads=int(rng.integers(1, 12))) for _ in range(30)]
    regions += [specgen.simple_region(rng, n_reads=int(rng.integers(5, 40))) for _ in range(10)]
    b8 = B.build_align_batch(regions, qual_bits=8)
    b4 = B.build_align_batch(regions, qual_bits=4)
    assert b4.used["qual"] < b8.used["qual"]
    want = reflib.ox_score(b8)
    assert np.array_equal(_bits(reflib.ox_score(b4)), _bits(want))
    assert np.array_equal(_bits(ctx.score_alignments(b4)), _bits(want))
    assert np.array_equal(_bits(ctx.score_alignments(b8)), _bits(want))


@pytest.mark.parametrize("mode", ["germline", "somatic", "nofilter", "edge"])
@pytest.mark.parametrize("seed", range(3))
def test_k4_pileup_reads(ctx, seed, mode):
    """K4 (SURVEY 8f1): the per-position tier1/tier2 base_call columns, in pile-up order, and the spanning-deletion / sub-mapped counts,
    against the oracle (itself pinned to the reference's pileup_read_segment)."""
    rng = np.random.default_rng(6000 + seed)
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=int(rng.integers(300, 1500)), ref_len=int(rng.integers(700, 4000)))
    opts = A.default_pileup_opts()
    if mode == "somatic":
        opts = A.SxPileupOpts(1, 0, 20, 3, 1, 10, 0, 0)
    elif mode == "nofilter":
        opts = A.SxPileupOpts(0, 17, 0, 0, 0, 10, 0, 0)
    elif mode == "edge":
        opts = A.SxPileupOpts(1, 17, 3, 1, 1, 2, 5, 0)
    lo, hi = ref_begin + 100, ref_begin + len(ref) - 150
    pb = B.PileupReadsBatch(reads, ref, ref_begin, lo, hi, cand, opts)
    want = reflib.ox_pileup_reads(pb)
    got = ctx.pileup_reads(pb)
    assert int(want[0][-1]) > 1000
    for w, g, name in zip(want, got, ("site_off", "calls", "t2_off", "t2_calls", "n_spandel", "n_submapped")):
        assert np.array_equal(w, g), name


def _buffer_order_case(rng, packed_quals, opts=None):
    """reads whose BEST alignment start differs from their read-buffer position (a realignment moved it, by up to +-25): the batch is in
    buffer order, the alignments are not sorted."""
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=int(rng.integers(600, 1500)), ref_len=int(rng.integers(900, 3000)))
    bpos = [int(r.pos) + (int(rng.integers(-25, 26)) if rng.random() < 0.4 else 0) for r in reads]
    order = np.argsort(np.asarray(bpos), kind="stable")
    reads, bpos = [reads[i] for i in order], [bpos[i] for i in order]
    qd = None
    if packed_quals:
        qd = sorted({int(q) for r in reads for q in r.quals})
        if len(qd) > 16:  # bin the qualities into a 16-entry dictionary first
            qd = qd[:: (len(qd) + 15) // 16][:16]
            for r in reads:
                r.quals = [min(qd, key=lambda v: abs(v - int(q))) for q in r.quals]
    lo, hi = ref_begin + 100, ref_begin + len(ref) - 150
    return B.PileupReadsBatch(reads, ref, ref_begin, lo, hi, cand, opts, buffer_pos=bpos, qual_dict=qd)


@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("seed", range(4))
def test_k4_pileup_in_read_buffer_order(ctx, seed, packed):
    """K4 keyed on the read-buffer position (starling_read_buffer.cpp:68-78): columns in the order the reference piles the reads up even
    where realignments moved the alignment starts past their neighbours'; dictionary-coded qualities."""
    pb = _buffer_order_case(np.random.default_rng(6300 + seed), packed)
    assert (np.diff(pb.reads["pos"][: pb.n_reads].astype(np.int64)) < 0).any()  # the alignments themselves are NOT sorted
    want = reflib.ox_pileup_reads(pb)
    got = ctx.pileup_reads(pb)
    assert int(want[0][-1]) > 1000
    for w, g, name in zip(want, got, ("site_off", "calls", "t2_off", "t2_calls", "n_spandel", "n_submapped")):
        assert np.array_equal(w, g), name


@pytest.mark.parametrize("mode", ["germline", "somatic", "edge"])
@pytest.mark.parametrize("packed", [False, True])
def test_k4_gather_plan(ctx, monkeypatch, mode, packed):
    """K4's second plan for the fill (SX_K4_PLAN=2: k4_bases_kernel, a thread per read, + k4_gather_kernel, a warp per 32 sites) gives the same
    columns as the oracle -- option modes, reads whose best alignment moved away from their buffer position, dictionary-coded qualities."""
    monkeypatch.setenv("SX_K4_PLAN", "2")
    opts = {"germline": None, "somatic": A.SxPileupOpts(1, 0, 20, 3, 1, 10, 0, 0), "edge": A.SxPileupOpts(1, 17, 3, 1, 1, 2, 5, 0)}[mode]
    pb = _buffer_order_case(np.random.default_rng(6400 + len(mode)), packed, opts)
    want = reflib.ox_pileup_reads(pb)
    got = ctx.pileup_reads(pb)
    assert int(want[0][-1]) > 1000
    for w, g, name in zip(want, got, ("site_off", "calls", "t2_off", "t2_calls", "n_spandel", "n_submapped")):
        assert np.array_equal(w, g), name


def test_k4_pileup_feeds_k2(ctx):
    """The columns K4 produces are an sx_pileup_batch: K2a on them == K2a on the oracle's columns."""
    rng = np.random.default_rng(6100)
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=1200, ref_len=2500, n_frac=0.0)
    lo, hi = ref_begin + 50, ref_begin + len(ref) - 50
    pb = B.PileupReadsBatch(reads, ref, ref_begin, lo, hi, cand)
    site_off, calls, t2_off, t2_calls, _, _ = ctx.pileup_reads(pb)
    ref_base = np.frombuffer(ref[lo - ref_begin: hi - ref_begin].encode(), dtype=np.uint8).copy()
    k2 = B.PileupBatch(site_off.copy(), np.concatenate([calls, np.zeros(16, np.uint16)]), ref_base, None)
    o = reflib.ox_pileup_reads(pb)
    k2o = B.PileupBatch(o[0].copy(), np.concatenate([o[1], np.zeros(16, np.uint16)]), ref_base, None)
    p = A.default_params()
    got, want = ctx.site_gl_germline(k2, True), reflib.ox_germline(p, k2o, True)
    for f in ("ref_gt", "is_computed", "n_used_calls", "phredLoghood"):
        assert np.array_equal(want[f], got[f]), f
    assert np.array_equal(_bits(want["lhood"]), _bits(got["lhood"]))


def test_k4_rejects_unsorted_reads(ctx):
    from strelka_b200.api import SxError

    rng = np.random.default_rng(6200)
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=50, ref_len=800)
    reads[10], reads[40] = reads[40], reads[10]
    pb = B.PileupReadsBatch(reads, ref, ref_begin, ref_begin, ref_begin + len(ref), cand)
    with pytest.raises(SxError) as e:
        ctx.pileup_reads(pb)
    assert e.value.code == A.SX_ERR_ARG


# ----------------------------------------------------------------------------------------------------------------------------
# K6 score_indels (SURVEY 8f2)
# ----------------------------------------------------------------------------------------------------------------------------
def _same_k6(want, got):
    for w, g in zip(want, got):
        assert w.dtype == g.dtype and w.shape == g.shape
        assert w.tobytes() == g.tobytes()


@pytest.mark.parametrize("case", range(16))
def test_k6_score_indels(ctx, case):
    """Records (ReadPathScores incl. alternate alleles, suboverlap marks), the arg-max and the evaluated alignment, byte for byte
    against the oracle; cases 0..7 also against what the REFERENCE's score_indels wrote (tests/golden/score_indels_ref.npz)."""
    import os

    sb, lnp = specgen.score_indels_case(case)
    got = ctx.score_indels(sb, lnp)
    _same_k6(reflib.ox_score_indels(sb, lnp), got)
    if case < specgen.SCORE_INDELS_GOLDEN_CASES:
        gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "score_indels_ref.npz"))
        assert got[0].tobytes() == gold[f"recs{case}"].tobytes()
        assert np.array_equal(got[1], gold[f"n_rec{case}"]) and np.array_equal(got[2], gold[f"max_aln{case}"])
    assert ctx.timing().launches == 5  # sizes + list, the list regrouped by alignment count (class, scan, scatter), score_indels


def test_k6_large_batch_with_deep_reads(ctx):
    """Thousands of regions (grid-stride over reads, every thread's scratch column in use) and reads with up to 60 candidate
    alignments (the per-batch scratch sizing)."""
    rng = np.random.default_rng(606)
    regions, lnp = specgen.random_score_indels_regions(rng, 3000, reads_per_region=(1, 8), alns_per_read=(1, 8))
    deep, lnp_deep = specgen.random_score_indels_regions(rng, 40, reads_per_region=(1, 4), alns_per_read=(20, 60), tie_rate=0.8)
    sb = B.ScoreIndelsBatch(regions + deep)
    lnp = np.concatenate([lnp[:-1], lnp_deep])
    assert lnp.size == sb.n_alns + 1 and sb.n_reads > 8000
    want = reflib.ox_score_indels(sb, lnp)
    _same_k6(want, ctx.score_indels(sb, lnp))
    assert int((want[0]["flags"] & A.SX_RIS_SCORED).sum()) > 5000 and int((want[2] != want[3]).sum()) > 50


def test_k6_consumes_k1_scores_on_device(ctx):
    """K1 -> K6 without the scores leaving HBM: sx_score_alignments_dev writes lnp, sx_score_indels_dev reads that buffer."""
    from strelka_b200.api import DevAlignBatch, DevScoreIndelsBatch

    rng = np.random.default_rng(607)
    regions = [specgen.simple_region(rng, n_reads=int(rng.integers(5, 40))) for _ in range(200)]
    ab = B.build_align_batch(regions, qual_bits=2, compact=True)
    sb = B.score_indels_batch_from_regions(regions)
    assert ab.n_alns == sb.n_alns
    dab, dsb = DevAlignBatch(ctx, ab), DevScoreIndelsBatch(ctx, sb)
    ctx.score_alignments_dev(dab)
    ctx.score_indels_dev(dsb, dab.out)
    want = reflib.ox_score_indels(sb, np.concatenate([reflib.ox_score(B.build_align_batch(regions)), [0.0]]))
    _same_k6(want, dsb.download())
    assert int((want[0]["flags"] & A.SX_RIS_SCORED).sum()) > 5000 and int((want[0]["n_alt"] > 0).sum()) > 1000


def test_k6_rejects_what_the_reference_asserts_on(ctx):
    from strelka_b200.api import SxError

    sb, lnp = specgen.score_indels_case(0)
    kind0 = int(sb.segs["kind"][0])
    sb.segs["kind"][0] = A.SX_SEG_SKIP  # score_indels' get_alignment_indel_bp_overlap asserts on SKIP (:176)
    with pytest.raises(SxError) as e:
        ctx.score_indels(sb, lnp)
    assert e.value.code == A.SX_ERR_UNSUPPORTED
    sb.segs["kind"][0] = kind0
    keep = sb.rec_off.copy()
    sb.rec_off[:] = 0  # no output slots at all
    with pytest.raises(SxError) as e:
        ctx.score_indels(sb, lnp)
    assert e.value.code == A.SX_ERR_NOMEM
    sb.rec_off[:] = keep
    k0 = int(sb.aln_keys[0]) if sb.n_aln_keys else 0
    if sb.n_aln_keys:
        sb.aln_keys[0] = 60000  # outside the region's window
        with pytest.raises(SxError) as e:
            ctx.score_indels(sb, lnp)
        assert e.value.code == A.SX_ERR_ARG
        sb.aln_keys[0] = k0
    _same_k6(reflib.ox_score_indels(sb, lnp), ctx.score_indels(sb, lnp))  # the context is usable again


def test_device_timer_brackets_the_entry_points(ctx):
    """sx_timer_mark / sx_timer_elapsed_ms (bench.py's timed region): the device time between two marks on the compute stream covers the kernels
    launched between them; a second pair of marks replaces the first; elapsed before both marks is an error, not a number."""
    from strelka_b200.api import Context, SxError

    fresh = Context(0)
    with pytest.raises(SxError):
        fresh.timer_elapsed_ms()
    fresh.close()
    rng = np.random.default_rng(5)
    pb = specgen.random_pileups(rng, 20000, depth=30.0, max_depth=96)
    ctx.site_gl_germline(pb, True)  # warm
    ctx.timer_mark(0)
    ctx.timer_mark(1)
    empty = ctx.timer_elapsed_ms()
    ctx.timer_mark(0)
    ctx.site_gl_germline(pb, True)
    k = ctx.timing().kernel_ms
    ctx.timer_mark(1)
    ms = ctx.timer_elapsed_ms()
    assert 0.0 <= empty < 1.0
    assert ms >= k > 0.0
