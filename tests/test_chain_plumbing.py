"""The device-resident realignment chain (strelka_b200.api.DevRealignChain: K7a -> K7 -> K7b -> K1 -> K6 + K9 with every intermediate in
"device" memory) dry-run on the CPU: tests/mockctx.py answers each `*_dev` entry point with the host-compiled body of that kernel (or
the oracle), so that the plumbing -- struct fields, buffer sizes, which totals size what -- is checked without a GPU.  The same chain on
an H100 against the same expectation: tests/test_zz_gpu_enumerate.py::test_device_resident_chain."""
import numpy as np
import pytest

import reflib
import refgold
import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B


def expected_chain(eb):
    """the chain on the CPU, step by step through the oracles (enumerate -> host flattening -> K1 oracle -> K6 oracle)."""
    out = reflib.ox_enumerate_alignments(eb, cap_alns=eb.n_reads * 64 + 64)
    regions = B.regions_from_enumeration(eb, out)
    lnp = reflib.ox_score(B.build_align_batch(regions))
    sb = specgen.score_indels_batch_from_enumeration(eb, out, ref_to_indel_lnp=0.0, indel_to_ref_lnp=0.0)
    recs, n_rec, max_aln, _ev = reflib.ox_score_indels(sb, np.concatenate([lnp, [0.0]]))
    return out, lnp, recs, n_rec, max_aln


def check_chain(chain, eb):
    out, lnp, recs, n_rec, max_aln = expected_chain(eb)
    g_out, g_lnp, g_n_rec, g_max_aln, g_recs = chain.download()
    for x, y in zip(out.trimmed(), g_out.trimmed()):
        assert x.tobytes() == y.tobytes()
    assert np.array_equal(lnp.view(np.uint64), g_lnp.view(np.uint64))
    assert np.array_equal(n_rec, g_n_rec) and np.array_equal(max_aln, g_max_aln)
    parts = [g_recs[int(chain.rec_off_host[r]) : int(chain.rec_off_host[r]) + int(g_n_rec[r])] for r in range(eb.n_reads)]
    got = np.concatenate(parts) if parts else g_recs[:0]
    assert got.tobytes() == recs.tobytes()
    # K9: the realignments, in K4's segment kinds -- against the reference itself where its library is built (the frozen reference
    # outputs cover the GPU box: tests/test_zz_gpu_enumerate.py::test_k9_choose_realignment)
    pos, n_seg, status, seg_off, segs = chain.download_realignments()
    assert int(seg_off[-1]) <= chain.realign["cap"] and set(np.unique(segs["kind"])) <= {0, 1, 3, 4, 5, 6}
    # ... and against the travelling oracle everywhere
    rb = B.RealignBatch(eb, out, k4_kinds=True, raw=getattr(chain, "raw_host", None))  # (with the mapper's alignments at hand K9 answers getBestAlignment())
    ox = reflib.ox_choose_realignment(rb, np.concatenate([lnp, [0.0]]))
    assert np.array_equal(ox.pos[: eb.n_reads], pos) and np.array_equal(ox.n_seg[: eb.n_reads], n_seg) and np.array_equal(ox.status[: eb.n_reads], status)
    assert np.array_equal(ox.seg_off[: eb.n_reads + 1], seg_off) and ox.segs[: int(seg_off[-1])].tobytes() == segs.tobytes()
    if reflib.have_ref():
        quals = np.full(int(eb.read_off[eb.n_reads]) + 1, 30, np.uint8)  # what B.read_pools_of gives every base
        ref_lnp, want = reflib.ref_choose_realignment(eb, out, quals)
        assert np.array_equal(ref_lnp.view(np.uint64), g_lnp.view(np.uint64))
        k4_char = {0: "M", 1: "I", 3: "S", 4: "H", 5: "D", 6: "N"}
        for r in range(eb.n_reads):
            if want[r] is None:
                assert not (int(status[r]) & A.SX_REALIGN_ST_REALIGNED)
                continue
            cig = "".join(f"{int(s['len'])}{k4_char[int(s['kind'])]}" for s in segs[int(seg_off[r]) : int(seg_off[r]) + int(n_seg[r])])
            assert (int(pos[r]), cig) == (want[r][0], want[r][1].replace("=", "M").replace("X", "M")), r
    return len(lnp), len(recs)


@pytest.mark.parametrize("case", [0, 1, 3, 5, 7])
def test_device_resident_chain_plumbing_on_the_cpu(case):
    from mockctx import MockContext
    from strelka_b200.api import DevRealignChain

    eb = specgen.enum_edge_case(case) if case % 2 else specgen.enum_case(case)
    pools = B.read_pools_of(eb)
    chain = DevRealignChain(MockContext(eb, pools), eb, pools, cap_alns_per_read=64)
    ms = chain.run()
    assert set(ms) == {"k7a_alignment_indels", "k7_enumerate", "k7b_link", "k1_score_alignments", "k6_score_indels", "k9_choose_realignment"}
    n_alns, n_recs = check_chain(chain, eb)
    assert n_alns > 50
    chain.run()  # a second pass over the same buffers
    check_chain(chain, eb)


def test_bench_chain_leg_on_the_mock():
    """bench.py's realign_chain leg (its numpy-built read pools included) through the mock context: the leg's own parity check passes
    and the K1 pools it builds obey K1's staging rule."""
    import os
    import sys

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    from mockctx import MockContext

    eb = bench.make_enum_workload(40, 30, 150, 7)
    pools = bench.make_enum_read_pools(eb, 30, 150, 7)
    assert not (pools.regions["seq_off"] % 16).any() and not (pools.regions["qual_off"] % 16).any() and not (pools.regions["ref_off"] % 16).any()
    leg = bench.realign_chain_leg(MockContext(eb, pools), 6572.2, n_loci=40, reps=1, check_loci=8)
    assert "identical to the oracle chain" in leg["parity"], leg
    assert leg["alignments"] > 40 * 30 * 5 and set(leg["kernel_ms"]) == {"k7a_alignment_indels", "k7_enumerate", "k7b_link", "k1_score_alignments", "k6_score_indels", "k9_choose_realignment"}
    # the numpy-built pools are what read_pools_of builds from the same workload (up to the qualities)
    ref = B.read_pools_of(eb)
    assert np.array_equal(pools.regions["read_begin"], ref.regions["read_begin"]) and np.array_equal(pools.regions["ref_begin"][:40], ref.regions["ref_begin"][:40])
    stride = int(ref.regions["seq_off"][1])
    used = 30 * 75  # 30 reads of 150 bases, two per byte; the rest of a region's slice is padding
    assert np.array_equal(pools.seq4[: 40 * stride].reshape(40, stride)[:, :used], ref.seq4[: 40 * stride].reshape(40, stride)[:, :used])
    rstride = int(ref.regions["ref_off"][1])
    assert np.array_equal(pools.ref[: 40 * rstride].reshape(40, rstride)[:, :1000], ref.ref[: 40 * rstride].reshape(40, rstride)[:, :1000])


def test_bench_pools_quality_packing():
    """the chain leg's numpy-built K1 pools with dictionary-coded qualities (qual_bits 4) describe the same reads as the one-byte-per-base
    pools: the K1 oracle scores the linked alignments identically on both."""
    import os
    import sys

    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    from mockctx import MockContext
    from strelka_b200.api import DevRealignChain

    eb = bench.make_enum_workload(12, 30, 150, 11)
    lnp = {}
    for bits in (4, 8):
        pools = bench.make_enum_read_pools(eb, 30, 150, 11, qual_bits=bits)
        chain = DevRealignChain(MockContext(eb, pools), eb, pools, cap_alns_per_read=16)
        chain.run()
        lnp[bits] = chain.download()[1]
    assert len(lnp[4]) > 12 * 30 * 5 and np.array_equal(lnp[4].view(np.uint64), lnp[8].view(np.uint64))
    assert len(np.unique(lnp[4])) > 50  # three quality values really vary the scores


def normalized_batch(eb, gb, gate_out):
    """the EnumBatch a host shim would build after the gates: the same reads with their NORMALIZED input alignment (pads dropped) and the
    gate bytes set -- built through the ordinary host builder, so in_keys come from batch.alignment_indels."""
    regions = []
    for g in range(eb.n_regions):
        k0, k1 = int(eb.region_key_off[g]), int(eb.region_key_off[g + 1])
        win = []
        for k in range(k0, k1):
            key, hap = eb.keys[k], eb.key_hap[k]
            ins = bytes(eb.ins_pool[int(eb.ins_off[k]) : int(eb.ins_off[k + 1])]).decode()
            fl = int(key["flags"])
            win.append(B.EnumKeySpec(int(key["pos"]), int(key["del_len"]), ins, mismatch=int(key["type"]) == A.SX_INDEL_TYPE_MISMATCH, candidate=bool(fl & 1),
                                     not_discovered=bool(fl & 2), forced=bool(fl & 4), active_region=int(hap["active_region_id"]),
                                     hap_ids=tuple(int(x) for x in hap["haplotype_id"]), bypass=int(hap["bypass_mask"])))
        reads = []
        for r in range(int(eb.region_read_off[g]), int(eb.region_read_off[g + 1])):
            seq = bytes(eb.read_pool[int(eb.read_off[r]) : int(eb.read_off[r + 1])]).decode()
            al = gate_out.alignment_of(r)
            if al is None:  # gated out: any valid alignment will do, the gate byte keeps the read out of the search
                al = (int(eb.in_pos[r]), "".join(f"{int(s['len'])}{B.AP_CHAR[int(s['kind'])]}" for s in eb.in_segs[int(eb.in_seg_off[r]) : int(eb.in_seg_off[r + 1])]))
            use = [int(x) for x in eb.use_keys[int(eb.use_key_off[r]) : int(eb.use_key_off[r + 1])]]
            reads.append(B.EnumReadSpec(seq, al[0], B.parse_cigar(al[1]), use))
        ref = bytes(eb.ref_pool[int(eb.ref_off[g]) : int(eb.ref_off[g + 1])]).decode()
        regions.append((ref, int(eb.ref_begin[g]), (int(eb.realign_begin[g]), int(eb.realign_end[g])), win, reads))
    nb = B.EnumBatch(regions, eb.opts, strict=False)
    nb.set_gate(gate_out.gate[: eb.n_reads + 1].copy())
    return nb


@pytest.mark.parametrize("case", [0, 1, 3, 4])
def test_chain_from_the_mappers_alignments_on_the_cpu(case):
    """the chain with K7g in front (mapper alignments in): identical to the chain run on the batch a host shim would build from the
    gates' answers with the ordinary host builder."""
    from mockctx import MockContext
    from strelka_b200.api import DevRealignChain

    eb = specgen.enum_edge_case(case) if case % 2 else specgen.enum_case(case)
    gb = B.GateBatch(eb, specgen.raw_alignments_for(eb, case))
    pools = B.read_pools_of(eb)
    chain = DevRealignChain(MockContext(eb, pools), eb, pools, cap_alns_per_read=64, raw=gb)
    ms = chain.run()
    assert "k7g_realign_gates" in ms
    rc, gates = reflib.k7gcore_gates(gb)
    assert rc == 0 and 0 < int((gates.gate[: eb.n_reads] & A.SX_GATE_REALIGN != 0).sum())
    check_chain(chain, normalized_batch(eb, gb, gates))


def chain_case(case):
    """seeded batch `case` of the comparisons with realignAndScoreRead: (eb, gb), the mapper's alignments in"""
    eb = specgen.enum_edge_case(case) if case % 2 else specgen.enum_case(case)
    return eb, B.GateBatch(eb, specgen.raw_alignments_for(eb, 100 + case))


def use_the_references_bound(eb):
    eb.opts.max_alns_per_read = 5000  # the reference's own bound (opt.max_realignment_candidates): no read is left to the caller for its alignment count
    eb.c.opts = eb.opts


def chain_inputs_digest(eb, gb):
    return refgold.inputs_digest(eb.read_pool, eb.ref_pool, gb.raw_pos, gb.raw_segs)


def raw_alignment(gb, r):
    return (int(gb.raw_pos[r]), "".join(f"{int(s['len'])}{B.AP_CHAR[int(s['kind'])]}" for s in gb.raw_segs[int(gb.seg_off[r]) : int(gb.seg_off[r + 1])]).replace("=", "M").replace("X", "M"))


def chain_reference(eb, gb):
    """the reference's realignAndScoreRead on every read: (items, indices of the reads it threw on).  Items: per read the reference does not
    throw on, (read, is_realigned, best alignment as (pos, cigar in K4 letters), #records, the records' bytes)."""
    n = eb.n_reads
    n_win = np.diff(eb.region_key_off.astype(np.int64))
    rec_off = np.concatenate([[0], np.cumsum(np.repeat(n_win, np.diff(eb.region_read_off.astype(np.int64))))]).astype(np.uint32)
    quals = np.full(int(eb.read_off[n]) + 1, 30, np.uint8)  # what B.read_pools_of gives every base
    ref_status, want, r_recs, r_n_rec = reflib.ref_realign_and_score_read(gb, quals, rec_off=rec_off)
    reads = []
    for r in range(n):
        if ref_status[r] == 2:
            continue
        best = raw_alignment(gb, r) if want[r] is None else (want[r][0], want[r][1].replace("=", "M").replace("X", "M"))
        o = int(rec_off[r])
        reads.append((r, want[r] is not None, best, int(r_n_rec[r]), r_recs[o : o + int(r_n_rec[r])].tobytes()))
    return {"reads": reads}, [int(r) for r in np.nonzero(ref_status == 2)[0]]


def chain_vs_realign_and_score_read(ctx, eb, gb, case, cap_alns_per_read=2048):
    """The chain K7g -> K7a -> K7 -> K7b -> K1 -> K6 + K9 from the mapper's alignments (chain_case(case)) against the reference's own
    realignAndScoreRead (starling_read_align.cpp:2026-2127) run per read on rebuilt objects -- or its frozen digests, tests/refgold.py:
    is_realigned, rseg.realignment segment for segment (hard clips included), getBestAlignment() of the reads that keep the mapper's alignment,
    and the ReadPathScores score_indels left in the indel buffer.  Returns (#realigned, #records, #reads the reference threw on)."""
    from strelka_b200.api import DevRealignChain

    use_the_references_bound(eb)
    entry = refgold.golden()["chain"].get(str(case))
    if entry is not None:
        assert entry["inputs"] == chain_inputs_digest(eb, gb), "the seeded inputs changed: regenerate tests/golden/window_ref_digests.json"
    want, threw = chain_reference(eb, gb) if reflib.have_ref() else (None, entry["threw"])
    pools = B.read_pools_of(eb)
    chain = DevRealignChain(ctx, eb, pools, cap_alns_per_read=cap_alns_per_read, raw=gb)
    chain.run()
    pos, n_seg, status, seg_off, segs = chain.download_realignments()
    g_out, _lnp, g_n_rec, _max_aln, g_recs = chain.download()
    k4_char = {0: "M", 1: "I", 3: "S", 4: "H", 5: "D", 6: "N"}
    reads = []
    for r in sorted(set(range(eb.n_reads)) - set(threw)):  # where the reference threw (blt_exception) the chain reports the read
        # (SX_ENUM_ST_EXCEPTION) or, where the throw comes from scoring a generator corner, answers something the reference does not define
        assert not (int(g_out.status[r]) & A.SX_ENUM_ST_LIMIT), (r, "per-read capacity of the test too small")
        cig = "".join(f"{int(s['len'])}{k4_char[int(s['kind'])]}" for s in segs[int(seg_off[r]) : int(seg_off[r]) + int(n_seg[r])])
        o = int(chain.rec_off_host[r])
        reads.append((r, bool(int(status[r]) & A.SX_REALIGN_ST_REALIGNED), (int(pos[r]), cig), int(g_n_rec[r]), g_recs[o : o + int(g_n_rec[r])].tobytes()))
    chain.free()
    refgold.compare({"reads": reads}, want, entry)
    return sum(x[1] for x in reads), sum(x[3] for x in reads), len(threw)


@pytest.mark.parametrize("case", range(10))
def test_chain_against_the_references_realignAndScoreRead(case):
    """end to end on the CPU mock (host-compiled device bodies): see chain_vs_realign_and_score_read; the same on an H100:
    tests/test_zz_gpu_enumerate.py::test_chain_equals_the_references_realignAndScoreRead."""
    from mockctx import MockContext

    eb, gb = chain_case(case)
    n_real, n_recs, n_threw = chain_vs_realign_and_score_read(MockContext(eb, B.read_pools_of(eb)), eb, gb, case)
    assert n_real > 0 and n_threw <= eb.n_reads // 2, (n_real, n_recs, n_threw)
