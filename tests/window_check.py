"""TEST INFRASTRUCTURE: sx_process_window_dev (the device-resident pass K7g -> K7a -> K7 -> K7b -> K1 -> K6 + K9 -> K4 -> K2a) against the
REFERENCE run stage by stage on the same window through oracle/_ref/libstrelka_ref.so:
    realignAndScoreRead per read            (ref_realign_and_score_read_ex: is_realigned, rseg.realignment, the ReadPathScores it left)
    pileup_read_segment per read            (ref_pileup_reads, in read-buffer order, each read through getBestAlignment())
    position_snp_call_pprob_digt per site   (ref_site_gl_germline)
Where the reference library is absent, check_window compares with the reference's frozen digests (tests/refgold.py)."""
import os
import sys

import numpy as np

import reflib
import refgold
import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import window_workload as WW  # noqa: E402

K4_CHAR = {0: "M", 1: "I", 3: "S", 4: "H", 5: "D", 6: "N"}
COL_NAMES = ("site_off", "calls", "t2_off", "t2_calls", "n_spandel", "n_submapped")


def buffer_pos_of(pos, path):
    """get_alignment_buffer_pos (starling_read_util.cpp:30-35): pos - unalignedPrefixSize"""
    lead = 0
    for t, ln in path:
        if t not in "IHS":
            break
        if t != "H":
            lead += ln
    return pos - lead


def single_region_windows(eb, raw):
    """every region of a test EnumBatch as a batch of its own (eb1, gb1) with its reads in READ-BUFFER order (the mapper's position minus the
    unaligned prefix; ties keep their order) -- a window on its own contig segment, as sx_process_window_dev takes it."""
    for g in range(eb.n_regions):
        k0, k1 = int(eb.region_key_off[g]), int(eb.region_key_off[g + 1])
        win = []
        for k in range(k0, k1):
            key, hap = eb.keys[k], eb.key_hap[k] if eb.has_hap else None
            ins = bytes(eb.ins_pool[int(eb.ins_off[k]) : int(eb.ins_off[k + 1])]).decode()
            fl = int(key["flags"])
            ks = B.EnumKeySpec(int(key["pos"]), int(key["del_len"]), ins, mismatch=int(key["type"]) == A.SX_INDEL_TYPE_MISMATCH, candidate=bool(fl & 1),
                               not_discovered=bool(fl & 2), forced=bool(fl & 4), active_region=int(hap["active_region_id"]) if hap is not None else -1,
                               hap_ids=tuple(int(x) for x in hap["haplotype_id"]) if hap is not None else (0, 0, 0, 0), bypass=int(hap["bypass_mask"]) if hap is not None else 0)
            win.append(ks)
        r0, r1 = int(eb.region_read_off[g]), int(eb.region_read_off[g + 1])
        order = sorted(range(r0, r1), key=lambda r: buffer_pos_of(*raw[r]))  # stable
        reads, raw1 = [], []
        for r in order:
            seq = bytes(eb.read_pool[int(eb.read_off[r]) : int(eb.read_off[r + 1])]).decode()
            # '=' and IUPAC codes cannot be piled up (base_to_id ends the reference's process; K4 reports them): such bases become 'N' here --
            # their handling by the search front is tests/test_enumerate.py's and the chain tests' subject
            seq = "".join(c if c in "ACGTN" else "N" for c in seq)
            al = (int(eb.in_pos[r]), [(B.AP_CHAR[int(s["kind"])], int(s["len"])) for s in eb.in_segs[int(eb.in_seg_off[r]) : int(eb.in_seg_off[r + 1])]])
            use = [int(x) for x in eb.use_keys[int(eb.use_key_off[r]) : int(eb.use_key_off[r + 1])]]
            reads.append(B.EnumReadSpec(seq, al[0], al[1], use))
            raw1.append(raw[r])
        if not reads:
            continue
        ref = bytes(eb.ref_pool[int(eb.ref_off[g]) : int(eb.ref_off[g + 1])]).decode()
        eb1 = B.EnumBatch([(ref, int(eb.ref_begin[g]), (int(eb.realign_begin[g]), int(eb.realign_end[g])), win, reads)], eb.opts, strict=False)
        yield eb1, B.GateBatch(eb1, raw1)


def cigar_of(segs):
    return "".join(f"{int(s['len'])}{K4_CHAR[int(s['kind'])]}" for s in segs if not (int(s["kind"]) == A.SX_SEG_HARDCLIP and int(s["len"]) == 0))


def parse_k4(cig):
    out, num = [], ""
    for ch in cig:
        if ch.isdigit():
            num += ch
        else:
            out.append((ch, int(num)))
            num = ""
    return out


def raw_of(gb, r):
    """the mapper's alignment of read r: ((pos, cigar in K4 letters), [(op, len)])"""
    raw_path = [(B.AP_CHAR[int(s["kind"])], int(s["len"])) for s in gb.raw_segs[int(gb.seg_off[r]) : int(gb.seg_off[r + 1])]]
    return (int(gb.raw_pos[r]), "".join(f"{ln}{t}" for t, ln in raw_path).replace("=", "M").replace("X", "M")), raw_path


def reference_window(eb, gb, w, quals=None, params=None):
    """the window through the reference, stage by stage: per-read (status, best alignment as (pos, cigar in K4 letters), records), the
    columns and the site results (None when the reference threw on a read: its process would have stopped there)"""
    n = eb.n_reads
    if quals is None:
        quals = np.full(int(eb.read_off[n]) + 1, 30, np.uint8)
    flags = w.a["read_flags"]
    k6_flags = (flags[: n + 1] & 3).astype(np.uint8)  # SX_SIF_FWD / SX_SIF_TIER1 are SX_PRF_FWD / SX_PRF_TIER1
    submapped = (flags[:n] & A.SX_PRF_TIER1OR2) == 0
    ref_status, want, r_recs, r_n_rec = reflib.ref_realign_and_score_read(gb, quals, read_flags=k6_flags, rec_off=w.a["rec_off"])
    exp = {"status": ref_status, "want": want, "recs": r_recs, "n_rec": r_n_rec, "submapped": submapped, "best": [], "cols": None, "gl": None}
    raws = []
    for r in range(n):
        raw, raw_path = raw_of(gb, r)
        raws.append((raw, raw_path))
        if submapped[r] or (ref_status[r] != 2 and want[r] is None):
            exp["best"].append(raw)
        elif ref_status[r] == 2:
            exp["best"].append(None)
        else:
            exp["best"].append((want[r][0], want[r][1].replace("=", "M").replace("X", "M")))
    exp["raw"] = [x[0] for x in raws]
    if (ref_status[~submapped] == 2).any():
        return exp
    # ---- the pile-up: the reference's pileup_read_segment on ITS best alignments, in read-buffer order
    specs, bpos = [], []
    for r in range(n):
        seq = bytes(eb.read_pool[int(eb.read_off[r]) : int(eb.read_off[r + 1])]).decode()
        q = quals[int(eb.read_off[r]) : int(eb.read_off[r + 1])]
        f = int(flags[r])
        tier = 1 if f & A.SX_PRF_TIER1 else (2 if f & A.SX_PRF_TIER1OR2 else 0)
        raw_path = raws[r][1]
        bpos.append(buffer_pos_of(int(gb.raw_pos[r]), raw_path))
        sp = B.PileupReadSpec(B.codes_of(seq), q, exp["best"][r][0], parse_k4(exp["best"][r][1]), fwd=bool(f & A.SX_PRF_FWD), mapq=int(w.a["mapq"][r]), tier=tier)
        # pileup_read_segment :1145-1148: a read that was not realigned and has no alignment with indels the caller handles is not piled up
        not_realigned = submapped[r] or want[r] is None
        sp.skip = bool(not_realigned and any(t in "ID" and ln > eb.opts.max_indel_size for t, ln in raw_path[1:-1]))
        specs.append(sp)
    ref_str = bytes(w.a["ref"][: w.used["ref"]]).decode()
    pb = B.PileupReadsBatch(specs, ref_str, w.ref_begin, w.report_begin, w.report_end, buffer_pos=bpos)
    for r, sp in enumerate(specs):
        if sp.skip:
            pb.reads["flags"][r] |= A.SX_PRF_SKIP
    cols = reflib.ref_pileup_reads(pb) if reflib.have_ref() else reflib.ox_pileup_reads(pb)
    exp["cols"] = cols
    ref_base = np.frombuffer(ref_str[w.report_begin - w.ref_begin : w.report_end - w.ref_begin].encode(), dtype=np.uint8).copy()
    k2 = B.PileupBatch(cols[0].copy(), np.concatenate([cols[1], np.zeros(16, np.uint16)]), ref_base, None)
    params = params or A.default_params()
    exp["gl"] = reflib.ref_germline(params, k2, True) if reflib.have_ref() else reflib.ox_germline(params, k2, True)
    return exp


def window_case(case):
    """the single-region windows of seeded batch `case`, each as (eb1, gb1, read_flags, mapq): strands, tiers (a few tier2 and sub-mapped
    reads), mapping qualities and indel error rates vary"""
    eb = specgen.enum_edge_case(case) if case % 2 else specgen.enum_case(case)
    raw = specgen.raw_alignments_for(eb, 100 + case)
    for eb1, gb1 in single_region_windows(eb, raw):
        rng = np.random.default_rng(77000 + case)
        n = eb1.n_reads
        tier = rng.choice([1, 1, 1, 1, 2, 0], size=n + 1)
        flags = ((rng.random(n + 1) < 0.5).astype(np.uint8) * A.SX_PRF_FWD) | np.where(tier == 1, A.SX_PRF_TIER1 | A.SX_PRF_TIER1OR2, 0).astype(np.uint8) | np.where(
            tier == 2, A.SX_PRF_TIER1OR2, 0).astype(np.uint8)
        eb1.keys["ref_to_indel_lnp"][: eb1.n_keys] = -rng.uniform(5.0, 12.0, eb1.n_keys)
        eb1.keys["indel_to_ref_lnp"][: eb1.n_keys] = -rng.uniform(5.0, 12.0, eb1.n_keys)
        mapq = rng.choice([60, 60, 60, 30, 3], size=n + 1).astype(np.uint8)
        yield eb1, gb1, flags, mapq


def reference_items(exp, w):
    """reference_window's answers as the items check_window compares: per read handed to realignAndScoreRead that the reference did not
    throw on, (read, is_realigned, best alignment, #records, the records' bytes); the columns and site results where it piled up"""
    ro = w.a["rec_off"]
    reads = []
    for r in range(len(exp["status"])):
        if exp["submapped"][r] or exp["status"][r] == 2:
            continue
        o, k = int(ro[r]), int(exp["n_rec"][r])
        reads.append((r, exp["want"][r] is not None, exp["best"][r], k, exp["recs"][o : o + k].tobytes()))
    it = {"reads": reads}
    if exp["cols"] is not None:
        it.update(zip(COL_NAMES, exp["cols"]))
        it.update(WW.site_gl_items(exp["gl"]))
    return it


def check_window(ctx, eb, gb, key, read_flags=None, mapq=None):
    """one window through sx_process_window_dev and through the reference (or its frozen digests under `key`, tests/refgold.py); returns
    counters.  Qualities: B.read_pools_of's constant 30, as the reference harness gets them."""
    n = eb.n_reads
    w = B.WindowBatch.from_enum(eb, gb, B.read_pools_of(eb), read_flags=read_flags, mapq=mapq)
    entry = refgold.golden()["window"].get(key)  # (the batches' seeded inputs are checked by the chain comparisons of the same cases)
    if reflib.have_ref():
        exp = reference_window(eb, gb, w)
        want, threw, piled = reference_items(exp, w), [int(r) for r in np.nonzero(exp["status"] == 2)[0]], exp["cols"] is not None
    else:
        want, threw, piled = None, entry["threw"], entry["piled"]
    submapped = (w.a["read_flags"][:n] & A.SX_PRF_TIER1OR2) == 0
    from strelka_b200.api import DevWindow

    dw = DevWindow(ctx, w)
    stage_ms = dw.run()
    d = dw.download()
    dw.free()
    seg_off, segs = d["best_seg_off"], d["best_segs"]
    reads = []
    for r in range(n):
        got = (int(d["best_pos"][r]), cigar_of(segs[int(seg_off[r]) : int(seg_off[r]) + int(d["best_n_seg"][r])]))
        if submapped[r]:  # align_pos :746: never handed to realignAndScoreRead
            raw = raw_of(gb, r)[0]
            assert not (int(d["gate"][r]) & A.SX_GATE_REALIGN) and got == raw, (r, got, raw)
            continue
        if r in threw:
            continue
        assert not (int(d["enum_status"][r]) & A.SX_ENUM_ST_LIMIT), (r, "a per-read capacity of the search")
        o, k = int(w.a["rec_off"][r]), int(d["n_rec"][r])
        reads.append((r, bool(int(d["realign_status"][r]) & A.SX_REALIGN_ST_REALIGNED), got, k, d["recs"][o : o + k].tobytes()))
    it = {"reads": reads}
    if piled:  # (else the reference process would have stopped at the throw: no pile-up to compare)
        it.update(zip(COL_NAMES, (d["site_off"], d["calls"], d["t2_off"], d["t2_calls"], d["n_spandel"], d["n_submapped"])))
        it.update(WW.site_gl_items(d["site_gl"]))
    refgold.compare(it, want, entry)
    return {"reads": n, "realigned": sum(x[1] for x in reads), "records": sum(x[3] for x in reads), "threw": len(threw),
            "calls": int(d["site_off"][-1]) if piled else 0, "sites": w.n_sites if piled else 0, "stage_ms": stage_ms}
