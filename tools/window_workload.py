"""BENCH/TEST TOOLING: BASELINE.json's cfg2 as whole-path windows (tools/synth_window.cpp): the synthetic input of sx_process_window_dev and --
the same arrays -- of the reference arm (the reference's own realignAndScoreRead / pileup_read_segment / position_snp_call_pprob_digt through
oracle/_ref/libstrelka_ref.so).  Nothing here is part of the product."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200 import batch as B  # noqa: E402

CELL_LEN, READS_PER_CELL, READ_LEN = 300, 60, 150  # 60 reads of 150 bp per 300 bp = 30x
REF_LEAD = 64
QUAL_DICT = [11, 25, 37]


class WindowSizes(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("n_regions", "n_reads", "n_keys", "n_raw_segs", "seq4_bytes", "qual_bytes", "ref_bytes", "key_ins_bytes", "n_sites")]


def load_synth():
    p = os.path.join(ROOT, "tools", "libsx_synth.so")
    if not os.path.exists(p) or os.path.getmtime(p) < os.path.getmtime(os.path.join(ROOT, "tools", "synth_window.cpp")):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tools")])
    lib = C.CDLL(p)
    lib.synth_pileups.restype = C.c_uint64
    lib.synth_ga.restype = C.c_uint64
    return lib


def make_window(synth, n_cells: int, seed: int, tile: int = 0, qual_bits: int = 4, threads: int = 8, ascii_reads: bool = False, alloc=None,
                ref_to_indel_lnp: float = -9.0, indel_to_ref_lnp: float = -7.0) -> B.WindowBatch:
    """One window of n_cells candidate loci (tile `tile` of a contig: its own coordinates and RNG streams).  alloc(nbytes, dtype) -> array (pinned
    host memory in bench.py's end-to-end leg); ascii_reads: also keep the reads as ASCII + one-byte qualities (what the reference harness takes)."""
    alloc = alloc or (lambda nbytes, dt: np.zeros(max(1, (nbytes + np.dtype(dt).itemsize - 1) // np.dtype(dt).itemsize), dtype=dt))
    contig_begin = 1024 + REF_LEAD + tile * (n_cells * CELL_LEN + 2048)  # (contig_begin - REF_LEAD) % 16 == 0
    contig_begin -= (contig_begin - REF_LEAD) % 16
    seed_t = seed * 1000003 + tile
    seg_count, ins_count = np.zeros(n_cells, np.uint32), np.zeros(n_cells, np.uint32)
    sz = WindowSizes()
    rc = synth.synth_window_plan(n_cells, READS_PER_CELL, READ_LEN, CELL_LEN, C.c_uint64(seed_t), contig_begin, qual_bits, threads, C.c_void_p(seg_count.ctypes.data),
                                 C.c_void_p(ins_count.ctypes.data), C.byref(sz))
    assert rc == 0, rc
    n, nk = int(sz.n_reads), int(sz.n_keys)
    S = A.SX_POOL_SLACK
    a = {
        "region_read_off": alloc((n_cells + 1) * 4, np.uint32), "region_key_off": alloc((n_cells + 1) * 4, np.uint32), "keys": alloc((nk + 1) * A.INDEL_KEY_DT.itemsize, A.INDEL_KEY_DT),
        "key_hap": None, "key_ins_off": alloc((nk + 1) * 4, np.uint32), "key_ins": alloc(int(sz.key_ins_bytes) + S, np.uint8), "realign_begin": alloc((n_cells + 1) * 4, np.int32),
        "realign_end": alloc((n_cells + 1) * 4, np.int32), "raw_pos": alloc((n + 1) * 4, np.int32), "raw_seg_off": alloc((n + 1) * 4, np.uint32),
        "raw_segs": alloc((int(sz.n_raw_segs) + 16) * 4, A.ALN_SEG_DT), "read_len": alloc((n + 8) * 2, np.uint16), "read_flags": alloc(n + 16, np.uint8), "mapq": alloc(n + 16, np.uint8),
        "use_key_off": alloc((n + 1) * 4, np.uint32), "use_keys": alloc(16, np.uint16), "rec_off": alloc((n + 1) * 4, np.uint32),
        "regions": alloc((n_cells + 1) * A.REGION_DT.itemsize, A.REGION_DT), "seq4": alloc(int(sz.seq4_bytes) + S, np.uint8), "qual": alloc(int(sz.qual_bytes) + S, np.uint8),
        "ref": alloc(int(sz.ref_bytes) + S, np.uint8), "cand_snv": None,
    }
    read_ascii = np.zeros(n * READ_LEN + 1, np.uint8) if ascii_reads else None
    qual_wide = np.zeros(n * READ_LEN + 1, np.uint8) if ascii_reads else None
    order = ("region_read_off", "region_key_off", "keys", "key_ins_off", "key_ins", "realign_begin", "realign_end", "raw_pos", "raw_seg_off", "raw_segs", "read_len", "read_flags", "mapq",
             "use_key_off", "rec_off", "regions", "seq4", "qual", "ref")
    rc = synth.synth_window_fill(n_cells, READS_PER_CELL, READ_LEN, CELL_LEN, C.c_uint64(seed_t), contig_begin, qual_bits, threads, C.c_void_p(seg_count.ctypes.data),
                                 C.c_void_p(ins_count.ctypes.data), *[C.c_void_p(a[k].ctypes.data) for k in order], C.c_void_p(read_ascii.ctypes.data) if ascii_reads else None,
                                 C.c_void_p(qual_wide.ctypes.data) if ascii_reads else None, C.c_double(ref_to_indel_lnp), C.c_double(indel_to_ref_lnp))
    assert rc == 0, rc
    w = B.WindowBatch(a, n_cells, n, nk, contig_begin - REF_LEAD, contig_begin, contig_begin + n_cells * CELL_LEN, qual_bits, QUAL_DICT if qual_bits == 4 else None, READ_LEN, True,
                      {"seq4": int(sz.seq4_bytes), "qual": int(sz.qual_bytes), "ref": int(sz.ref_bytes)})
    w.read_ascii, w.qual_wide, w.n_raw_segs, w.n_cells = read_ascii, qual_wide, int(sz.n_raw_segs), n_cells
    return w


def input_bytes(w: B.WindowBatch) -> int:
    """bytes of a window's input arrays as they cross PCIe (used bytes, no slack)"""
    n, nr, nk = w.n_reads, w.n_regions, w.n_keys
    return (w.used["seq4"] + w.used["qual"] + w.used["ref"] + (nr + 1) * (4 + 4 + 48) + nr * 8 + nk * A.INDEL_KEY_DT.itemsize + (nk + 1) * 4 + int(w.a["key_ins_off"][nk])
            + n * (4 + 2 + 1 + 1) + (n + 1) * 12 + w.n_raw_segs * 4)


def algorithmic_bytes(w: B.WindowBatch, totals) -> int:
    """what one pass has to move at the least: every input byte once, every result once (best alignments, score_indels records, the columns, the site records)"""
    n = w.n_reads
    return int(input_bytes(w) + n * (4 + 4 + 2 + 3) + int(totals[5]) * 4 + n * 3 * 32 // 3 + int(totals[6]) * 2 + w.n_sites * (16 + A.DIGT_RESULT_DT.itemsize))


# ------------------------------------------------------------------------------------------------------------------------------
# the reference arm: the same window through the reference's own functions (oracle/_ref/libstrelka_ref.so)
# ------------------------------------------------------------------------------------------------------------------------------
def _ref_lib():
    p = os.path.join(ROOT, "oracle", "_ref", "libstrelka_ref.so")
    return C.CDLL(p) if os.path.exists(p) else None


def gate_batch_of(w: B.WindowBatch) -> A.SxGateBatch:
    a = w.a
    return A.SxGateBatch(w.n_regions, w.n_reads, A.ptr(a["region_read_off"]), A.ptr(a["region_key_off"]), A.ptr(a["keys"]), A.ptr(a["realign_begin"]), A.ptr(a["realign_end"]),
                         A.ptr(a["raw_pos"]), A.ptr(a["raw_seg_off"]), A.ptr(a["raw_segs"]), A.ptr(a["read_len"]), None, 49)


def reference_pass(w: B.WindowBatch, params=None, max_segs: int = 16):
    """The window through the reference, stage by stage; returns (results dict, seconds dict).  Seconds: the time inside the reference's own
    functions (the harness's object construction around them is not the reference's work and is left out; the *_call entries include it)."""
    rf = _ref_lib()
    assert rf is not None and w.read_ascii is not None, "reference library not built / window made without ascii_reads"
    a, n, ns = w.a, w.n_reads, w.n_sites
    _P = C.c_void_p
    err = C.create_string_buffer(1024)
    gb = gate_batch_of(w)
    status, pos, nseg = np.zeros(n + 1, np.uint8), np.zeros(n + 1, np.int32), np.zeros(n + 1, np.uint16)
    segs = np.zeros((n + 1) * max_segs, dtype=A.ALN_SEG_DT)
    recs, n_rec = np.zeros(int(a["rec_off"][n]) + 1, A.READ_INDEL_SCORE_DT), np.zeros(n + 1, np.uint32)
    read_off = (np.arange(n + 1, dtype=np.int64) * READ_LEN).astype(np.uint32)
    reg = a["regions"]
    ref_off, ref_len, ref_begin = reg["ref_off"][: w.n_regions + 1].astype(np.uint32), reg["ref_len"][: w.n_regions + 1].astype(np.uint32), reg["ref_begin"][: w.n_regions + 1].astype(np.int32)
    k6_flags = (a["read_flags"][: n + 1] & 3).astype(np.uint8)
    secs = C.c_double(0.0)
    fn = rf.ref_realign_and_score_read_ex
    fn.argtypes = [C.POINTER(A.SxGateBatch), _P] + [_P] * 10 + [C.c_int, C.c_int, C.c_double] + [_P] * 4 + [C.c_uint32] + [_P] * 4 + [C.c_char_p, C.c_int]
    t0 = time.perf_counter()
    rc = fn(C.byref(gb), None, A.ptr(a["key_ins"]), A.ptr(a["key_ins_off"]), A.ptr(a["ref"]), A.ptr(ref_off), A.ptr(ref_len), A.ptr(ref_begin), A.ptr(w.read_ascii), A.ptr(read_off),
            A.ptr(w.qual_wide), A.ptr(k6_flags), 0, 1, 2.302585092994046, A.ptr(status), A.ptr(pos), A.ptr(nseg), A.ptr(segs), max_segs, A.ptr(a["rec_off"]), A.ptr(recs), A.ptr(n_rec),
            C.addressof(secs), err, 1024)
    t_realign_call = time.perf_counter() - t0
    if rc != 0:
        raise RuntimeError(err.value.decode(errors="replace"))
    # getBestAlignment() of every read, as K4-kind CSR (what pileup_read_segment piles up)
    rso = a["raw_seg_off"][: n + 1].astype(np.int64)
    realigned = status[:n] == 1
    n_best = np.where(realigned, nseg[:n].astype(np.int64), np.diff(rso))
    best_off = np.concatenate([[0], np.cumsum(n_best)]).astype(np.uint32)
    best = np.zeros(int(best_off[n]) + 16, dtype=A.ALN_SEG_DT)
    kind_map = np.array([4, 0, 1, 5, 6, 3, 4, 4, 0, 0], np.uint8)  # SX_AP_* -> K4's SX_SEG_* ('=' / 'X' as MATCH)
    src_seg = segs.reshape(n + 1, max_segs)
    idx_real = np.nonzero(realigned)[0]
    for r in idx_real:  # (realigned reads: a minority; the mapper's paths are copied vectorised below)
        k = int(nseg[r])
        best[int(best_off[r]) : int(best_off[r]) + k] = src_seg[r, :k]
    raw_mask = np.repeat(~realigned, np.diff(rso))
    dst_idx = np.concatenate([np.arange(int(best_off[r]), int(best_off[r + 1])) for r in np.nonzero(~realigned)[0]]) if (~realigned).any() else np.zeros(0, np.int64)
    best[dst_idx] = a["raw_segs"][: int(rso[n])][raw_mask]
    best["kind"] = kind_map[best["kind"]]
    best_pos = np.where(realigned, pos[:n], a["raw_pos"][:n]).astype(np.int32)
    # pile-up in read-buffer order
    hdr = np.zeros(n + 1, dtype=A.PILEUP_READ_DT)
    hdr["seq_off"][:n] = (reg["seq_off"][: w.n_regions].astype(np.int64).repeat(READS_PER_CELL) + np.tile(np.arange(READS_PER_CELL, dtype=np.int64) * ((READ_LEN + 1) // 2), w.n_regions))
    hdr["qual_off"][:n] = np.arange(n, dtype=np.int64) * READ_LEN
    hdr["seg_off"] = best_off
    hdr["pos"][:n], hdr["len"][:n], hdr["mapq"][:n], hdr["flags"][:n] = best_pos, a["read_len"][:n], a["mapq"][:n], a["read_flags"][:n]
    bpos = a["raw_pos"][: n + 1].astype(np.int32).copy()  # (the synthetic mapper alignments carry no clips: buffer position = position)
    shift = int(np.abs(best_pos.astype(np.int64) - bpos[:n]).max(initial=0))
    pb = A.SxPileupReadsBatch(n, int(best_off[n]), A.ptr(hdr), A.ptr(a["seq4"]), A.ptr(w.qual_wide), A.ptr(best), A.ptr(a["ref"]), w.ref_begin, w.used["ref"], w.report_begin,
                              w.report_end, None, 0, READ_LEN + 64, READ_LEN, 0, A.default_pileup_opts())
    pb.buffer_pos, pb.max_pos_shift = A.ptr(bpos), shift
    so, t2o = np.zeros(ns + 1, np.uint32), np.zeros(ns + 1, np.uint32)
    cl, t2c = np.zeros(n * READ_LEN + 16, np.uint16), np.zeros(16, np.uint16)
    sd, sm = np.zeros(ns, np.uint32), np.zeros(ns, np.uint32)
    fnp = rf.ref_pileup_reads_timed
    fnp.argtypes = [C.POINTER(A.SxPileupReadsBatch), _P, _P, C.c_uint64, _P, _P, C.c_uint64, _P, _P, _P, C.c_char_p, C.c_int]
    s_pile = C.c_double(0.0)
    t0 = time.perf_counter()
    rc = fnp(C.byref(pb), A.ptr(so), A.ptr(cl), cl.size, A.ptr(t2o), A.ptr(t2c), t2c.size, A.ptr(sd), A.ptr(sm), C.addressof(s_pile), err, 1024)
    t_pileup = time.perf_counter() - t0
    if rc != 0:
        raise RuntimeError(err.value.decode(errors="replace"))
    # per-site genotyping
    ref_base = a["ref"][w.report_begin - w.ref_begin : w.report_end - w.ref_begin]
    k2 = A.SxPileupBatch(ns, A.ptr(so), A.ptr(cl), None, None, A.ptr(np.ascontiguousarray(ref_base)), None)
    gl = np.zeros(ns, A.DIGT_RESULT_DT)
    params = params or A.default_params()
    s_gl = C.c_double(0.0)
    t0 = time.perf_counter()
    rc = rf.ref_site_gl_germline_timed(C.byref(params), C.byref(k2), 1, _P(gl.ctypes.data), _P(C.addressof(s_gl)), err, 1024)
    t_gl = time.perf_counter() - t0
    if rc != 0:
        raise RuntimeError(err.value.decode(errors="replace"))
    res = {"status": status[:n], "best_pos": best_pos, "best_off": best_off, "best_segs": best[: int(best_off[n])], "recs": recs, "n_rec": n_rec[:n], "site_off": so,
           "calls": cl[: int(so[ns])], "t2_off": t2o, "n_spandel": sd, "n_submapped": sm, "site_gl": gl}
    # seconds inside the reference's own functions (realignAndScoreRead, pileup_read_segment, CleanPileup* + position_snp_call_pprob_digt); the *_call
    # entries are the whole harness calls, object construction included
    return res, {"realign": secs.value, "pileup": s_pile.value, "site_gl": s_gl.value, "realign_call": t_realign_call, "pileup_call": t_pileup, "site_gl_call": t_gl}


def site_gl_items(gl) -> dict:
    """the compared fields of position_snp_call_pprob_digt's results, floats as their bits"""
    it = {f: np.ascontiguousarray(gl[f]) for f in ("ref_gt", "is_computed", "n_used_calls", "phredLoghood")}
    it["lhood"] = np.ascontiguousarray(gl["lhood"]).view(np.uint32)
    for rs in ("genome", "poly"):
        for f in ("max_gt", "snp_qphred", "max_gt_qphred"):
            it[f"{rs}.{f}"] = np.ascontiguousarray(gl[rs][f])
        it[f"{rs}.ref_pprob"] = np.ascontiguousarray(gl[rs]["ref_pprob"]).view(np.uint64)
    return it


def _packed(arr, off, cnt):
    """arr[off[r] : off[r] + cnt[r]] of every r, back to back"""
    n = len(cnt)
    idx = np.concatenate([np.arange(int(off[r]), int(off[r]) + int(cnt[r])) for r in range(n)]) if n else np.zeros(0, np.int64)
    return arr[idx.astype(np.int64)]


def reference_items(w: B.WindowBatch, res: dict) -> dict:
    """reference_pass' results as the items a comparison with the device pass compares (tests/refgold.py)"""
    assert not (res["status"] == 2).any(), "the reference threw on a synthetic read"
    it = {"is_realigned": res["status"] == 1, "best_pos": res["best_pos"], "best_n_seg": np.diff(res["best_off"].astype(np.int64)), "best_segs": res["best_segs"],
          "n_rec": res["n_rec"], "recs": _packed(res["recs"], w.a["rec_off"], res["n_rec"])}
    for name in ("site_off", "calls", "t2_off", "n_spandel", "n_submapped"):
        it[name] = res[name]
    it.update(site_gl_items(res["site_gl"]))
    return it


def window_items(w: B.WindowBatch, d: dict) -> dict:
    """DevWindow.download() of the window as the items reference_items describes (pads of the device's slot layout dropped), after the
    checks that need no reference: no read left to the caller, and the compacted call records are the computed non-reference sites in
    position order, each with its record and depth"""
    n = w.n_reads
    assert not (d["enum_status"] & (A.SX_ENUM_ST_LIMIT | A.SX_ENUM_ST_EXCEPTION)).any(), "reads left to the caller"
    g = d["site_gl"]
    if "variant_sites" in d:
        sel = np.nonzero((g["is_computed"] != 0) & (g["genome"]["max_gt"] != g["ref_gt"]))[0]
        v = d["variant_sites"]
        assert np.array_equal(v["pos"], (w.report_begin + sel).astype(np.int32)), "variant site positions"
        assert v["gl"].tobytes() == g[sel].tobytes(), "variant site records"
        assert np.array_equal(v["n_calls"], np.diff(d["site_off"].astype(np.int64))[sel].astype(np.uint32)), "variant site depths"
    it = {"is_realigned": (d["realign_status"][:n] & A.SX_REALIGN_ST_REALIGNED) != 0, "best_pos": d["best_pos"][:n], "best_n_seg": d["best_n_seg"][:n],
          "best_segs": _packed(d["best_segs"], d["best_seg_off"], d["best_n_seg"][:n]), "n_rec": d["n_rec"][:n], "recs": _packed(d["recs"], w.a["rec_off"], d["n_rec"][:n])}
    for name in ("site_off", "calls", "t2_off", "n_spandel", "n_submapped"):
        it[name] = d[name]
    it.update(site_gl_items(g))
    return it


def window_stats(w: B.WindowBatch, it: dict) -> dict:
    return {"reads": w.n_reads, "realigned": int(it["is_realigned"].sum()), "records": int(np.asarray(it["n_rec"]).sum()), "calls": int(it["site_off"][w.n_sites]),
            "sites": w.n_sites, "variant_sites": int((it["genome.max_gt"] != it["ref_gt"]).sum())}

