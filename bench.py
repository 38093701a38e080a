#!/usr/bin/env python
"""bench.py -- Strelka2's per-locus hot path on BASELINE.json's cfg2 ("synthetic 30x germline pileup, 150 bp reads, 1M candidate loci").

One "step" = one pass of the WHOLE path over the step's candidate loci, from the mapper's alignments to call records:
    per read    realignAndScoreRead: gates -> candidate-alignment search -> scoreCandidateAlignment of every candidate -> score_indels,
                choice of rseg.realignment                                   (K7g, K7a, K7, K7b, K1, K6, K9)
    per read    pileup_read_segment in read-buffer order                     (K4)
    per site    position_snp_call_pprob_digt, every position (gVCF)         (K2a)
    per region  GlobalAligner haplotype-vs-reference DP for the loci in an active region (half of them, 3 haplotypes each)   (K3)
on ONE description of the data (tools/synth_window.cpp: a contig tiled by candidate loci 300 bp apart, 60 reads of 150 bp per locus = 30x,
mapper-style alignments, 3 candidate alleles per locus), processed window by window (sx_process_window_dev, every intermediate in HBM).
At N GPUs the windows shard across ranks with no data-path collective; each step ends with ONE NCCL gather (variable block sizes) of the
variant-site call records to rank 0 (weak scaling: per-GPU work is fixed).

    python bench.py [--gpus N --steps K --warmup W]            our arm (CUDA, sm_90a)
    python bench.py --impl reference [...]                      the CPU arm: the reference's own functions on the host cores, one process per core
    python bench.py --config cfg2-scoring                       round 1's step (scoring only: K1 + read-max + K2a + K3 on pre-enumerated alignments)

Prints ONE JSON line (see the contract in the task statement): value = candidate loci / s with inputs resident in HBM, e2e = the same through
the C ABI with pinned HOST arrays (H2D + kernels + D2H inside the timed region).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200 import batch as B  # noqa: E402

CONFIGS = {  # the scoring-only step's configurations: name: (n_loci, depth, read_len, n_haps, description)
    "cfg2": (1_000_000, 30, 150, 4, "synthetic 30x germline pileup, 150 bp reads, 1M candidate loci, 4 haplotypes/locus"),
    "cfg5": (10_000, 300, 150, 32, "300x high-depth amplicon, 32 haplotypes/locus (regions of 16 reads)"),
    "tiny": (20_000, 30, 150, 4, "cfg2 shape at 20k loci (plumbing)"),
}
WHOLE_PATH = {  # the whole-path step: name: (candidate loci per GPU, loci per window, description)
    # (50k-locus windows: a context's scratch grows with its window, and the end-to-end leg's four contexts must share an 80 GB card)
    "cfg2": (1_000_000, 50_000, "synthetic 30x germline pileup, 150 bp reads, 1M candidate loci (300 bp apart, 3 candidate alleles each): whole path, mapper alignments in, call records out"),
    "tiny": (20_000, 10_000, "cfg2 shape at 20k loci (plumbing)"),
}


# ----------------------------------------------------------------------------------------------------------------------
# synthetic workload (tools/libsx_synth.so)
# ----------------------------------------------------------------------------------------------------------------------
class SynthSizes(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("n_regions", "n_reads", "n_alns", "n_segs", "seq4_bytes", "qual_bytes", "ref_bytes", "ins_bytes", "cells")]


def run_threads(fns):
    """Run the callables on a thread each; an exception in any of them is re-raised here (a worker that died would otherwise just look fast)."""
    errs = []

    def wrap(f):
        def g():
            try:
                f()
            except BaseException as e:  # noqa: BLE001
                errs.append(e)
        return g

    ths = [threading.Thread(target=wrap(f)) for f in fns]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    if errs:
        raise errs[0]


def _leaves(a: np.ndarray, name: str):
    if a.dtype.names:
        for f in a.dtype.names:
            if f != "pad":
                yield from _leaves(a[f], f"{name}.{f}")
    else:
        yield name, a


def dump_outputs(out_dir: str, tables: dict, max_bytes: int = 60 << 20):
    """tables: name -> array of rows (structured or plain).  Every leaf field goes to out_dir/<name>.<field>.npy as float64 (exact for the
    int32 / uint32 / float32 / float64 fields of the ABI records).  A table whose rows exceed its share of max_bytes is cut to a fixed seeded
    sample of rows, whose indices go to out_dir/<name>.rows.npy."""
    os.makedirs(out_dir, exist_ok=True)
    share = (max_bytes - (64 << 10)) // len(tables)  # (64 KB for the .npy headers)
    for name, a in tables.items():
        leaves = list(_leaves(a, name))
        row_bytes = 8 * (1 + sum(int(np.prod(x.shape[1:])) for _, x in leaves))
        if len(a) * row_bytes > share:
            rows = np.sort(np.random.default_rng(0).choice(len(a), share // row_bytes, replace=False))
            np.save(os.path.join(out_dir, f"{name}.rows.npy"), rows.astype(np.float64))
            leaves = [(k, x[rows]) for k, x in leaves]
        for k, x in leaves:
            np.save(os.path.join(out_dir, f"{k}.npy"), np.ascontiguousarray(x, dtype=np.float64))


def load_synth():
    p = os.path.join(ROOT, "tools", "libsx_synth.so")
    if not os.path.exists(p):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "tools")])
    lib = C.CDLL(p)
    lib.synth_pileups.restype = C.c_uint64
    lib.synth_ga.restype = C.c_uint64
    return lib


class HostAlloc:
    """numpy arrays over pinned host memory (sx_host_alloc) when a CUDA runtime is usable, else plain numpy."""

    def __init__(self, lib, pinned: bool):
        self.lib, self.pinned, self.ptrs = lib, pinned, []

    def array(self, nbytes: int, dtype) -> np.ndarray:
        dt = np.dtype(dtype)
        n = max(1, (nbytes + dt.itemsize - 1) // dt.itemsize)
        if self.pinned:
            p = self.lib.sx_host_alloc(n * dt.itemsize)
            if p:
                self.ptrs.append(p)
                buf = (C.c_char * (n * dt.itemsize)).from_address(p)
                return np.frombuffer(buf, dtype=dt, count=n)
        return np.zeros(n, dtype=dt)

    def free(self):
        for p in self.ptrs:
            self.lib.sx_host_free(p)
        self.ptrs = []


def make_workload(synth, alloc: HostAlloc, n_loci: int, depth: int, read_len: int, n_haps: int, seed: int, threads: int, qual_bits: int = 2, reads_per_region: int = 0,
                  fmt: int = A.SX_FMT_ALN8 | A.SX_FMT_SEG2 | A.SX_FMT_BASEQ | A.SX_FMT_REF4):
    """The K1/K2a/K3 inputs of n_loci candidate loci.  Defaults = the most compact wire formats of include/strelka_b200.h (base and
    2-bit quality code in one nibble, 8-byte alignment headers, 2-byte segments, packed reference windows): the host entry points
    are PCIe-bound, so bytes are throughput."""
    if qual_bits != 2:
        fmt &= ~A.SX_FMT_BASEQ
    rpr = min(reads_per_region, depth) if reads_per_region else depth
    n_regions = n_loci * ((depth + rpr - 1) // rpr)  # a locus deeper than rpr reads is cut into regions sharing its reference window
    regions = alloc.array((n_regions + 1) * A.REGION_DT.itemsize, A.REGION_DT)
    sz = SynthSizes()
    rc = synth.synth_k1_plan(n_loci, depth, read_len, n_haps, C.c_uint64(seed), threads, qual_bits, reads_per_region, fmt, C.c_void_p(regions.ctypes.data), C.byref(sz))
    assert rc == 0, rc
    S = A.SX_POOL_SLACK
    aln_dt = A.ALN8_DT if fmt & A.SX_FMT_ALN8 else A.ALN_DT
    seg_dt = np.dtype(np.uint16) if fmt & A.SX_FMT_SEG2 else A.ALN_SEG_DT
    read_lens = alloc.array(sz.n_reads * 2 + 16, np.uint16)
    seq4 = alloc.array(sz.seq4_bytes + S, np.uint8)
    qual = alloc.array(sz.qual_bytes + S, np.uint8)
    ref = alloc.array(sz.ref_bytes + S, np.uint8)
    alns = alloc.array((sz.n_alns + 3) * aln_dt.itemsize, aln_dt)  # + slack: an sx_aln8 slice is staged from a 16-byte boundary
    segs = alloc.array((sz.n_segs + 16) * seg_dt.itemsize, seg_dt)
    ins = alloc.array(sz.ins_bytes + S, np.uint8)
    rc = synth.synth_k1_fill(n_loci, depth, read_len, n_haps, C.c_uint64(seed), threads, qual_bits, reads_per_region, fmt, C.c_void_p(regions.ctypes.data),
                             C.c_void_p(read_lens.ctypes.data), C.c_void_p(seq4.ctypes.data), C.c_void_p(qual.ctypes.data), C.c_void_p(ref.ctypes.data),
                             C.c_void_p(alns.ctypes.data), C.c_void_p(segs.ctypes.data), C.c_void_p(ins.ctypes.data))
    assert rc == 0, rc
    used = {"seq4": int(sz.seq4_bytes), "qual": int(sz.qual_bytes), "ref": int(sz.ref_bytes), "ins": int(sz.ins_bytes)}
    exc_off = exc = None
    if fmt & A.SX_FMT_BASEQ:  # the generator emits A/C/G/T only: an empty exception list
        exc_off, exc = alloc.array((n_regions + 1) * 4, np.uint32), alloc.array(16, np.uint32)
        exc_off[:] = 0
        exc[:] = 0
    ab = B.AlignBatch(regions[: n_regions + 1], read_lens[: sz.n_reads], seq4, qual, ref, alns[: sz.n_alns + 3], segs, ins, used, qual_bits,
                      [11, 25, 37] if qual_bits in (2, 4) else None, fmt, int(sz.n_segs), int(sz.n_alns),
                      exc_off, exc)
    # K2a: one pileup column per locus
    site_off = alloc.array((n_loci + 1) * 4, np.uint32)
    n_calls = synth.synth_pileups(n_loci, C.c_double(float(depth)), 0, C.c_uint64(seed), threads, C.c_void_p(site_off.ctypes.data), None, None)
    calls = alloc.array(n_calls * 2 + 16, np.uint16)
    ref_base = alloc.array(n_loci, np.uint8)
    synth.synth_pileups(n_loci, C.c_double(float(depth)), 0, C.c_uint64(seed), threads, C.c_void_p(site_off.ctypes.data), C.c_void_p(calls.ctypes.data),
                        C.c_void_p(ref_base.ctypes.data))
    pb = B.PileupBatch.__new__(B.PileupBatch)
    pb.site_off, pb.calls, pb.ref_base, pb.ploidy, pb.t2_off, pb.t2_calls, pb.n_sites = site_off[: n_loci + 1], calls, ref_base[:n_loci], None, None, None, n_loci
    pb.c = A.SxPileupBatch(n_loci, A.ptr(pb.site_off), A.ptr(pb.calls), None, None, A.ptr(pb.ref_base), None)
    # K3: 3 haplotypes for half of the loci
    n_ga = (n_loci // 2) * 3
    q_off = alloc.array((n_ga + 1) * 4, np.uint32)
    r_off = alloc.array((n_ga + 1) * 4, np.uint32)
    tot = synth.synth_ga(n_ga, C.c_uint64(seed), threads, C.c_void_p(q_off.ctypes.data), C.c_void_p(r_off.ctypes.data), None, None)
    qb, rb = tot & 0xFFFFFFFF, tot >> 32
    query = alloc.array(qb + 16, np.uint8)
    gref = alloc.array(rb + 16, np.uint8)
    synth.synth_ga(n_ga, C.c_uint64(seed), threads, C.c_void_p(q_off.ctypes.data), C.c_void_p(r_off.ctypes.data), C.c_void_p(query.ctypes.data), C.c_void_p(gref.ctypes.data))
    gb = B.GaBatch.__new__(B.GaBatch)
    gb.n, gb.query, gb.ref, gb.query_off, gb.ref_off, gb.max_ops = n_ga, query, gref, q_off[: n_ga + 1], r_off[: n_ga + 1], 24
    gb.c = A.SxGaBatch(n_ga, A.ptr(query), A.ptr(gref), A.ptr(gb.query_off), A.ptr(gb.ref_off), gb.max_ops)
    return ab, pb, gb


def make_pileup_reads_workload(n_sites: int, depth: int, read_len: int, seed: int):
    """K4 input: reads over one contig segment in pile-up order (vectorised numpy): 90 % plain matches, 5 % with a 3-base deletion,
    5 % with a 3-base insertion, 0.5 % base errors, qualities {11, 25, 37}, both strands, tier1 mapping."""
    rng = np.random.default_rng(seed)
    L = read_len
    n_reads = n_sites * depth // L
    ref_len = n_sites + 2 * L + 16
    ref_id = rng.integers(0, 4, ref_len, dtype=np.uint8)
    starts = np.sort(rng.integers(0, n_sites + L - 8, n_reads)).astype(np.int64)  # window-relative; report range starts at L
    shape = rng.random(n_reads)
    is_del, is_ins = shape < 0.05, (shape >= 0.05) & (shape < 0.10)
    cut = rng.integers(20, L - 20, n_reads)
    j = np.arange(L, dtype=np.int64)[None, :]
    # reference offset of read base j: deletions skip 3 reference bases after `cut`, insertions hold the reference for 3 read bases
    roff = j + np.where(is_del[:, None] & (j >= cut[:, None]), 3, 0) - np.where(is_ins[:, None], np.clip(j - cut[:, None], 0, 3), 0)
    base = ref_id[np.minimum(starts[:, None] + roff, ref_len - 1)]
    err = rng.random((n_reads, L)) < 0.005
    base = np.where(err, rng.integers(0, 4, (n_reads, L), dtype=np.uint8), base).astype(np.uint8)
    code = (1 << base).astype(np.uint8)
    if L & 1:
        code = np.concatenate([code, np.zeros((n_reads, 1), np.uint8)], axis=1)
    seq4 = ((code[:, 0::2] << 4) | code[:, 1::2]).astype(np.uint8).reshape(-1)
    qual = rng.choice(np.array([11, 25, 37], np.uint8), size=(n_reads, L), p=[0.03, 0.07, 0.90]).reshape(-1)
    n_seg = np.where(is_del | is_ins, 3, 1)
    seg_off = np.concatenate([[0], np.cumsum(n_seg)]).astype(np.uint32)
    segs = np.zeros(int(seg_off[-1]) + 16, dtype=A.ALN_SEG_DT)
    plain = ~(is_del | is_ins)
    segs["len"][seg_off[:-1][plain]] = L
    for mask, kind, tail in ((is_del, A.SX_SEG_DELETE, 0), (is_ins, A.SX_SEG_INSERT, 3)):
        o = seg_off[:-1][mask]
        segs["len"][o], segs["len"][o + 1], segs["len"][o + 2] = cut[mask], 3, L - cut[mask] - tail
        segs["kind"][o + 1] = kind
    hdr = np.zeros(n_reads + 1, dtype=A.PILEUP_READ_DT)
    packed = (L + 1) // 2
    hdr["seq_off"][:-1] = np.arange(n_reads, dtype=np.uint64) * packed
    hdr["qual_off"][:-1] = np.arange(n_reads, dtype=np.uint64) * L
    hdr["seg_off"] = seg_off
    hdr["pos"][:-1] = starts
    hdr["len"][:-1] = L
    hdr["mapq"][:-1] = 60
    hdr["flags"][:-1] = (A.SX_PRF_TIER1 | A.SX_PRF_TIER1OR2) | (rng.random(n_reads) < 0.5).astype(np.uint8)
    hdr[n_reads] = (n_reads * packed, n_reads * L, seg_off[-1], 0, 0, 0, 0)
    ref = np.frombuffer(b"ACGT", dtype=np.uint8)[ref_id]
    return {"reads": hdr, "seq4": np.concatenate([seq4, np.zeros(64, np.uint8)]), "qual": np.concatenate([qual, np.zeros(64, np.uint8)]), "segs": segs,
            "ref": np.concatenate([ref, np.zeros(64, np.uint8)]), "ref_len": ref_len, "n_reads": n_reads, "n_segs": int(seg_off[-1]),
            "report_begin": L, "report_end": L + n_sites, "max_ref_span": L + 3, "bases": n_reads * L}


def k4_pileup_leg(ctx, peak_gbs: float, n_sites: int = 2_000_000, depth: int = 30, read_len: int = 150, reps: int = 5, cpu_reads: int = 20000):
    """SURVEY 8f1 measured beside the headline step (not part of `value`): K4 pileup_reads, inputs and outputs resident in HBM;
    the reference's own pileup_read_segment on one host thread over the first `cpu_reads` reads as the CPU figure."""
    from strelka_b200.api import DeviceArray

    w = make_pileup_reads_workload(n_sites, depth, read_len, 12345)
    dev = {k: DeviceArray(ctx, w[k].nbytes + 64).upload(w[k]) for k in ("reads", "seq4", "qual", "segs", "ref")}
    opts = A.default_pileup_opts()
    bc = A.SxPileupReadsBatch(w["n_reads"], w["n_segs"], dev["reads"].ptr, dev["seq4"].ptr, dev["qual"].ptr, dev["segs"].ptr, dev["ref"].ptr, 0, w["ref_len"],
                              w["report_begin"], w["report_end"], None, 0, w["max_ref_span"], read_len, 0, opts)
    cap = w["bases"] + 16
    out = {"site_off": DeviceArray(ctx, (n_sites + 1) * 4), "t2_off": DeviceArray(ctx, (n_sites + 1) * 4), "n_spandel": DeviceArray(ctx, n_sites * 4),
           "n_submapped": DeviceArray(ctx, n_sites * 4), "calls": DeviceArray(ctx, cap * 2), "t2_calls": DeviceArray(ctx, 64)}
    cols = A.SxPileupColumns(out["site_off"].ptr, out["calls"].ptr, out["t2_off"].ptr, out["t2_calls"].ptr, out["n_spandel"].ptr, out["n_submapped"].ptr, cap, 16)
    ms = []
    for i in range(reps + 2):
        ctx._chk(ctx.lib.sx_pileup_reads_dev(ctx.h, C.byref(bc), C.byref(cols)))
        if i >= 2:
            ms.append(ctx.timing().kernel_ms)
    n_calls = int(out["site_off"].download(np.uint32, n_sites + 1)[-1])
    t = float(np.mean(ms)) * 1e-3
    # algorithmic bytes: every read byte once (packed bases + qualities + header + segments), every call once, the per-site arrays
    alg = w["bases"] * 1.5 + w["n_reads"] * 20 + w["n_segs"] * 4 + n_calls * 2 + n_sites * 16 + w["ref_len"]
    leg = {"what": f"K4 pileup_reads: {n_sites} positions at {depth}x, {read_len} bp reads, resident in HBM", "bases_per_s": w["bases"] / t, "ms": 1e3 * t,
           "calls": n_calls, "roofline": {"bound": "hbm", "achieved": alg / t / 1e9, "peak": peak_gbs, "unit": "GB/s", "frac": alg / t / 1e9 / peak_gbs,
                                          "algorithmic_bytes": int(alg)}}
    # CPU figure: the reference's member function on a prefix of the reads (one thread: the pos processor is not thread safe)
    p = os.path.join(ROOT, "oracle", "_ref", "libstrelka_ref.so")
    if os.path.exists(p):
        rf = C.CDLL(p)
        m = min(cpu_reads, w["n_reads"])
        hdr = w["reads"][: m + 1].copy()
        hdr[m] = (m * ((read_len + 1) // 2), m * read_len, hdr["seg_off"][m], 0, 0, 0, 0)
        hi = int(hdr["pos"][m - 1]) + read_len + 8
        hb = A.SxPileupReadsBatch(m, int(hdr["seg_off"][m]), A.ptr(hdr), A.ptr(w["seq4"]), A.ptr(w["qual"]), A.ptr(w["segs"]), A.ptr(w["ref"]), 0, w["ref_len"],
                                  w["report_begin"], min(hi, w["report_end"]), None, 0, w["max_ref_span"], read_len, 0, opts)
        ns = hb.report_end - hb.report_begin
        so, t2o = np.zeros(ns + 1, np.uint32), np.zeros(ns + 1, np.uint32)
        cl, t2c = np.zeros(m * read_len + 16, np.uint16), np.zeros(16, np.uint16)
        sd, sm = np.zeros(ns, np.uint32), np.zeros(ns, np.uint32)
        err = C.create_string_buffer(512)
        fn = rf.ref_pileup_reads
        fn.argtypes = [C.POINTER(A.SxPileupReadsBatch), C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int]
        t0 = time.perf_counter()
        rc = fn(C.byref(hb), A.ptr(so), A.ptr(cl), cl.size, A.ptr(t2o), A.ptr(t2c), t2c.size, A.ptr(sd), A.ptr(sm), err, 512)
        dt_cpu = time.perf_counter() - t0
        if rc == 0:
            leg["cpu_reference"] = {"bases_per_s": m * read_len / dt_cpu, "cores": 1,
                                    "sample": f"first {m} reads through starling_pos_processor_base::pileup_read_segment (incl. the shim's read construction)"}
    for d in list(dev.values()) + list(out.values()):
        d.free()
    return leg


class SynthK6Sizes(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("n_regions", "n_reads", "n_alns", "n_keys", "n_segs", "n_aln_keys", "n_slots")]


def make_score_indels_workload(synth, n_loci: int, depth: int, read_len: int, n_haps: int, seed: int, threads: int, reads_per_region: int = 0) -> B.ScoreIndelsBatch:
    """The K6 view of the SAME loci make_workload() builds for K1 (same seed -> same reads, alleles and alignment order, so K1's
    lnp[a] is the score of K6's alignment a): per region the window of distinct alt alleles, per alignment its path and indel."""
    rpr = min(reads_per_region, depth) if reads_per_region else depth
    n_regions = n_loci * ((depth + rpr - 1) // rpr)
    counts = np.zeros(3 * n_regions + 3, np.uint32)
    sz = SynthK6Sizes()
    rc = synth.synth_k6_plan(n_loci, depth, read_len, n_haps, C.c_uint64(seed), threads, reads_per_region, C.c_void_p(counts.ctypes.data), C.byref(sz))
    assert rc == 0, rc
    a = {
        "region_read_off": np.zeros(n_regions + 1, np.uint32), "region_key_off": np.zeros(n_regions + 1, np.uint32),
        "keys": np.zeros(sz.n_keys + 1, A.INDEL_KEY_DT), "aln_off": np.zeros(sz.n_reads + 1, np.uint32), "aln_pos": np.zeros(sz.n_alns + 1, np.int32),
        "aln_seg_off": np.zeros(sz.n_alns + 1, np.uint32), "segs": np.zeros(sz.n_segs + 16, A.ALN_SEG_DT), "aln_key_off": np.zeros(sz.n_alns + 1, np.uint32),
        "aln_keys": np.zeros(sz.n_aln_keys + 8, np.uint16), "read_len": np.zeros(sz.n_reads + 8, np.uint16), "non_ambig": np.zeros(sz.n_reads + 8, np.uint16),
        "read_flags": np.zeros(sz.n_reads + 8, np.uint8), "rec_off": np.zeros(sz.n_reads + 1, np.uint32),
    }
    order = ("region_read_off", "region_key_off", "keys", "aln_off", "aln_pos", "aln_seg_off", "segs", "aln_key_off", "aln_keys", "read_len", "non_ambig",
             "read_flags", "rec_off")
    key_ins = np.zeros(32 * (sz.n_keys + 1), np.uint8)  # the insert sequences (test / reference-harness side information)
    rc = synth.synth_k6_fill(n_loci, depth, read_len, n_haps, C.c_uint64(seed), threads, reads_per_region, C.c_void_p(counts.ctypes.data),
                             *[C.c_void_p(a[k].ctypes.data) for k in order], C.c_void_p(key_ins.ctypes.data))
    assert rc == 0, rc
    sb = B.ScoreIndelsBatch.from_arrays(a)
    lens = sb.keys["ins_len"][: sb.n_keys].astype(np.int64)
    sb.ins_off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint32)
    rows = key_ins[: 32 * sb.n_keys].reshape(-1, 32)
    sb.ins_pool = np.concatenate([rows[np.arange(32)[None, :] < lens[:, None]], np.zeros(1, np.uint8)]).astype(np.uint8)
    return sb


def k6_score_indels_leg(ctx, synth, peak_gbs: float, n_loci: int, depth: int, read_len: int, n_haps: int, seed: int, threads: int, rpr: int, lnp_dev=None,
                        reps: int = 5, cpu_regions: int = 3000):
    """SURVEY 8f2 measured beside the headline step (not part of `value`): K6 score_indels on the step's own loci, reading the
    scores K1 left in HBM (`lnp_dev` = DevAlignBatch.out after a K1 pass); inputs and records resident.  CPU figure: the reference's
    own score_indels on one host thread over the first `cpu_regions` regions."""
    from strelka_b200.api import DevScoreIndelsBatch, DeviceArray

    sb = make_score_indels_workload(synth, n_loci, depth, read_len, n_haps, seed, threads, rpr)
    own = None
    if lnp_dev is None:  # stand-alone run (tools/k6_leg.py): synthetic scores with the structure K1 gives (one haplotype fits, the rest do not)
        rng = np.random.default_rng(1)
        lnp = -(rng.integers(0, 4, sb.n_alns + 1) * 30.0 + rng.random(sb.n_alns + 1))
        own = lnp_dev = DeviceArray(ctx, lnp.nbytes).upload(lnp)
    dsb = DevScoreIndelsBatch(ctx, sb)
    ms = []
    for i in range(reps + 2):
        ctx.score_indels_dev(dsb, lnp_dev)
        if i >= 2:
            ms.append(ctx.timing().kernel_ms)
    n_rec = dsb.n_rec.download(np.uint32, sb.n_reads)
    t = float(np.mean(ms)) * 1e-3
    n_records = int(n_rec.sum())
    alg = sb.algorithmic_bytes() + n_records * 32
    leg = {"what": f"K6 score_indels on the step's {n_loci} loci ({sb.n_reads} reads, {sb.n_alns} alignments), scores read where K1 wrote them", "ms": 1e3 * t,
           "reads_per_s": sb.n_reads / t, "loci_per_s": n_loci / t, "records": n_records,
           "roofline": {"bound": "hbm", "achieved": alg / t / 1e9, "peak": peak_gbs, "unit": "GB/s", "frac": alg / t / 1e9 / peak_gbs, "algorithmic_bytes": int(alg)}}
    p = os.path.join(ROOT, "oracle", "_ref", "libstrelka_ref.so")
    if os.path.exists(p) and hasattr(C.CDLL(p), "ref_score_indels_ex"):
        rf = C.CDLL(p)
        m = min(cpu_regions, sb.n_regions)
        n_reads_m, n_alns_m = int(sb.region_read_off[m]), int(sb.aln_off[int(sb.region_read_off[m])])
        sub = A.SxScoreIndelsBatch(m, n_reads_m, n_alns_m, int(sb.region_key_off[m]), *[getattr(sb.c, f) for f, _ in A.SxScoreIndelsBatch._fields_[4:-1]], sb.opts)
        lnp_h = lnp_dev.download(np.float64, n_alns_m + 1)
        pool, ins_off = sb.ins_pool, sb.ins_off
        recs = np.zeros(int(sb.rec_off[n_reads_m]) + 1, A.READ_INDEL_SCORE_DT)
        nr, ma = np.zeros(n_reads_m + 1, np.uint32), np.zeros(n_reads_m + 1, np.uint32)
        err = C.create_string_buffer(512)
        fn = rf.ref_score_indels_ex  # allow_unordered: one alignment per haplotype in haplotype order -> the harness builds the std::set
        fn.argtypes = [C.POINTER(A.SxScoreIndelsBatch)] + [C.c_void_p] * 6 + [C.c_int, C.c_char_p, C.c_int]
        t0 = time.perf_counter()
        rc = fn(C.byref(sub), A.ptr(lnp_h), A.ptr(pool), A.ptr(ins_off), A.ptr(recs), A.ptr(nr), A.ptr(ma), 1, err, 512)
        dt_cpu = time.perf_counter() - t0
        if rc == 0:
            leg["cpu_reference"] = {"reads_per_s": n_reads_m / dt_cpu, "cores": 1,
                                    "sample": f"first {m} regions ({n_reads_m} reads) through the reference's score_indels (incl. the shim's object construction)"}
        else:
            leg["cpu_reference"] = {"error": err.value.decode(errors="replace")}
    for d in list(dsb.bufs.values()) + [dsb.recs, dsb.n_rec, dsb.max_aln, dsb.eval_aln] + ([own] if own else []):
        d.free()
    return leg


def make_enum_workload(n_loci: int, depth: int, read_len: int, seed: int) -> B.EnumBatch:
    """The K7 view of cfg2-shaped loci: per candidate locus a window of three candidate alleles around the locus centre (a deletion
    and an insertion at the same position and a second deletion one base on: overlapping alleles, as alternatives at one locus are),
    `depth` reads that cover it, each with the mapper's plain `read_len`M alignment -- the enumerator finds the alignments that carry
    the alleles.  Built with numpy (no per-read Python)."""
    rng = np.random.default_rng(seed)
    span = 1000
    ref_begin = (np.arange(n_loci, dtype=np.int64) * span + 1000).astype(np.int32)
    centre = ref_begin + 400
    geo = lambda n: np.minimum(rng.geometric(0.4, n), 20).astype(np.uint16)  # noqa: E731  (SURVEY 8d: indel lengths Geom(0.4) capped at 20)
    d0, i1, d2 = geo(n_loci), geo(n_loci), geo(n_loci)
    keys = np.zeros(3 * n_loci + 1, dtype=A.INDEL_KEY_DT)
    k = keys[: 3 * n_loci].reshape(n_loci, 3)
    k["pos"][:, 0], k["pos"][:, 1], k["pos"][:, 2] = centre, centre, centre + 1
    k["del_len"][:, 0], k["del_len"][:, 2] = d0, d2
    k["ins_len"][:, 1] = i1
    k["ins_id"][:, 1] = 1
    k["type"], k["flags"] = A.SX_INDEL_TYPE_INDEL, A.SX_IKF_CANDIDATE
    n_reads = n_loci * depth
    start = (np.repeat(centre, depth) - rng.integers(10, read_len - 10, n_reads)).astype(np.int32)
    eb = B.EnumBatch.__new__(B.EnumBatch)
    eb.opts = A.default_enum_opts()
    eb.n_regions, eb.n_reads, eb.n_keys = n_loci, n_reads, 3 * n_loci
    u32 = lambda a: np.ascontiguousarray(a, dtype=np.uint32)  # noqa: E731
    eb.region_read_off, eb.region_key_off = u32(np.arange(n_loci + 1, dtype=np.int64) * depth), u32(np.arange(n_loci + 1, dtype=np.int64) * 3)
    eb.keys, eb.key_hap, eb.has_hap = keys, np.zeros(1, dtype=A.KEY_HAP_DT), False
    eb.realign_begin, eb.realign_end = ref_begin.copy(), (ref_begin + span - 100).astype(np.int32)
    eb.in_pos = np.concatenate([start, [0]]).astype(np.int32)
    eb.in_seg_off = u32(np.arange(n_reads + 1, dtype=np.int64))
    eb.in_segs = np.zeros(n_reads + 4, dtype=A.ALN_SEG_DT)
    eb.in_segs["len"][:n_reads], eb.in_segs["kind"][:n_reads] = read_len, A.SX_AP_MATCH
    eb.in_key_off = eb.use_key_off = np.zeros(n_reads + 1, np.uint32)
    eb.in_keys = eb.use_keys = np.zeros(4, np.uint16)
    eb.in_lead_key = eb.in_trail_key = np.full(n_reads + 1, A.SX_NO_KEY, np.uint16)
    eb.read_len = np.full(n_reads + 1, read_len, np.uint16)
    # what the reference harness needs to rebuild its objects: all-'A' reference and reads (no mismatch entries in these windows, so
    # the bases never matter), insert sequences of 'C'
    eb.ins_off = np.zeros(3 * n_loci + 1, np.uint32)
    eb.ins_off[1:] = np.cumsum(keys["ins_len"][: 3 * n_loci])
    eb.ins_pool = np.full(int(eb.ins_off[-1]) + 1, ord("C"), np.uint8)
    eb.ref_pool = np.full(n_loci * span + 1, ord("A"), np.uint8)
    eb.ref_off, eb.ref_begin = u32(np.arange(n_loci + 1, dtype=np.int64) * span), np.concatenate([ref_begin, [0]]).astype(np.int32)
    eb.read_pool = np.full(n_reads * read_len + 1, ord("A"), np.uint8)
    eb.read_off = u32(np.arange(n_reads + 1, dtype=np.int64) * read_len)
    eb.c = A.SxEnumBatch(eb.n_regions, eb.n_reads, eb.n_keys, A.ptr(eb.region_read_off), A.ptr(eb.region_key_off), A.ptr(eb.keys), None, A.ptr(eb.realign_begin),
                         A.ptr(eb.realign_end), A.ptr(eb.in_pos), A.ptr(eb.in_seg_off), A.ptr(eb.in_segs), A.ptr(eb.in_key_off), A.ptr(eb.in_keys), A.ptr(eb.use_key_off),
                         A.ptr(eb.use_keys), A.ptr(eb.in_lead_key), A.ptr(eb.in_trail_key), A.ptr(eb.read_len), None, eb.opts)
    return eb


def enum_subbatch(eb: B.EnumBatch, m: int) -> A.SxEnumBatch:
    """the first m regions of eb as an sx_enum_batch (the CSR arrays are prefixes)."""
    return A.SxEnumBatch(m, int(eb.region_read_off[m]), int(eb.region_key_off[m]), *[getattr(eb.c, f) for f, _ in A.SxEnumBatch._fields_[3:-1]], eb.opts)


def k7_enumerate_leg(ctx, peak_gbs: float, n_loci: int = 200_000, depth: int = 30, read_len: int = 150, seed: int = 7, reps: int = 3, cpu_regions: int = 400,
                     fast: bool = False):
    """SURVEY 8a row a3 / 8f3 measured beside the headline step (not part of `value`): K7 enumerate_alignments on cfg2-shaped loci,
    inputs and the CSR it writes resident in HBM.  CPU figure: the reference's own getCandidateAlignments on one host thread over the
    first `cpu_regions` regions (the oracle port where the reference library is absent)."""
    from strelka_b200.api import DevEnumBatch

    eb = make_enum_workload(n_loci, depth, read_len, seed)
    eb.opts.flags = A.SX_ENUM_F_FAST if fast else 0  # (the fast plan is sx_default_enum_opts' default)
    eb.c.opts = eb.opts
    db = DevEnumBatch(ctx, eb, cap_alns=eb.n_reads * 16, cap_segs=eb.n_reads * 64, cap_keys=eb.n_reads * 32)
    ms = []
    for i in range(reps + 1):
        ctx.enumerate_alignments_dev(db)
        if i >= 1:
            ms.append(ctx.timing().kernel_ms)
    totals = db.obufs["totals"].download(np.uint32, 4)
    status = db.obufs["status"].download(np.uint8, eb.n_reads)
    nA, nS, nK = (int(x) for x in totals[:3])
    t = float(np.mean(ms)) * 1e-3
    alg = eb.algorithmic_bytes(nA, nS, nK)
    leg = {"plan": "SX_ENUM_F_FAST (local-memory tier + arena tier, one search, log + gather)" if fast else "original (arena scratch, count / scan / write)",
           "what": f"K7 enumerate_alignments: {n_loci} cfg2-shaped loci ({eb.n_reads} reads, 3 overlapping candidate alleles each) -> {nA} candidate alignments, resident in HBM",
           "ms": 1e3 * t, "reads_per_s": eb.n_reads / t, "loci_per_s": n_loci / t, "alignments_per_s": nA / t, "alignments": nA,
           "reads_flagged": {"max_toggle": int((status & A.SX_ENUM_ST_MAX_TOGGLE != 0).sum()), "exception": int((status & A.SX_ENUM_ST_EXCEPTION != 0).sum()),
                             "limit": int((status & A.SX_ENUM_ST_LIMIT != 0).sum())},
           "roofline": {"bound": "hbm", "achieved": alg / t / 1e9, "peak": peak_gbs, "unit": "GB/s", "frac": alg / t / 1e9 / peak_gbs, "algorithmic_bytes": int(alg)}}
    # parity spot check inside the leg: the first regions against the CPU checker, alignment by alignment
    m = min(cpu_regions, eb.n_regions)
    sub = enum_subbatch(eb, m)
    n_reads_m = int(eb.region_read_off[m])
    host = B.EnumOut(eb, cap_alns=n_reads_m * 64 + 64)
    p = os.path.join(ROOT, "oracle", "_ref", "libstrelka_ref.so")
    err = C.create_string_buffer(512)
    kind = "port"
    t0 = time.perf_counter()
    if os.path.exists(p) and hasattr(C.CDLL(p), "ref_enumerate_alignments"):
        fn = C.CDLL(p).ref_enumerate_alignments
        fn.argtypes = [C.POINTER(A.SxEnumBatch)] + [C.c_void_p] * 7 + [C.POINTER(A.SxEnumOut), C.c_char_p, C.c_int]
        rc = fn(C.byref(sub), A.ptr(eb.ins_pool), A.ptr(eb.ins_off), A.ptr(eb.ref_pool), A.ptr(eb.ref_off), A.ptr(eb.ref_begin), A.ptr(eb.read_pool), A.ptr(eb.read_off),
                C.byref(host.c), err, 512)
        kind = "reference"
    else:
        ox = C.CDLL(os.path.join(ROOT, "oracle", "liboracle.so"))
        ox.ox_enumerate_alignments.argtypes = [C.POINTER(A.SxEnumBatch), C.POINTER(A.SxEnumOut), C.c_int]
        rc = ox.ox_enumerate_alignments(C.byref(sub), C.byref(host.c), 0)
    dt_cpu = time.perf_counter() - t0
    if rc == 0:
        n_m = int(host.totals[0])
        got_off = db.obufs["aln_off"].download(np.uint32, n_reads_m + 1)
        got_pos = db.obufs["aln_pos"].download(np.int32, n_m)
        same = bool(np.array_equal(got_off, host.aln_off[: n_reads_m + 1]) and np.array_equal(got_pos, host.aln_pos[:n_m]))
        leg["cpu_reference"] = {"reads_per_s": n_reads_m / dt_cpu, "cores": 1, "kind": kind, "matches_gpu": same,
                                "sample": f"first {m} regions ({n_reads_m} reads, {n_m} alignments) through "
                                          + ("the reference's getCandidateAlignments (incl. the shim's object construction)" if kind == "reference"
                                             else "oracle/enumerate_oracle.cpp")}
    else:
        leg["cpu_reference"] = {"error": err.value.decode(errors="replace") or f"rc {rc}"}
    for d in list(db.bufs.values()) + list(db.obufs.values()):
        d.free()
    return leg


def make_enum_read_pools(eb: B.EnumBatch, depth: int, read_len: int, seed: int, qual_bits: int = 4) -> B.AlignBatch:
    """The reads, qualities and reference windows of make_enum_workload's loci where K1 keeps them, built with numpy: all-'A' reads on an
    all-'A' reference (the workload's windows hold no mismatch entries), qualities from the cfg2 dictionary {11, 25, 37} -- dictionary-coded
    two per byte (qual_bits 4: K1's byte-entry kernel) or one byte per base (qual_bits 8).  Bases and reference stay in the wide formats K7a reads."""
    rng = np.random.default_rng(seed + 1)
    n_loci, n_reads = eb.n_regions, eb.n_reads
    span = int(eb.ref_off[1] - eb.ref_off[0])
    pad16 = lambda x: (x + 15) & ~15  # noqa: E731
    read_bytes = (read_len + 1) // 2
    per_read_q = read_bytes if qual_bits == 4 else read_len
    seq_stride, qual_stride, ref_stride = pad16(depth * read_bytes), pad16(depth * per_read_q), pad16(span)
    reg = np.zeros(n_loci + 1, dtype=A.REGION_DT)
    g = np.arange(n_loci + 1, dtype=np.int64)
    reg["seq_off"], reg["qual_off"], reg["ref_off"], reg["read_begin"] = g * seq_stride, g * qual_stride, g * ref_stride, g * depth
    reg["ref_begin"][:n_loci], reg["ref_len"][:n_loci] = eb.ref_begin[:n_loci], span
    seq4 = np.full(n_loci * seq_stride + A.SX_POOL_SLACK, 0x11, np.uint8)
    qual = np.zeros(n_loci * qual_stride + A.SX_POOL_SLACK, np.uint8)
    dictionary = np.array([11, 25, 37], np.uint8)
    codes = rng.choice(np.arange(3, dtype=np.uint8), size=(min(n_loci, 512), depth, read_len), p=[0.03, 0.07, 0.90])  # tiled: values, not entropy, matter here
    if qual_bits == 4:  # two codes per byte, high nibble first, every read on a byte boundary -- laid out like seq4
        c = np.concatenate([codes, np.zeros((codes.shape[0], depth, read_len & 1), np.uint8)], axis=2)
        block = ((c[:, :, 0::2] << 4) | c[:, :, 1::2]).reshape(codes.shape[0], depth * read_bytes)
    else:
        block = dictionary[codes].reshape(codes.shape[0], depth * read_len)
    qv = qual[: n_loci * qual_stride].reshape(n_loci, qual_stride)
    for g0 in range(0, n_loci, block.shape[0]):
        qv[g0 : g0 + block.shape[0], : block.shape[1]] = block[: min(block.shape[0], n_loci - g0)]
    ref = np.full(n_loci * ref_stride + A.SX_POOL_SLACK, ord("A"), np.uint8)
    alns = np.zeros(1, dtype=A.ALN_DT)
    alns[0] = (n_reads, 0, 0, 0)
    segs = np.zeros(16, dtype=A.ALN_SEG_DT)
    segs["kind"] = A.SX_SEG_HARDCLIP
    used = {"seq4": n_loci * seq_stride, "qual": n_loci * qual_stride, "ref": n_loci * ref_stride, "ins": 0}
    return B.AlignBatch(reg, eb.read_len[:n_reads].copy(), seq4, qual, ref, alns, segs, np.zeros(A.SX_POOL_SLACK, np.uint8), used, qual_bits=qual_bits,
                        qual_dict=[11, 25, 37] if qual_bits == 4 else None, n_segs=0, n_alns=0)


def realign_chain_leg(ctx, peak_gbs: float, n_loci: int = 100_000, depth: int = 30, read_len: int = 150, seed: int = 7, reps: int = 2, fast: bool = False,
                      check_loci: int = 60):
    """The device-resident chain of realignAndScoreRead measured beside the headline step (not part of `value`): K7a -> K7 -> K7b -> K1 ->
    K6 on cfg2-shaped loci, every intermediate in HBM (strelka_b200.api.DevRealignChain).  A small instance of the same chain is first
    compared, array by array, with the chain run step by step through the CPU oracles."""
    from strelka_b200.api import DevRealignChain

    leg = {"plan": "K7 SX_ENUM_F_FAST" if fast else "K7 original"}
    try:  # parity of a small instance (the oracles and the host flattening are Python-speed)
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from test_chain_plumbing import check_chain

        small = make_enum_workload(check_loci, depth, read_len, seed + 100)
        small.opts.flags = A.SX_ENUM_F_FAST if fast else 0
        small.c.opts = small.opts
        sp = B.read_pools_of(small)
        ch = DevRealignChain(ctx, small, sp, cap_alns_per_read=64)
        ch.run()
        n_alns, n_recs = check_chain(ch, small)
        ch.free()
        leg["parity"] = f"{check_loci} loci ({n_alns} alignments, {n_recs} score_indels records): identical to the oracle chain"
    except AssertionError as e:
        leg["parity"] = f"MISMATCH on the {check_loci}-locus instance: {e}"
    eb = make_enum_workload(n_loci, depth, read_len, seed)
    eb.opts.flags = A.SX_ENUM_F_FAST if fast else 0
    eb.c.opts = eb.opts
    pools = make_enum_read_pools(eb, depth, read_len, seed)
    chain = DevRealignChain(ctx, eb, pools, cap_alns_per_read=16)
    acc = {}
    for i in range(reps + 1):
        ms = chain.run()
        if i >= 1:
            for k, v in ms.items():
                acc[k] = acc.get(k, 0.0) + v / reps
    total = sum(acc.values())
    nA = chain.totals[0]
    n_rec = int(chain.n_rec.download(np.uint32, eb.n_reads).sum())
    leg.update({"what": f"realignAndScoreRead chain K7a -> K7 -> K7b -> K1 -> K6 + K9 on {n_loci} cfg2-shaped loci ({eb.n_reads} reads -> {nA} candidate alignments -> "
                        f"{n_rec} score_indels records), device-resident", "kernel_ms": acc, "ms": total, "loci_per_s": n_loci / max(total * 1e-3, 1e-12),
                "reads_per_s": eb.n_reads / max(total * 1e-3, 1e-12), "alignments": nA})
    chain.free()
    return leg


def workload_cells(ab: B.AlignBatch, gb: B.GaBatch) -> int:
    return ab.cells() + gb.cells()


# ----------------------------------------------------------------------------------------------------------------------
# clocks
# ----------------------------------------------------------------------------------------------------------------------
class ClockSampler:
    Q = "index,clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, gpu_index: int):
        self.gpu, self.samples, self.stop_flag, self.thread = gpu_index, [], False, None

    def _run(self):
        while not self.stop_flag:
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-i", str(self.gpu)], capture_output=True, text=True, timeout=5).stdout
                for line in out.strip().splitlines():
                    f = [x.strip() for x in line.split(",")]
                    self.samples.append((float(f[1]), float(f[2]), f[3:]))
            except Exception:
                pass
            time.sleep(0.2)

    def start(self):
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    def stop(self):
        self.stop_flag = True
        if self.thread:
            self.thread.join(timeout=6)
        if not self.samples:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": []}
        sm = sorted(s[0] for s in self.samples)
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({names[i] for s in self.samples for i, v in enumerate(s[2]) if v.lower().startswith("active")})
        return {"sm_mhz": sm[len(sm) // 2], "sm_max_mhz": self.samples[0][1], "reasons": reasons}


# ----------------------------------------------------------------------------------------------------------------------
# CPU arm (oracle / reference on the host cores)
# ----------------------------------------------------------------------------------------------------------------------
def cpu_pass(ab: B.AlignBatch, pb: B.PileupBatch, gb: B.GaBatch, n_sample_loci: int, threads: int):
    """One pass of the hot path on the first n_sample_loci loci with `threads` host threads (ctypes releases the GIL).
    Uses oracle/liboracle.so (kind "port"): plain scalar C++ of the reference algorithms, same arithmetic, none of the
    reference's container overhead -- a conservative (fast) CPU baseline."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import reflib

    rpl = max(1, ab.n_regions // max(1, pb.n_sites))  # regions per locus (deep loci are cut into several regions)
    n = min(n_sample_loci, pb.n_sites)
    lnp = np.zeros(ab.n_alns, np.float64)
    gout = np.zeros(n, A.DIGT_RESULT_DT)
    n_ga = min(gb.n, (n // 2) * 3)
    gres = np.zeros(max(1, n_ga), A.GA_RESULT_DT)
    gcig = np.zeros((max(1, n_ga), gb.max_ops), np.uint32)
    sc = A.SxGaScores(1, -4, -5, -1, -100, -5, 1, 1)
    params = A.default_params()
    use_ref = reflib.have_ref() and not os.environ.get("SX_BENCH_CPU_PORT")
    busy = [0.0] * threads  # per-thread time inside the scored functions

    if use_ref:
        # kind "reference": the reference's own functions (oracle/_ref/libstrelka_ref.so, compiled from /root/reference).  The shim
        # rebuilds the reference's objects from the flat batch; for K1 only the scoreCandidateAlignment calls are timed.
        rf = reflib.ref()
        _P = C.c_void_p

        def work(t):
            a, b = n * t // threads, n * (t + 1) // threads
            secs = C.c_double(0.0)
            err = C.create_string_buffer(512)
            rc = rf.ref_score_flat_batch(C.byref(ab.c), C.c_uint32(a * rpl), C.c_uint32(b * rpl), _P(lnp.ctypes.data), C.byref(secs), err, 512)
            assert rc == 0, err.value
            t1 = time.perf_counter()
            if b > a:
                sub = A.SxPileupBatch(b - a, pb.site_off.ctypes.data + 4 * a, pb.c.calls, None, None, pb.ref_base.ctypes.data + a, None)
                rc = rf.ref_site_gl_germline(C.byref(params), C.byref(sub), 1, _P(gout.ctypes.data + a * A.DIGT_RESULT_DT.itemsize), err, 512)
                assert rc == 0, err.value
            ga, gbb = n_ga * t // threads, n_ga * (t + 1) // threads
            if gbb > ga:  # offsets are absolute into the pools, so a sub-batch is just a shifted view of the offset arrays
                subg = A.SxGaBatch(gbb - ga, gb.c.query, gb.c.ref, gb.query_off.ctypes.data + 4 * ga, gb.ref_off.ctypes.data + 4 * ga, gb.max_ops)
                rc = rf.ref_global_align(C.byref(sc), C.byref(subg), 0, _P(gres.ctypes.data + 16 * ga), _P(gcig.ctypes.data + 4 * gb.max_ops * ga), err, 512)
                assert rc == 0, err.value
            busy[t] = secs.value + (time.perf_counter() - t1)
    else:
        ox = reflib.oracle()

        def work(t):
            t1 = time.perf_counter()
            a, b = n * t // threads, n * (t + 1) // threads
            ox.ox_score_alignments_range(C.byref(ab.c), a * rpl, b * rpl, lnp.ctypes.data)
            ox.ox_site_gl_germline_range(C.byref(params), C.byref(pb.c), 1, a, b, gout.ctypes.data)
            ga, gbb = n_ga * t // threads, n_ga * (t + 1) // threads
            if gbb > ga:
                sub = A.SxGaBatch(gbb - ga, gb.c.query, gb.c.ref, gb.query_off.ctypes.data + 4 * ga, gb.ref_off.ctypes.data + 4 * ga, gb.max_ops)
                ox.ox_global_align(C.byref(sc), C.byref(sub), gres.ctypes.data + 16 * ga, gcig.ctypes.data + 4 * gb.max_ops * ga)
            busy[t] = time.perf_counter() - t1

    run_threads([(lambda t=t: work(t)) for t in range(threads)])
    # the pass is as long as its slowest thread's time inside the scored functions (threads run concurrently on distinct cores)
    return n, max(busy), ("reference" if use_ref else "port")


def scoring_step_main(args):
    """round 1's step (--config cfg2-scoring / cfg5 / tiny-scoring): K1 + read-max + K2a + K3 on pre-enumerated candidate alignments"""
    assert args.warmup >= 0 and args.steps >= 1

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    cfg_name = args.config.replace("-scoring", "")
    n_loci, depth, read_len, n_haps, desc = CONFIGS[cfg_name]
    rpr = 16 if depth > 64 else 0  # deep loci are cut into regions small enough for the K1 fast path's 60 KB of shared memory
    if args.loci:
        n_loci = args.loci
    ncpu = os.cpu_count() or 8
    threads = max(1, ncpu // max(1, world))
    synth = load_synth()

    # ------------------------------------------------------------------------------------------------------------------
    if args.impl == "reference":
        if rank != 0:
            return
        lib = None
        alloc = HostAlloc(lib, False)
        sample = args.cpu_sample_loci or min(n_loci, max(2000, 600 * ncpu))
        ab, pb, gb = make_workload(synth, alloc, sample, depth, read_len, n_haps, args.seed, ncpu, 2, rpr)
        for _ in range(args.warmup):
            cpu_pass(ab, pb, gb, sample, ncpu)
        t_tot, n_tot = 0.0, 0
        for _ in range(args.steps):
            n, dt, kind = cpu_pass(ab, pb, gb, sample, ncpu)
            t_tot += dt
            n_tot += n
        value = n_tot / t_tot
        cells = workload_cells(ab, gb)
        line = {
            "impl": "reference", "metric": "candidate_loci_per_sec", "value": value, "unit": "loci/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": 1e3 * t_tot / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
            "config": {"workload": f"{args.config}: {desc}", "loci_per_step": sample, "depth": depth, "read_len": read_len, "haplotypes": n_haps,
                       "note": "bounded sample of the workload; throughput is per locus"},
            "gcups": cells * args.steps / t_tot / 1e9,
            "cpu_baseline": {"value": value, "unit": "loci/s", "cores": ncpu, "kind": kind,
                             "sample": f"{sample} loci x {args.steps} passes, {ncpu} host threads, " + ("oracle/_ref/libstrelka_ref.so (the reference's own functions)" if kind == "reference" else "oracle/liboracle.so")},
            "e2e": {"value": value, "unit": "loci/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0,
        }
        print(json.dumps(line))
        return

    # ------------------------------------------------------------------------------------------------------------------
    import torch
    import torch.distributed as dist

    from strelka_b200.api import Context, DevAlignBatch, DevGaBatch, DeviceArray, DevPileupBatch

    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; strelka_b200 has no CPU fallback (use --impl reference for the CPU arm)")
    torch.cuda.set_device(local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    ctx = Context(local_rank)
    lib = ctx.lib
    alloc = HostAlloc(lib, True)
    t_gen = time.perf_counter()
    ab, pb, gb = make_workload(synth, alloc, n_loci, depth, read_len, n_haps, args.seed + 1000 * rank, threads, 2, rpr)
    t_gen = time.perf_counter() - t_gen
    cells_k1, cells_k3 = ab.cells(), gb.cells()
    sc = ctx.active_region_scores()

    # inputs resident in HBM before the timed region
    dab = DevAlignBatch(ctx, ab)
    dpb = DevPileupBatch(ctx, pb)
    dgb = DevGaBatch(ctx, gb)
    d_gl = DeviceArray(ctx, pb.n_sites * A.DIGT_RESULT_DT.itemsize)
    d_max = DeviceArray(ctx, ab.n_reads * 8)
    d_maxa = DeviceArray(ctx, ab.n_reads * 4)
    rec_bytes = pb.n_sites * A.DIGT_RESULT_DT.itemsize
    d_all = DeviceArray(ctx, rec_bytes * world) if (world > 1 and rank == 0) else None
    if world > 1:
        idbuf = torch.zeros(A.SX_NCCL_ID_BYTES, dtype=torch.uint8)
        if rank == 0:
            raw = (C.c_ubyte * A.SX_NCCL_ID_BYTES)()
            ctx._chk(lib.sx_comm_get_unique_id(raw))
            idbuf = torch.tensor(list(raw), dtype=torch.uint8)
        idbuf = idbuf.cuda()
        dist.broadcast(idbuf, 0)
        raw = (C.c_ubyte * A.SX_NCCL_ID_BYTES)(*idbuf.cpu().tolist())
        ctx._chk(lib.sx_comm_init(ctx.h, raw, rank, world))

    k1_ms = []
    parts = {"k1_score": 0.0, "k1_read_max": 0.0, "k2a_germline": 0.0, "k3_global_align": 0.0}

    def step_resident():
        ctx.score_alignments_dev(dab)
        k1_ms.append(ctx.timing().kernel_ms)
        parts["k1_score"] += ctx.timing().kernel_ms
        ctx.read_max_dev(dab, d_max, d_maxa)
        parts["k1_read_max"] += ctx.timing().kernel_ms
        ctx.site_gl_germline_dev(dpb, d_gl, True)
        parts["k2a_germline"] += ctx.timing().kernel_ms
        ctx.global_align_dev(sc, dgb)
        parts["k3_global_align"] += ctx.timing().kernel_ms
        if world > 1:
            ctx._chk(lib.sx_gather_records(ctx.h, d_gl.ptr, rec_bytes, d_all.ptr if d_all else None, 0))

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        ctx.synchronize()

    for _ in range(args.warmup):
        step_resident()
    launches0 = ctx.total_launches()
    k1_ms.clear()
    for k in parts:
        parts[k] = 0.0
    clocks = ClockSampler(local_rank)
    if rank == 0:
        clocks.start()
    barrier()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step_resident()
    barrier()
    dt = time.perf_counter() - t0
    launches = ctx.total_launches() - launches0
    k1_avg_ms = float(np.mean(k1_ms))

    # end to end: pinned host buffers through the C ABI, H2D + kernels + D2H inside the timed region
    e2e = None
    if not args.no_e2e:
        lnp_host = alloc.array(ab.n_alns * 8, np.float64)
        gl_host = alloc.array(pb.n_sites * A.DIGT_RESULT_DT.itemsize, A.DIGT_RESULT_DT)
        ga_res = alloc.array(gb.n * A.GA_RESULT_DT.itemsize, A.GA_RESULT_DT)
        ga_cig = alloc.array(gb.n * gb.max_ops * 4, np.uint32)

        # The three entry points are independent for a batch of loci, so a caller overlaps them: one sx_ctx (own streams) per
        # host thread -- the ABI's threading model (one ctx per GPU and host thread).  The pileup and DP calls then hide under
        # the read/alignment transfer of K1.
        ctx_b, ctx_c = Context(local_rank), Context(local_rank)

        def step_e2e():
            run_threads([lambda: ctx_b.site_gl_germline(pb, True, gl_host),
                         lambda: ctx_c._chk(lib.sx_global_align(ctx_c.h, C.byref(sc), C.byref(gb.c), ga_res.ctypes.data, ga_cig.ctypes.data)),
                         lambda: ctx.score_alignments(ab, lnp_host)])

        for _ in range(min(3, args.warmup)):
            step_e2e()
        barrier()
        t1 = time.perf_counter()
        for _ in range(args.steps):
            step_e2e()
        barrier()
        dt_e2e = time.perf_counter() - t1
        h2d = ab.algorithmic_bytes() - ab.n_alns * 8 + pb.n_calls * 2 + pb.n_sites * 5 + int(gb.query_off[-1]) + int(gb.ref_off[-1]) + (gb.n + 1) * 8
        d2h = ab.n_alns * 8 + pb.n_sites * A.DIGT_RESULT_DT.itemsize + gb.n * (16 + gb.max_ops * 4)
        e2e = (dt_e2e, h2d, d2h)
    clk = clocks.stop() if rank == 0 else None

    # max over ranks
    if world > 1:
        tt = torch.tensor([dt, e2e[0] if e2e else 0.0, k1_avg_ms], dtype=torch.float64, device="cuda")
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        dt, dt_e2e_max, k1_avg_ms = tt.tolist()
        if e2e:
            e2e = (dt_e2e_max, e2e[1], e2e[2])
    if rank == 0:
        peaks = {}
        try:
            peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        except Exception:
            pass
        peak = float(peaks.get("hbm_gbs", 3350.0))
        peak_src = "measured (MEASURED_PEAKS.json hbm_gbs)" if "hbm_gbs" in peaks else "fallback 3350 GB/s (H100 SXM data sheet)"
        total_loci = n_loci * world
        value = total_loci * args.steps / dt
        alg_bytes = ab.algorithmic_bytes()
        achieved = alg_bytes / (k1_avg_ms * 1e-3) / 1e9
        traffic = None  # measured DRAM bytes of the launch: no capture is stored for this card
        line = {
            "metric": "candidate_loci_per_sec", "value": value, "unit": "loci/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
            "config": {"workload": f"{args.config}: {desc}", "loci_per_gpu": n_loci, "depth": depth, "read_len": read_len, "haplotypes": n_haps,
                       "parallelism": f"region-shard x{world}, one NCCL gather of call records per step" if world > 1 else "single GPU",
                       "l2": "inputs (%.1f GB per GPU) far exceed the 50 MB L2; no flush needed" % (alg_bytes / 1e9), "gen_seconds": round(t_gen, 1)},
            "gcups": (cells_k1 + cells_k3) * world * args.steps / dt / 1e9,
            "k1_gcups_kernel_only": cells_k1 / (k1_avg_ms * 1e-3) / 1e9,
            "roofline": {"bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak, "traffic": traffic,
                         "kernel": "k1q_score_kernel (K1 fast path, k1_score4.cu)" if ab.qual_bits in (2, 4) else "k1_score_kernel","algorithmic_bytes_per_launch": alg_bytes, "kernel_ms": k1_avg_ms, "peak_source": peak_src},
            "gpu_launches": launches,
            "kernel_ms_per_step": {k: v / args.steps for k, v in parts.items()},
            "clocks": clk,
        }
        if e2e:
            line["e2e"] = {"value": total_loci * args.steps / e2e[0], "unit": "loci/s", "h2d_bytes_per_step": int(e2e[1]), "d2h_bytes_per_step": int(e2e[2]),
                           "ms_per_step": 1e3 * e2e[0] / args.steps}
        # reported CPU baseline: bounded sample of the same workload on the host cores
        if world == 1:
            sample = args.cpu_sample_loci or min(n_loci, max(2000, 600 * ncpu))
            n, t_cpu, kind = cpu_pass(ab, pb, gb, sample, ncpu)
            line["cpu_baseline"] = {"value": n / t_cpu, "unit": "loci/s", "cores": ncpu, "kind": kind,
                                    "sample": f"first {n} loci of the workload, one pass, {ncpu} host threads, "
                                              + ("oracle/_ref/libstrelka_ref.so (the reference's own functions)" if kind == "reference" else "oracle/liboracle.so")}
            if args.legs and cfg_name != "tiny":
                line["k4_pileup"] = k4_pileup_leg(ctx, peak)
                ctx.score_alignments_dev(dab)  # the scores K6 consumes: K1's own output buffer, never copied out
                line["k6_score_indels"] = k6_score_indels_leg(ctx, synth, peak, n_loci, depth, read_len, n_haps, args.seed + 1000 * rank, threads, rpr, dab.out)
                # K7 had not run on a GPU when this was written: its leg runs in a process of its own with a time limit, so that nothing it
                # does (an exception, a sticky CUDA error, a search that does not end) can take the headline line down with it
                # (the second K7 plan, K7a and the chain have never run on a GPU; the fast plan's own K7 time is kernel_ms["k7_enumerate"] of its chain leg)
                for key, tool, plan in (("k7_enumerate", "k7_leg.py", "original"), ("realign_chain", "chain_leg.py", "original"), ("realign_chain_fast", "chain_leg.py", "fast")):
                    try:
                        r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", tool), "200000" if tool == "k7_leg.py" else "100000", str(min(depth, 30)),
                                            str(read_len), str(peak), plan], capture_output=True, text=True, timeout=180)
                        last = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
                        line[key] = json.loads(last[-1]) if r.returncode == 0 and last else {"error": (r.stderr or r.stdout)[-600:]}
                    except Exception as e:  # noqa: BLE001
                        line[key] = {"error": f"{type(e).__name__}: {e}"}
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


# ----------------------------------------------------------------------------------------------------------------------
# host cores this process may really use
# ----------------------------------------------------------------------------------------------------------------------
def usable_cpus():
    """(count, cpu ids to pin to, how it was found).  os.cpu_count() is the machine's; what a container may use is the smaller of its CPU
    affinity and its cgroup CPU quota (the round-1 CPU arm ran 128 threads under a 16-CPU quota and measured the throttling)."""
    aff = sorted(os.sched_getaffinity(0))
    n, how = len(aff), f"affinity {len(aff)}"
    quota = None
    try:
        q, per = open("/sys/fs/cgroup/cpu.max").read().split()[:2]
        if q != "max":
            quota = float(q) / float(per)
    except Exception:
        try:
            q = int(open("/sys/fs/cgroup/cpu/cpu.cfs_quota_us").read())
            per = int(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
            if q > 0:
                quota = q / per
        except Exception:
            pass
    if quota is not None and quota < n:
        n, how = max(1, int(quota)), f"cgroup cpu quota {quota:g} (affinity {len(aff)}, machine {os.cpu_count()})"
    # one hardware thread per physical core first
    seen, first, rest = set(), [], []
    for c in aff:
        try:
            sib = open(f"/sys/devices/system/cpu/cpu{c}/topology/thread_siblings_list").read().strip()
        except Exception:
            sib = str(c)
        (rest if sib in seen else first).append(c)
        seen.add(sib)
    ids = (first + rest)[:n]
    return n, ids, how


# ----------------------------------------------------------------------------------------------------------------------
# the CPU arm: the reference's own functions, one PROCESS per usable core (its likelihood caches are function-local statics), pinned
# ----------------------------------------------------------------------------------------------------------------------
def reference_worker(args):
    """one worker of the CPU arm: its own window of --worker-loci candidate loci through the reference (tools/window_workload.reference_pass)
    + its share of the haplotype DP problems; prints one JSON line with the seconds of every pass"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import window_workload as WW

    if args.worker_cpu >= 0:
        try:
            os.sched_setaffinity(0, {args.worker_cpu})
        except Exception:
            pass
    synth = WW.load_synth()
    L = args.worker_loci
    w = WW.make_window(synth, L, args.seed, tile=1000 + args.worker_index, qual_bits=8, threads=1, ascii_reads=True)
    n_ga = (L // 2) * 3
    q_off, r_off = np.zeros(n_ga + 1, np.uint32), np.zeros(n_ga + 1, np.uint32)
    tot = synth.synth_ga(n_ga, C.c_uint64(args.seed + args.worker_index), 1, C.c_void_p(q_off.ctypes.data), C.c_void_p(r_off.ctypes.data), None, None)
    query, gref = np.zeros((tot & 0xFFFFFFFF) + 16, np.uint8), np.zeros((tot >> 32) + 16, np.uint8)
    synth.synth_ga(n_ga, C.c_uint64(args.seed + args.worker_index), 1, C.c_void_p(q_off.ctypes.data), C.c_void_p(r_off.ctypes.data), C.c_void_p(query.ctypes.data), C.c_void_p(gref.ctypes.data))
    gb = A.SxGaBatch(n_ga, A.ptr(query), A.ptr(gref), A.ptr(q_off), A.ptr(r_off), 24)
    gres, gcig = np.zeros(max(1, n_ga), A.GA_RESULT_DT), np.zeros((max(1, n_ga), 24), np.uint32)
    sc = A.SxGaScores(1, -4, -5, -1, -100, -5, 1, 1)
    rf = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "libstrelka_ref.so"))
    err = C.create_string_buffer(512)
    passes = []
    for i in range(args.warmup + args.steps):
        res, secs = WW.reference_pass(w)
        t0 = time.perf_counter()
        rc = rf.ref_global_align(C.byref(sc), C.byref(gb), 0, C.c_void_p(gres.ctypes.data), C.c_void_p(gcig.ctypes.data), err, 512)
        assert rc == 0, err.value
        secs["global_align"] = time.perf_counter() - t0
        if i >= args.warmup:
            passes.append(secs)
    print(json.dumps({"worker": args.worker_index, "loci": L, "passes": passes, "realigned": int((res["status"] == 1).sum()), "threw": int((res["status"] == 2).sum())}))


def run_reference_workers(n_workers, cpu_ids, loci, steps, warmup, seed, timeout=900):
    procs = []
    for i in range(n_workers):
        cmd = [sys.executable, os.path.abspath(__file__), "--impl", "reference-worker", "--worker-index", str(i), "--worker-loci", str(loci), "--worker-cpu",
               str(cpu_ids[i % len(cpu_ids)] if cpu_ids else -1), "--steps", str(steps), "--warmup", str(warmup), "--seed", str(seed)]
        procs.append(subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True))  # (stderr: the reference's theta-file warning, once per options object)
    outs = []
    for pr in procs:
        try:
            o, _ = pr.communicate(timeout=timeout)
        except subprocess.TimeoutExpired:
            pr.kill()
            raise SystemExit("bench.py: a reference worker did not finish")
        lines = [ln for ln in o.splitlines() if ln.startswith("{")]
        if pr.returncode != 0 or not lines:
            raise SystemExit(f"bench.py: a reference worker failed (rc {pr.returncode})")
        outs.append(json.loads(lines[-1]))
    return outs


PASS_PARTS = ("realign", "pileup", "site_gl", "global_align")


def summarize_reference(outs, steps):
    """per pass the workers run concurrently on distinct cores: a pass lasts as long as its slowest worker"""
    loci = sum(o["loci"] for o in outs)
    per_pass = [max(sum(o["passes"][k][p] for p in PASS_PARTS) for o in outs) for k in range(steps)]
    per_worker = [sum(sum(o["passes"][k][p] for p in PASS_PARTS) for k in range(steps)) / steps for o in outs]
    t = sum(per_pass)
    parts = {p: float(np.mean([o["passes"][k][p] for o in outs for k in range(steps)])) for p in PASS_PARTS}
    return {"loci_per_pass": loci, "seconds": t, "value": loci * steps / t, "per_core_loci_per_s_median": float(np.median([outs[0]["loci"] / x for x in per_worker])),
            "per_core_loci_per_s_min": float(min(outs[0]["loci"] / x for x in per_worker)), "mean_seconds_per_part": parts, "threw": sum(o["threw"] for o in outs)}


def reference_main(args):
    if int(os.environ.get("RANK", "0")) != 0:
        return
    n_loci, tile_loci, desc = WHOLE_PATH[args.config]
    n, ids, how = usable_cpus()
    L = args.cpu_sample_loci or 240
    outs = run_reference_workers(n, ids, L, args.steps, args.warmup, args.seed)
    r = summarize_reference(outs, args.steps)
    if r["per_core_loci_per_s_median"] < 60:
        raise SystemExit(f"bench.py --impl reference: {r['per_core_loci_per_s_median']:.1f} loci/s per core -- the host cores are oversubscribed or throttled; not a usable baseline")
    line = {
        "impl": "reference", "metric": "candidate_loci_per_sec", "value": r["value"], "unit": "loci/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": 1e3 * r["seconds"] / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
        "config": {"workload": f"{args.config}: {desc}", "loci_per_step": r["loci_per_pass"], "depth": 30, "read_len": 150, "step": "whole path (realignAndScoreRead + pileup_read_segment + "
                   "position_snp_call_pprob_digt at every position + GlobalAligner)", "note": "bounded sample of the workload (one window per core); throughput is per locus"},
        "cpu_baseline": {"value": r["value"], "unit": "loci/s", "cores": n, "kind": "reference", "cores_how": how,
                         "sample": f"{n} processes x {L} loci x {args.steps} passes, each pinned to one core, oracle/_ref/libstrelka_ref.so (the reference's own functions, timed inside the harness: "
                                   "the object construction around them is left out)",
                         "per_core_loci_per_s": {"median": r["per_core_loci_per_s_median"], "min": r["per_core_loci_per_s_min"]}, "mean_seconds_per_part": r["mean_seconds_per_part"]},
        "e2e": {"value": r["value"], "unit": "loci/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line))


# ----------------------------------------------------------------------------------------------------------------------
# our arm: the whole path, window by window
# ----------------------------------------------------------------------------------------------------------------------
def stage_bytes(w, t):
    """algorithmic bytes of every stage of one window (t: its totals): what the stage must read and write at the least, every array once"""
    n, nr, nk, ns = w.n_reads, w.n_regions, w.n_keys, w.n_sites
    nA, nS, nK, k1S, k1I, bestS, calls = (int(x) for x in t[:7])
    qual = w.used["qual"]
    raw = n * (4 + 4) + w.n_raw_segs * 4
    win = nk * A.INDEL_KEY_DT.itemsize + (nr + 1) * 8
    enum_csr = nA * (4 + 4 + 4 + 2 + 2) + nS * 4 + nK * 2 + n * 5
    return {
        "prep": w.used["seq4"] + raw + n * 16,
        "k7g_gates": raw + win + n * 3 + n * 5 + w.n_raw_segs * 4,
        "k7a_keys": w.used["seq4"] + w.used["ref"] + raw + win + n * 10,
        "k7_enumerate": raw + win + n * 12 + enum_csr,
        "k7b_link": enum_csr + win + nA * 16 + k1S * 4 + k1I + nS * 4,
        "k1_score": w.used["seq4"] + qual + w.used["ref"] + nr * 48 + nA * 16 + k1S * 4 + k1I + nA * 8,
        "k6_score_indels": enum_csr + nA * 8 + win + n * 9 + n * 3 * 32 + n * 12,
        "k9_choose": enum_csr + nA * 8 + raw + win + bestS * 4 + n * 15,
        "k4_pileup": w.used["seq4"] + qual + w.used["ref"] + bestS * 4 + n * 24 + calls * 2 + ns * 16,
        "k2a_site_gl": calls * 2 + ns * 5 + ns * A.DIGT_RESULT_DT.itemsize,
    }


def bind_to_gpu_numa(local_rank: int):
    """Run this rank on the host cores of its GPU's NUMA node BEFORE any pinned memory is allocated or touched: the pinned pages then live on
    that node, and the H2D / D2H copies of the end-to-end leg do not cross the socket interconnect (round 1's 8-GPU e2e efficiency was 0.65 with
    unbound generator threads).  Returns a description for the bench line; silently does nothing where the topology is not readable."""
    try:
        import torch

        bus = torch.cuda.get_device_properties(local_rank).pci_bus_id if hasattr(torch.cuda.get_device_properties(local_rank), "pci_bus_id") else None
        dom = getattr(torch.cuda.get_device_properties(local_rank), "pci_domain_id", 0)
        dev = getattr(torch.cuda.get_device_properties(local_rank), "pci_device_id", 0)
        if bus is None:
            return "pci id not available"
        path = f"/sys/bus/pci/devices/{dom:04x}:{bus:02x}:{dev:02x}.0/numa_node"
        node = int(open(path).read())
        if node < 0:
            return "single NUMA node"
        cpus = set()
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.update(range(int(a), int(b or a) + 1))
        allowed = os.sched_getaffinity(0) & cpus
        if allowed:
            os.sched_setaffinity(0, allowed)
            return f"NUMA node {node} ({len(allowed)} cpus)"
        return f"NUMA node {node}: no allowed cpu there"
    except Exception as e:  # noqa: BLE001
        return f"not bound ({type(e).__name__})"


def whole_path_main(args):
    import torch
    import torch.distributed as dist

    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import window_workload as WW
    from strelka_b200.api import Context, DevGaBatch, DeviceArray, DevWindow

    assert args.warmup >= 0 and args.steps >= 1
    rank, local_rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    n_loci, tile_loci, desc = WHOLE_PATH[args.config]
    if args.loci:
        n_loci = args.loci
    tile_loci = min(args.tile_loci or tile_loci, n_loci)
    n_tiles = (n_loci + tile_loci - 1) // tile_loci
    n_loci = n_tiles * tile_loci
    ncpu, cpu_ids, cpu_how = usable_cpus()
    threads = max(1, ncpu // max(1, world))
    if not torch.cuda.is_available():
        raise SystemExit("bench.py: no CUDA device; strelka_b200 has no CPU fallback (use --impl reference for the CPU arm)")
    host_wait = "spin (driver default)"
    if os.environ.get("SX_BLOCKING_WAIT") == "1":  # (A/B knob: blocking waits from the start)
        from strelka_b200 import _abi as _A0
        host_wait = "blocking" if _A0.load().sx_set_host_wait_policy(local_rank, 1) == 0 else "spin (blocking policy refused)"
    torch.cuda.set_device(local_rank)
    numa = bind_to_gpu_numa(local_rank) if world > 1 else "single rank: not bound"
    if world > 1:
        ncpu, cpu_ids, cpu_how = usable_cpus()  # (now the node's)
        threads = max(1, min(threads, ncpu))
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    ctx = Context(local_rank)
    lib = ctx.lib
    synth = WW.load_synth()
    alloc = HostAlloc(lib, True)
    t_gen = time.perf_counter()
    tiles = [WW.make_window(synth, tile_loci, args.seed + 7919 * rank, tile=t, qual_bits=4, threads=threads, alloc=alloc.array) for t in range(n_tiles)]
    # K3: 3 haplotypes for half of the loci
    n_ga = (n_loci // 2) * 3
    q_off, r_off = alloc.array((n_ga + 1) * 4, np.uint32), alloc.array((n_ga + 1) * 4, np.uint32)
    tot = synth.synth_ga(n_ga, C.c_uint64(args.seed + rank), threads, C.c_void_p(q_off.ctypes.data), C.c_void_p(r_off.ctypes.data), None, None)
    query, gref = alloc.array((tot & 0xFFFFFFFF) + 16, np.uint8), alloc.array((tot >> 32) + 16, np.uint8)
    synth.synth_ga(n_ga, C.c_uint64(args.seed + rank), threads, C.c_void_p(q_off.ctypes.data), C.c_void_p(r_off.ctypes.data), C.c_void_p(query.ctypes.data), C.c_void_p(gref.ctypes.data))
    gb = B.GaBatch.__new__(B.GaBatch)
    gb.n, gb.query, gb.ref, gb.query_off, gb.ref_off, gb.max_ops = n_ga, query, gref, q_off[: n_ga + 1], r_off[: n_ga + 1], 24
    gb.c = A.SxGaBatch(n_ga, A.ptr(query), A.ptr(gref), A.ptr(gb.query_off), A.ptr(gb.ref_off), gb.max_ops)
    t_gen = time.perf_counter() - t_gen
    sc = ctx.active_region_scores()

    # inputs resident in HBM before the timed region.  The windows of a step are independent, and no single stage fills the machine (the search
    # is latency-bound, the site model issue-bound), so they are processed on `lanes` contexts -- each with its own stream and buffers, one host
    # thread each -- concurrently; every window's call records land in its own slice of one buffer (slice = the window's capacity), compacted
    # into gather order by one device-to-device copy per window at the end of the step.
    lanes = max(1, min(args.lanes, n_tiles))
    lane_ctx = [ctx] + [Context(local_rank) for _ in range(lanes - 1)]
    dws = [DevWindow(lane_ctx[i % lanes], w, keep_outputs=False) for i, w in enumerate(tiles)]
    dgb = DevGaBatch(ctx, gb)
    cap_each = [d.out.cap_variant_sites for d in dws]
    cap_v = sum(cap_each)
    d_var_raw = DeviceArray(ctx, cap_v * A.SITE_CALL_DT.itemsize)
    d_var = DeviceArray(ctx, cap_v * A.SITE_CALL_DT.itemsize)
    off_each = np.concatenate([[0], np.cumsum(cap_each)])
    for i, d in enumerate(dws):
        d.out.variant_sites = d_var_raw.ptr + int(off_each[i]) * A.SITE_CALL_DT.itemsize
    d_all = DeviceArray(ctx, cap_v * A.SITE_CALL_DT.itemsize * world) if (world > 1 and rank == 0) else None
    if world > 1:
        idbuf = torch.zeros(A.SX_NCCL_ID_BYTES, dtype=torch.uint8)
        if rank == 0:
            raw = (C.c_ubyte * A.SX_NCCL_ID_BYTES)()
            ctx._chk(lib.sx_comm_get_unique_id(raw))
            idbuf = torch.tensor(list(raw), dtype=torch.uint8)
        idbuf = idbuf.cuda()
        dist.broadcast(idbuf, 0)
        raw = (C.c_ubyte * A.SX_NCCL_ID_BYTES)(*idbuf.cpu().tolist())
        ctx._chk(lib.sx_comm_init(ctx.h, raw, rank, world))

    stage_ms = {k: 0.0 for k in A.SX_WIN_STAGE_NAMES + ("k3_global_align",)}
    totals = np.zeros(A.SX_WIN_TOTALS, np.int64)
    gather_off = np.zeros(world + 1, np.uint64)

    lane_ms = [dict() for _ in range(lanes)]

    def lane_work(li):
        acc = lane_ms[li]
        if li and args.lane_offset_ms:  # stagger the contexts so that one's latency-bound stages (K7, K6) run beside the other's issue-bound ones (K2a, K4)
            time.sleep(li * args.lane_offset_ms / 1e3)
        for i in range(li, n_tiles, lanes):
            for k, v in dws[i].run().items():
                acc[k] = acc.get(k, 0.0) + v
        if li == lanes - 1:  # the haplotype DP batch rides on the last lane
            lane_ctx[li].global_align_dev(sc, dgb)
            acc["k3_global_align"] = acc.get("k3_global_align", 0.0) + lane_ctx[li].timing().kernel_ms

    def step_resident():
        if lanes == 1:
            lane_work(0)
        else:
            run_threads([(lambda li=li: lane_work(li)) for li in range(lanes)])
        n_var = 0
        for i, d in enumerate(dws):  # compact the windows' records into one block (gather order = window order)
            nv = int(d.totals[8])
            if nv:
                ctx._chk(lib.sx_memcpy_d2d(ctx.h, d_var.ptr + n_var * A.SITE_CALL_DT.itemsize, d.out.variant_sites, nv * A.SITE_CALL_DT.itemsize))
            totals[:] += d.totals
            n_var += nv
        for li in range(lanes):
            for k, v in lane_ms[li].items():
                stage_ms[k] += v
            lane_ms[li].clear()
        if world > 1:
            ctx._chk(lib.sx_gatherv_records(ctx.h, d_var.ptr, n_var * A.SITE_CALL_DT.itemsize, d_all.ptr if d_all else None, (cap_v * A.SITE_CALL_DT.itemsize * world) if d_all else 0,
                                            gather_off.ctypes.data, 0))
        return n_var

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        ctx.synchronize()

    for _ in range(args.warmup):
        step_resident()
    launches0 = ctx.total_launches()
    for k in stage_ms:
        stage_ms[k] = 0.0
    totals[:] = 0
    clocks = ClockSampler(local_rank)
    if rank == 0:
        clocks.start()
    barrier()
    t0 = time.perf_counter()
    ctx.timer_mark(0)  # CUDA events on the stream the stages are launched on: the timed region is measured on the device
    for _ in range(args.steps):
        n_var_step = step_resident()
    for c in lane_ctx[1:]:  # the other contexts' streams join the timed one: the closing event waits for all of them
        ctx._chk(lib.sx_stream_join(ctx.h, c.h))
    ctx.timer_mark(1)
    dt_dev = ctx.timer_elapsed_ms() / 1e3
    barrier()
    dt_wall = time.perf_counter() - t0
    # one context: every stage, copy and gather of the step is on that stream, so the event time IS the step (the host clock is kept beside it);
    # several contexts: the other streams are not between the marks, so the bracketed host clock is the measure
    dt = dt_dev
    launches = ctx.total_launches() - launches0
    step_totals = totals // args.steps
    if args.dump_outputs and rank == 0:  # what the last timed step handed its caller: the step's variant-site records and the DP results
        ga_res = dgb.res.download(A.GA_RESULT_DT, gb.n)
        ga_cig = dgb.cigar.download(np.uint32, gb.n * gb.max_ops).reshape(gb.n, gb.max_ops)
        ga_cig[np.arange(gb.max_ops)[None, :] >= np.minimum(ga_res["n_ops"], gb.max_ops)[:, None]] = 0  # (slots past a matrix's ops are not written)
        # (several GPUs: the step's records gathered from every rank, rank p's block at byte offset gather_off[p]; the DP results are rank 0's)
        var = d_all.download(A.SITE_CALL_DT, int(gather_off[world]) // A.SITE_CALL_DT.itemsize) if world > 1 else d_var.download(A.SITE_CALL_DT, n_var_step)
        dump_outputs(args.dump_outputs, {"variant_sites": var, "global_align": ga_res, "global_align_cigar": ga_cig})
    # the resident windows give their HBM back before the end-to-end leg: an 80 GB card does not hold both legs' buffers at the default size
    for buf in dws + [d_var_raw, d_var] + ([d_all] if d_all else []) + list(dgb.bufs.values()) + [dgb.res, dgb.cigar]:
        buf.free()

    # end to end: pinned host arrays through the host-array entry, H2D + kernels + D2H inside the timed region.  Two host threads with a context
    # each take the windows alternately (one window's transfers overlap the other's kernels); the DP batch runs on a third.
    e2e = None
    if not args.no_e2e:
        n_workers = max(1, min(args.e2e_workers, n_tiles))
        # the end-to-end leg keeps n_workers + 1 host threads per rank waiting on the device.  Where the ranks together have more waiting threads
        # than the job has CPUs (8 ranks x 4 on the GPU boxes' 16-CPU quota) spinning waiters exhaust the quota and every rank stalls: they block instead
        if host_wait.startswith("spin") and os.environ.get("SX_BLOCKING_WAIT") != "0":
            if lib.sx_set_host_wait_policy(local_rank, 1) == 0:
                host_wait = "spin for the resident step, blocking for the end-to-end leg"
        ctxs = [Context(local_rank) for _ in range(n_workers)]
        ctx_ga = Context(local_rank)
        ga_res, ga_cig = alloc.array(gb.n * A.GA_RESULT_DT.itemsize, A.GA_RESULT_DT), alloc.array(gb.n * gb.max_ops * 4, np.uint32)
        hosts = []
        for wi in range(n_workers):
            w0 = tiles[0]
            n_slots = int(w0.a["rec_off"][w0.n_reads])
            cap1 = w0.n_sites // 8 + 1024
            hosts.append({"recs": alloc.array((n_slots + 1) * A.READ_INDEL_SCORE_DT.itemsize, A.READ_INDEL_SCORE_DT), "n_rec": alloc.array((w0.n_reads + 1) * 4, np.uint32),
                          "var": alloc.array(cap1 * A.SITE_CALL_DT.itemsize, A.SITE_CALL_DT), "cap": cap1, "totals": np.zeros(A.SX_WIN_TOTALS, np.uint32)})
        batches = []
        for w in tiles:  # the host-side structs (host pointers) are built once
            c = A.SxWindowBatch()
            lib.sx_default_window_opts(C.byref(c))
            c.n_regions, c.n_reads, c.n_keys = w.n_regions, w.n_reads, w.n_keys
            for name in B.WindowBatch.ARRAYS:
                if name != "cand_snv":
                    setattr(c, name, A.ptr(w.a[name]) if w.a.get(name) is not None else None)
            c.seq4_bytes, c.qual_bytes, c.ref_bytes = w.used["seq4"], w.used["qual"], w.used["ref"]
            c.qual_bits = w.qual_bits
            c.qual_dict = (C.c_uint8 * 16)(*(w.qual_dict + [0] * (16 - len(w.qual_dict))))
            c.ref_begin, c.report_begin, c.report_end = w.ref_begin, w.report_begin, w.report_end
            c.max_read_len, c.do_site_gl = w.max_read_len, 1
            batches.append(c)
        d2h_step = [0]

        def worker(wi):
            h, cx = hosts[wi], ctxs[wi]
            o = A.SxWindowOut()
            o.recs, o.n_rec, o.variant_sites, o.cap_variant_sites = A.ptr(h["recs"]), A.ptr(h["n_rec"]), A.ptr(h["var"]), h["cap"]
            for ti in range(wi, n_tiles, n_workers):
                cx._chk(lib.sx_process_window(cx.h, C.byref(batches[ti]), C.byref(o), h["totals"].ctypes.data))
                d2h_step[0] += int(tiles[ti].a["rec_off"][tiles[ti].n_reads]) * 32 + tiles[ti].n_reads * 4 + int(h["totals"][8]) * A.SITE_CALL_DT.itemsize

        def step_e2e():
            d2h_step[0] = 0
            run_threads([(lambda wi=wi: worker(wi)) for wi in range(n_workers)] +
                        [lambda: ctx_ga._chk(lib.sx_global_align(ctx_ga.h, C.byref(sc), C.byref(gb.c), ga_res.ctypes.data, ga_cig.ctypes.data))])

        for _ in range(min(3, max(1, args.warmup))):  # (the resident steps before it have warmed the device; these size the workers' buffers)
            step_e2e()
        barrier()
        cpu0 = os.times()
        t1 = time.perf_counter()
        for _ in range(args.steps):
            step_e2e()
        barrier()
        dt_e2e = time.perf_counter() - t1
        cpu1 = os.times()
        e2e_cpu_s = (cpu1.user + cpu1.system - cpu0.user - cpu0.system) / args.steps  # this rank's host CPU seconds per step (spinning waiters show here)
        h2d = sum(WW.input_bytes(w) for w in tiles) + int(gb.query_off[-1]) + int(gb.ref_off[-1]) + (gb.n + 1) * 8
        d2h = d2h_step[0] + gb.n * (16 + gb.max_ops * 4)
        e2e = (dt_e2e, h2d, d2h)
        for c in ctxs + [ctx_ga]:
            c.close()
    clk = clocks.stop() if rank == 0 else None

    if world > 1:
        tt = torch.tensor([dt, e2e[0] if e2e else 0.0], dtype=torch.float64, device="cuda")
        dist.all_reduce(tt, op=dist.ReduceOp.MAX)
        dt, dt_e2e_max = tt.tolist()
        if e2e:
            e2e = (dt_e2e_max, e2e[1], e2e[2])
    if rank == 0:
        peaks = {}
        try:
            peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
        except Exception:
            pass
        peak = float(peaks.get("hbm_gbs", 3350.0))
        peak_src = "measured (MEASURED_PEAKS.json hbm_gbs)" if "hbm_gbs" in peaks else "fallback 3350 GB/s (H100 SXM data sheet)"
        total_loci = n_loci * world
        value = total_loci * args.steps / dt
        per_step = {k: v / args.steps for k, v in stage_ms.items()}
        # per-stage algorithmic bytes of one step (all windows) and the roofline of the stage that takes longest
        sb = {}
        for w in tiles:
            for k, v in stage_bytes(w, step_totals // n_tiles).items():
                sb[k] = sb.get(k, 0) + v
        sb["k3_global_align"] = int(gb.query_off[-1]) + int(gb.ref_off[-1]) + gb.n * (16 + 8)
        stage_roof = {k: {"ms": per_step[k], "algorithmic_bytes": int(sb[k]), "achieved_gbs": sb[k] / max(per_step[k], 1e-9) / 1e6, "frac": sb[k] / max(per_step[k], 1e-9) / 1e6 / peak}
                      for k in per_step if k in sb}
        dom = max((k for k in stage_roof), key=lambda k: per_step[k])
        traffic = None  # measured DRAM bytes of the stage: no capture is stored for this card
        # cell updates of a step: one per base of every candidate alignment scored (scoreCandidateAlignment walks the read once per alignment)
        # + 3 states x Q x R per haplotype DP matrix
        cells_k1 = int(step_totals[0]) * WW.READ_LEN
        cells_k3 = gb.cells()
        whole_bytes = sum(WW.algorithmic_bytes(w, step_totals // n_tiles) for w in tiles)
        line = {
            "metric": "candidate_loci_per_sec", "value": value, "unit": "loci/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": 1e3 * dt / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f64", "data": "synthetic",
            "timing": {"how": "CUDA events on the launching stream around the K steps, max over ranks" if lanes == 1 else
                       f"CUDA events around the K steps on the first of the {lanes} contexts' streams, which the others join before the closing event (sx_stream_join); max over ranks",
                       "device_ms_per_step_rank0": 1e3 * dt_dev / args.steps, "host_clock_ms_per_step_rank0": 1e3 * dt_wall / args.steps},
            "config": {"workload": f"{args.config}: {desc}", "loci_per_gpu": n_loci, "windows_per_gpu": n_tiles, "loci_per_window": tile_loci, "reads_per_locus": WW.READS_PER_CELL,
                       "read_len": WW.READ_LEN, "sites_per_locus": WW.CELL_LEN, "step": "whole path: K7g, K7a, K7, K7b, K1, K6, K9, K4, K2a per window (sx_process_window_dev) + K3",
                       "concurrency": f"{lanes} contexts (own stream + buffers, one host thread each) take the windows in turn; kernel_ms_per_step sums each stage's device time "
                                      "over the contexts, so the stages add up to more than ms_per_step",
                       "parallelism": f"window-shard x{world}, one NCCL gatherv of variant-site records per step" if world > 1 else "single GPU",
                       "l2": "inputs (%.1f GB per GPU) far exceed the 50 MB L2; no flush needed" % (sum(WW.input_bytes(w) for w in tiles) / 1e9), "gen_seconds": round(t_gen, 1), "host_binding": numa, "host_wait": host_wait},
            "roofline": {"bound": "hbm", "achieved": stage_roof[dom]["achieved_gbs"], "peak": peak, "unit": "GB/s", "frac": stage_roof[dom]["frac"], "traffic": traffic,
                         "kernel": f"stage {dom} (the longest of the step)", "algorithmic_bytes_per_step": stage_roof[dom]["algorithmic_bytes"], "kernel_ms_per_step": per_step[dom],
                         "peak_source": peak_src, "whole_step": {"algorithmic_bytes": int(whole_bytes), "achieved_gbs": whole_bytes / (dt / args.steps) / 1e9,
                                                                 "frac": whole_bytes / (dt / args.steps) / 1e9 / peak}},
            "stage_roofline": stage_roof,
            "gpu_launches": launches,
            "gcups": (cells_k1 + cells_k3) * world / (dt / args.steps) / 1e9,
            "gcups_parts": {"k1_score": cells_k1 / max(per_step["k1_score"], 1e-9) / 1e6, "k3_global_align": cells_k3 / max(per_step["k3_global_align"], 1e-9) / 1e6,
                            "cells_per_step_per_gpu": {"k1": cells_k1, "k3": cells_k3},
                            "definition": "k1: candidate alignments x read length (one cell per read base per scored alignment); k3: 3 x Q x R per matrix; "
                                          "gcups = all cells / step time (the step also enumerates, piles up and genotypes), parts = a kernel's cells / its own time"},
            "kernel_ms_per_step": per_step,
            "per_step_totals": {"candidate_alignments": int(step_totals[0]), "k1_segments": int(step_totals[3]), "pileup_calls": int(step_totals[6]), "variant_sites": int(step_totals[8]),
                                "variant_sites_last_step": int(n_var_step)},
            "clocks": clk,
        }
        if e2e:
            line["e2e"] = {"value": total_loci * args.steps / e2e[0], "unit": "loci/s", "h2d_bytes_per_step": int(e2e[1]), "d2h_bytes_per_step": int(e2e[2]),
                           "ms_per_step": 1e3 * e2e[0] / args.steps, "how": f"sx_process_window (host arrays in pinned memory) per window, {n_workers} host threads with a context each; "
                           "sx_global_align on one more; D2H = score_indels records + variant-site records + DP results", "host_cpu_seconds_per_step_rank0": round(e2e_cpu_s, 3),
                           "warmup_steps": min(3, max(1, args.warmup))}
        if world == 1 and not args.no_cpu:
            # the reported CPU baseline: the reference's own functions, one pinned process per usable core, a bounded sample
            try:
                outs = run_reference_workers(ncpu, cpu_ids, args.cpu_sample_loci or 160, 2, 1, args.seed, timeout=600)
                r = summarize_reference(outs, 2)
                line["cpu_baseline"] = {"value": r["value"], "unit": "loci/s", "cores": ncpu, "kind": "reference", "cores_how": cpu_how,
                                        "sample": f"{ncpu} processes x {args.cpu_sample_loci or 160} loci x 2 passes (1 warm-up), one pinned process per core, "
                                                  "oracle/_ref/libstrelka_ref.so (the reference's own realignAndScoreRead, pileup_read_segment, position_snp_call_pprob_digt, GlobalAligner)",
                                        "per_core_loci_per_s": {"median": r["per_core_loci_per_s_median"], "min": r["per_core_loci_per_s_min"]}, "mean_seconds_per_part": r["mean_seconds_per_part"]}
            except SystemExit as e:
                line["cpu_baseline"] = {"error": str(e)}
        if world == 1:
            if args.legs:
                for key, cmd in (("scoring_only_step", [sys.executable, os.path.abspath(__file__), "--config", "cfg2-scoring", "--steps", str(args.steps), "--warmup", str(args.warmup), "--no-legs"]),
                                 ("k2b_somatic_cfg3", [sys.executable, os.path.join(ROOT, "tools", "site_legs.py"), "k2b", str(peak)]),
                                 ("k5_indel_gl", [sys.executable, os.path.join(ROOT, "tools", "site_legs.py"), "k5", str(peak)])):
                    try:
                        r = subprocess.run(cmd, capture_output=True, text=True, timeout=420)
                        last = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
                        line[key] = json.loads(last[-1]) if r.returncode == 0 and last else {"error": (r.stderr or r.stdout)[-600:]}
                    except Exception as e:  # noqa: BLE001
                        line[key] = {"error": f"{type(e).__name__}: {e}"}
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference", "reference-worker"])
    ap.add_argument("--config", default="cfg2", choices=["cfg2", "tiny", "cfg2-scoring", "cfg5", "tiny-scoring"])
    ap.add_argument("--loci", type=int, default=0, help="override the number of candidate loci per GPU")
    ap.add_argument("--tile-loci", type=int, default=0, help="candidate loci per window (whole-path step)")
    ap.add_argument("--e2e-workers", type=int, default=3, help="host threads (one context each) of the end-to-end leg")
    ap.add_argument("--lanes", type=int, default=1, help="contexts that process the windows of a step concurrently (whole-path step)")
    ap.add_argument("--lane-offset-ms", type=float, default=0.0, help="delay of context i's first window in a step: i x this (with --lanes > 1)")
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--no-cpu", action="store_true", help="skip the cpu_baseline leg (tuning runs)")
    ap.add_argument("--no-legs", dest="legs", action="store_false", help="skip the single-kernel legs measured beside the headline step")
    ap.add_argument("--cpu-sample-loci", type=int, default=0)
    ap.add_argument("--worker-index", type=int, default=0)
    ap.add_argument("--worker-loci", type=int, default=240)
    ap.add_argument("--worker-cpu", type=int, default=-1)
    ap.add_argument("--dump-outputs", metavar="DIR", default="",
                    help="after the timed steps, write what the last one computed (the variant-site records gathered from every rank, rank 0's haplotype-DP "
                         "results) as DIR/<table>.<field>.npy, float64, at most 64 MB; a larger table is cut to a fixed seeded sample of rows whose indices go to "
                         "DIR/<table>.rows.npy")
    args = ap.parse_args()
    if args.dump_outputs and (args.config not in WHOLE_PATH or args.impl != "b200"):
        ap.error("--dump-outputs is implemented for the GPU's whole-path step (--config cfg2 / tiny)")
    if args.impl == "reference-worker":
        return reference_worker(args)
    if args.config in ("cfg2-scoring", "cfg5", "tiny-scoring"):
        return scoring_step_main(args)
    if args.impl == "reference":
        return reference_main(args)
    return whole_path_main(args)


if __name__ == "__main__":
    main()
