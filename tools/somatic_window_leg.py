"""The somatic window pass on cfg2-shaped two-sample windows: sx_process_somatic_window_dev (one call) against the composition it replaces --
two DevWindow passes, sx_site_gl_somatic_dev on their columns, DevSomaticIndelChain on their records, and the SNV / indel records filtered on
the host -- alternating in one process, with the results compared byte for byte.  Prints one JSON line.

    python tools/somatic_window_leg.py [--cells 50000] [--steps 5] [--warmup 2]

The helpers that make a two-sample window out of one (split_window, inject_snvs, somatic_loci, host_records) are also the GPU tests'."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200 import batch as B  # noqa: E402

def _pad16(n: int) -> int:
    return (n + 15) & ~15


def read_offsets(w: B.WindowBatch):
    """each read's byte offset in seq4 and in qual (a region's reads back to back from its seq_off / qual_off), its packed base bytes and its
    quality bytes"""
    a, n = w.a, w.n_reads
    rro = a["region_read_off"].astype(np.int64)
    region = np.repeat(np.arange(w.n_regions), np.diff(rro))
    ln = a["read_len"][:n].astype(np.int64)
    packed = (ln + 1) // 2
    per_q = packed if w.qual_bits == 4 else ln

    def starts(size, base):
        excl = np.concatenate([[0], np.cumsum(size)[:-1]]) if n else np.zeros(0, np.int64)
        return base[region].astype(np.int64) + excl - excl[rro[region]] if n else excl

    return starts(packed, a["regions"]["seq_off"]), starts(per_q, a["regions"]["qual_off"]), packed, per_q


def _csr_count(off, flags, n):
    cs = np.concatenate([[0], np.cumsum(flags.astype(np.int64))])
    o = off.astype(np.int64)
    return cs[o[1 : n + 1]] - cs[o[:n]]


def non_ambig_of(w: B.WindowBatch) -> np.ndarray:
    """each read's count of bases that are not 'N' (code 15), as the window pass's prep computes it for K6"""
    seq, _, packed, _ = read_offsets(w)
    n, ln = w.n_reads, w.a["read_len"][: w.n_reads].astype(np.int64)
    s4 = w.a["seq4"]
    hi, lo = (s4 >> 4) == 15, (s4 & 15) == 15
    cs = np.concatenate([[0], np.cumsum(hi.astype(np.int32) + lo, dtype=np.int64)])
    n_amb = cs[seq + packed] - cs[seq] - ((ln % 2 == 1) & lo[np.maximum(seq + packed - 1, 0)])
    out = np.zeros(n + 1, np.uint16)
    out[:n] = ln - n_amb
    return out


def has_indel(w: B.WindowBatch) -> np.ndarray:
    """reads whose mapper's alignment holds an insertion or a deletion"""
    a = w.a
    return _csr_count(a["raw_seg_off"], np.isin(a["raw_segs"]["kind"], (A.SX_AP_INSERT, A.SX_AP_DELETE)), w.n_reads) > 0


def tumor_mask(w: B.WindowBatch) -> np.ndarray:
    """the reads that go to the tumor sample: every read with an indel in its alignment (tumor-only indel evidence) and every other one of
    the rest"""
    ind = has_indel(w)
    return ind | ((np.cumsum(~ind) % 2 == 0) & ~ind)


def _gather(src_pool, src_start, size, dst_start, dst_len, chunk=1 << 18):
    """a pool of dst_len bytes holding src_pool[src_start[i] : + size[i]] at dst_start[i]"""
    out = np.zeros(dst_len, np.uint8)
    for c in range(0, src_start.size, chunk):
        s, z, d = src_start[c : c + chunk], size[c : c + chunk], dst_start[c : c + chunk]
        tot = int(z.sum())
        within = np.arange(tot) - np.repeat(np.concatenate([[0], np.cumsum(z)[:-1]]), z)
        out[np.repeat(d, z) + within] = src_pool[np.repeat(s, z) + within]
    return out


def split_window(w: B.WindowBatch, keep: np.ndarray) -> B.WindowBatch:
    """the window with only the reads in `keep` (same regions, window entries and reference): each region's read pool repacked (16-byte aligned
    region slices), the per-read arrays and CSR arrays cut, do_site_gl off"""
    a, n, nr = w.a, w.n_reads, w.n_regions
    seq, qual, packed, per_q = read_offsets(w)
    rro = a["region_read_off"].astype(np.int64)
    region = np.repeat(np.arange(nr), np.diff(rro))
    sel = np.nonzero(keep[:n])[0]
    m = sel.size
    reg = a["regions"].copy()
    new_rro = np.concatenate([[0], np.cumsum(np.bincount(region[sel], minlength=nr))]).astype(np.int64)
    pools = {}
    for name, start, size in (("seq", seq, packed), ("qual", qual, per_q)):
        tot = np.bincount(region[sel], weights=size[sel], minlength=nr).astype(np.int64)
        base = np.zeros(nr + 1, np.int64)
        for g in range(nr):
            base[g + 1] = _pad16(int(base[g] + tot[g]))
        base[nr] = int(base[nr - 1] + tot[nr - 1]) if nr else 0
        excl = np.concatenate([[0], np.cumsum(size[sel])[:-1]]) if m else np.zeros(0, np.int64)
        dst = base[region[sel]] + excl - (excl[new_rro[region[sel]]] if m else 0)
        pools[name] = (_gather(a["seq4" if name == "seq" else "qual"], start[sel], size[sel], dst, int(base[nr]) + A.SX_POOL_SLACK), int(base[nr]), base)
    reg["seq_off"][: nr + 1], reg["qual_off"][: nr + 1], reg["read_begin"][: nr + 1] = pools["seq"][2], pools["qual"][2], new_rro
    for f in ("aln_begin", "seg_begin", "ins_begin"):
        reg[f] = 0

    def csr(off, vals):
        o = off.astype(np.int64)
        cnt = o[sel + 1] - o[sel]
        new_off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.uint32)
        within = np.arange(int(cnt.sum())) - np.repeat(new_off[:-1].astype(np.int64), cnt)
        return new_off, np.concatenate([vals[np.repeat(o[sel], cnt) + within], np.zeros(16, vals.dtype)])

    raw_seg_off, raw_segs = csr(a["raw_seg_off"], a["raw_segs"])
    use_key_off, use_keys = csr(a["use_key_off"], a["use_keys"])
    n_win = np.diff(a["region_key_off"].astype(np.int64))
    rec_off = np.concatenate([[0], np.cumsum(np.repeat(n_win, np.diff(new_rro)))]).astype(np.uint32)
    pad = lambda x: np.concatenate([x[sel], np.zeros(8, x.dtype)])
    b = dict(a)
    b.update(region_read_off=new_rro.astype(np.uint32), regions=reg, raw_pos=pad(a["raw_pos"]), raw_seg_off=raw_seg_off, raw_segs=raw_segs, read_len=pad(a["read_len"]),
             read_flags=pad(a["read_flags"]), mapq=pad(a["mapq"]), use_key_off=use_key_off, use_keys=use_keys, rec_off=rec_off, seq4=pools["seq"][0], qual=pools["qual"][0])
    out = B.WindowBatch(b, nr, m, w.n_keys, w.ref_begin, w.report_begin, w.report_end, w.qual_bits, w.qual_dict, w.max_read_len, False,
                        {"seq4": pools["seq"][1], "qual": pools["qual"][1], "ref": w.used["ref"]})
    if getattr(w, "enum_opts", None) is not None:
        out.enum_opts = w.enum_opts
    return out


def inject_snvs(w: B.WindowBatch, every: int, seed: int, frac: float = 0.7) -> np.ndarray:
    """tumor-only SNVs: at every `every`-th position of the report range, `frac` of the reads whose mapper's alignment is one match segment
    over it read the next base instead of the reference's (in place); returns the positions"""
    a, n, rng = w.a, w.n_reads, np.random.default_rng(seed)
    seq, _, _, _ = read_offsets(w)
    positions = np.arange(w.report_begin + every // 2, w.report_end, every, dtype=np.int64)
    off = a["raw_seg_off"].astype(np.int64)
    single = ((off[1 : n + 1] - off[:n]) == 1) & (a["raw_segs"]["kind"][np.minimum(off[:n], max(0, a["raw_segs"].size - 1))] == A.SX_AP_MATCH)
    r = np.nonzero(single)[0]
    p0, ln = a["raw_pos"][r].astype(np.int64), a["read_len"][r].astype(np.int64)
    i0, i1 = np.searchsorted(positions, p0), np.searchsorted(positions, p0 + ln)
    rr = np.repeat(np.arange(r.size), i1 - i0)
    p = positions[np.repeat(i0, i1 - i0) + (np.arange(rr.size) - np.repeat(np.concatenate([[0], np.cumsum(i1 - i0)[:-1]]), i1 - i0))]
    lut = np.zeros(256, np.int64)
    for k, c in enumerate(b"ACGT"):
        lut[c] = k + 1
    refk = lut[a["ref"][p - w.ref_begin]]
    take = (refk > 0) & (rng.random(p.size) < frac)
    rr, p, refk = rr[take], p[take], refk[take]
    alt = np.array([1, 2, 4, 8], np.int64)[refk % 4]  # the next base of A C G T
    i = p - p0[rr]
    at = seq[r[rr]] + (i >> 1)
    sh = np.where(i % 2 == 0, 4, 0)
    v = a["seq4"][at].astype(np.int64)
    a["seq4"][at] = ((v & ~(15 << sh)) | (alt << sh)).astype(np.uint8)
    return positions


def somatic_loci(w: B.WindowBatch, seed: int, n_extra: int = 4):
    """every INDEL entry of the window as a candidate locus (its index is its id in both samples), plus `n_extra` ids no read names (empty
    lists); a few forced, among them extra ones.  Returns (IndelLoci, key_gid)."""
    rng = np.random.default_rng(seed)
    keys = w.a["keys"][: w.n_keys]
    gid = np.nonzero(keys["type"] == A.SX_INDEL_TYPE_INDEL)[0]
    extra = keys[gid[: min(n_extra, gid.size)]].copy() if gid.size else np.zeros(0, A.INDEL_KEY_DT)
    extra["pos"] += 1
    gid_key = np.concatenate([keys, extra])
    gid = np.concatenate([gid, w.n_keys + np.arange(extra.size)]).astype(np.uint32)
    forced = (rng.random(gid.size) < 0.1).astype(np.uint8)
    forced[-extra.size // 2 :] = 1 if extra.size else forced[-extra.size // 2 :]
    err_prob = np.array([1e-4, 5e-4, 2e-3, 1e-2], np.float64)
    err_idx = rng.integers(0, err_prob.size, gid.size).astype(np.uint32)
    loci = B.IndelLoci(gid, gid_key[gid], forced, err_idx, gid_key if gid_key.size else np.zeros(1, A.INDEL_KEY_DT), err_prob)
    return loci, np.arange(w.n_keys, dtype=np.uint32)


def forced_positions(w: B.WindowBatch, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return (rng.random(w.n_sites) < 0.02).astype(np.uint8)


def host_records(site_snv, forced, ref_base, n_depth, t_depth, report_begin, indel, loci, status, read_off):
    """the two record lists by the reference's rules, from per-position and per-locus results (the host filter of the composed route)"""
    keep = ((site_snv["is_computed"] != 0) & (site_snv["qphred"] != 0)) | ((forced != 0) & (ref_base != ord("N")))
    idx = np.nonzero(keep)[0]
    snv = np.zeros(idx.size, A.SOMATIC_SITE_CALL_DT)
    snv["pos"] = report_begin + idx
    snv["n_calls"][:, 0], snv["n_calls"][:, 1] = n_depth[idx], t_depth[idx]
    snv["r"] = site_snv[idx]
    n = loci.n_loci
    ro = read_off.astype(np.int64)
    empty = ro[2 : 2 * n + 1 : 2] == ro[0 : 2 * n : 2]
    kl = (status[:n] != 0) | (loci.is_forced_output != 0) | ((indel["qphred"] != 0) & ~empty)
    li = np.nonzero(kl)[0]
    ind = np.zeros(li.size, A.SOMATIC_INDEL_CALL_DT)
    ind["locus"] = li
    ind["r"] = indel[li]
    return snv, ind


def two_sample_window(w: B.WindowBatch, seed: int):
    """(normal, tumor, loci, key_gid, snv_forced) of one window"""
    mask = tumor_mask(w)
    normal, tumor = split_window(w, ~mask), split_window(w, mask)
    inject_snvs(tumor, 97, seed)
    loci, key_gid = somatic_loci(w, seed)
    return normal, tumor, loci, key_gid, forced_positions(w, seed)


class Composed:
    """the route the one-call pass replaces, on the same inputs"""

    def __init__(self, ctx, normal, tumor, loci, key_gid, forced):
        from strelka_b200 import api

        self.ctx, self.loci, self.forced = ctx, loci, forced
        self.windows = [api.DevWindow(ctx, w) for w in (normal, tumor)]
        for dw in self.windows:
            dw.out.site_gl = None
        self.samples = [api.DevIndelReadsSample.from_window(ctx, dw, key_gid, None, non_ambig_of(w)) for dw, w in zip(self.windows, (normal, tumor))]
        self.chain = api.DevSomaticIndelChain(ctx, self.samples[0], self.samples[1], loci)
        self.link = api.DevIndelLoci(ctx, loci)
        n_sites = normal.n_sites
        self.ref_base = np.ascontiguousarray(normal.a["ref"][normal.report_begin - normal.ref_begin : normal.report_end - normal.ref_begin])
        self.d_ref = api.DeviceArray(ctx, self.ref_base.nbytes + 64).upload(self.ref_base)
        self.d_forced = api.DeviceArray(ctx, forced.nbytes + 64).upload(forced)
        self.snv = api.DeviceArray(ctx, (n_sites + 1) * A.SSNV_RESULT_DT.itemsize)
        self.pb = [A.SxPileupBatch(n_sites=n_sites, site_off=dw.obufs["site_off"].ptr, calls=dw.obufs["calls"].ptr, ref_base=self.d_ref.ptr) for dw in self.windows]
        self.n_sites, self.report_begin = n_sites, normal.report_begin

    def run(self, opts):
        import ctypes as C

        ctx = self.ctx
        for dw in self.windows:
            dw.run()
        ctx._chk(ctx.lib.sx_site_gl_somatic_dev(ctx.h, C.byref(self.pb[0]), C.byref(self.pb[1]), self.d_forced.ptr, self.snv.ptr))
        self.chain.run(opts)

    def results(self, opts):
        """(site_snv, snv records, indel, indel records) with the host filter; the link's status / offsets come from the link entry"""
        ctx, loci = self.ctx, self.loci
        d = [dw.download() for dw in self.windows]
        snv = self.snv.download(A.SSNV_RESULT_DT, self.n_sites)
        indel = self.chain.download()
        cr = sum(int(x["n_rec"].sum()) for x in d) + 1
        linked = ctx.link_indel_reads_dev(self.samples[0], self.samples[1], self.link, cr, min(2 * cr, A.SX_SINDEL_MAX_ALTS * max(1, loci.n_loci)))
        depth = [np.diff(x["site_off"].astype(np.int64)) for x in d]
        rec = host_records(snv, self.forced, self.ref_base, depth[0], depth[1], self.report_begin, indel, loci, linked.status, linked.read_off)
        return d, snv, rec[0], indel, rec[1]

    def free(self):
        for dw in self.windows:
            dw.free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=50_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import window_workload as WW
    from strelka_b200.api import Context, DevSomaticWindow

    t0 = time.time()
    w = WW.make_window(WW.load_synth(), args.cells, args.seed)
    normal, tumor, loci, key_gid, forced = two_sample_window(w, args.seed)
    setup_s = time.time() - t0
    ctx = Context(0)
    opts = A.default_sindel_opts()
    opts.useTier2Evidence = 0
    one = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced, opts=opts)
    comp = Composed(ctx, normal, tumor, loci, key_gid, forced)
    for _ in range(args.warmup):
        one.run()
        comp.run(opts)
    one_ms, comp_ms, stages = [], [], []
    for _ in range(args.steps):
        ctx.timer_mark(0)
        st = one.run()
        ctx.timer_mark(1)
        one_ms.append(ctx.timer_elapsed_ms())
        stages.append(st)
        ctx.timer_mark(0)  # (both routes timed alike: CUDA events on the context's compute stream around the call(s))
        comp.run(opts)
        ctx.timer_mark(1)
        comp_ms.append(ctx.timer_elapsed_ms())
    g = one.download()
    d, snv, snv_rec, indel, indel_rec = comp.results(opts)
    same = {"site_snv": g["site_snv"].tobytes() == snv.tobytes(), "snv_calls": g["snv_calls"].tobytes() == snv_rec.tobytes(),
            "indel": g["indel"].tobytes() == indel.tobytes(), "indel_calls": g["indel_calls"].tobytes() == indel_rec.tobytes()}
    for s, name in enumerate(("normal", "tumor")):
        same[name] = all(np.asarray(g[name][k]).tobytes() == np.asarray(d[s][k]).tobytes() for k in d[s] if k != "totals")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    med = lambda x: float(np.median(x))
    print(json.dumps({"leg": "somatic_window", "cells": args.cells, "reads": [normal.n_reads, tumor.n_reads], "loci": loci.n_loci, "sites": normal.n_sites,
                      "snv_records": int(g["totals"][0]), "indel_records": int(g["totals"][1]),
                      "qss_nonzero": int((g["site_snv"]["qphred"] != 0).sum()), "qsi_nonzero": int((g["indel"]["qphred"] != 0).sum()),
                      "one_call_ms": med(one_ms), "composed_ms": med(comp_ms), "one_call_loci_per_s": loci.n_loci / (med(one_ms) / 1e3),
                      "stage_ms": {k: med([s[k] for s in stages]) for k in A.SX_SWIN_STAGE_NAMES}, "identical": same, "steps": args.steps, "warmup": args.warmup,
                      "setup_s": round(setup_s, 1), "gpu": q[0] if q else "unknown"}))
    one.free()
    comp.free()
    ctx.close()
    if not all(same.values()):
        sys.exit(1)


if __name__ == "__main__":
    main()
