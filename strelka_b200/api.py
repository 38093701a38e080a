"""Python face of the C ABI (ctypes): what tests and bench.py call.  It adds nothing to the data path -- every method is one
``sx_*`` call on libstrelka_b200.so with numpy (host) buffers or raw device pointers.
"""
from __future__ import annotations

import ctypes as C
from types import SimpleNamespace
from typing import Optional, Tuple

import numpy as np

from . import _abi as A
from . import batch as B


class SxError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"strelka_b200 error {code}: {msg}")
        self.code = code


class DeviceArray:
    """A cudaMalloc'd buffer owned by a Context (freed on close or __del__)."""

    def __init__(self, ctx: "Context", nbytes: int):
        self.ctx = ctx
        self.nbytes = int(nbytes)
        self.ptr = ctx.lib.sx_dev_alloc(ctx.h, max(1, self.nbytes))
        if not self.ptr:
            raise SxError(A.SX_ERR_NOMEM, ctx.last_error())

    def upload(self, a: np.ndarray) -> "DeviceArray":
        a = np.ascontiguousarray(a)
        assert a.nbytes <= self.nbytes
        self.ctx._chk(self.ctx.lib.sx_memcpy_h2d(self.ctx.h, self.ptr, a.ctypes.data, a.nbytes))
        return self

    def download(self, dtype, count: int) -> np.ndarray:
        out = np.empty(count, dtype=dtype)
        self.ctx._chk(self.ctx.lib.sx_memcpy_d2h(self.ctx.h, out.ctypes.data, self.ptr, out.nbytes))
        return out

    def free(self):
        if self.ptr and self.ctx.h:
            self.ctx.lib.sx_dev_free(self.ctx.h, self.ptr)
        self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _device_twin(ctx: "Context", host: C.Structure, owner, slack: int, adopt: Optional[dict] = None):
    """The device twin of ABI struct `host`: a copy whose every non-NULL pointer field points at `adopt[field]` where given, else at an
    upload of the owner's array of the field's name into a buffer `slack` bytes longer.  NULL fields stay NULL.  Returns (struct,
    {field: DeviceArray})."""
    c = type(host).from_buffer_copy(host)
    bufs = {}
    for name, typ in type(host)._fields_:
        if typ is not C.c_void_p or not getattr(host, name):
            continue
        if adopt and name in adopt:
            setattr(c, name, adopt[name])
            continue
        arr = getattr(owner, name, None)
        if arr is None:
            raise ValueError(f"{type(host).__name__}.{name} is set on the host, but {type(owner).__name__} has no array of that name to upload")
        bufs[name] = DeviceArray(ctx, arr.nbytes + slack).upload(arr)
        setattr(c, name, bufs[name].ptr)
    return c, bufs


class DevAlignBatch:
    """sx_align_batch whose pools live in HBM (inputs resident before the timed region)."""

    def __init__(self, ctx: "Context", hb: B.AlignBatch):
        self.host = hb
        self.c, self.bufs = _device_twin(ctx, hb.c, hb, 64)
        self.out = DeviceArray(ctx, hb.n_alns * 8)


class DevPileupBatch:
    def __init__(self, ctx: "Context", hb: B.PileupBatch):
        self.host = hb
        self.c, self.bufs = _device_twin(ctx, hb.c, hb, 64)


class DevGaBatch:
    def __init__(self, ctx: "Context", hb: B.GaBatch):
        self.host = hb
        self.c, self.bufs = _device_twin(ctx, hb.c, hb, 64)
        self.res = DeviceArray(ctx, hb.n * A.GA_RESULT_DT.itemsize)
        self.cigar = DeviceArray(ctx, hb.n * hb.max_ops * 4 + 16)


class Context:
    """One sx_ctx (one GPU, one host thread)."""

    def __init__(self, device: int = 0, params: Optional[A.SxParams] = None):
        self.lib = A.load()
        self.params = params or A.default_params()
        h = C.c_void_p()
        rc = self.lib.sx_create(device, C.byref(self.params), C.byref(h))
        if rc != 0:
            raise SxError(rc, (self.lib.sx_last_error(None) or b"").decode())
        self.h = h
        self.device = device

    def close(self):
        if getattr(self, "h", None):
            self.lib.sx_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def last_error(self) -> str:
        return (self.lib.sx_last_error(self.h) or b"").decode()

    def _chk(self, rc: int):
        if rc != 0:
            raise SxError(rc, self.last_error())

    def timing(self) -> A.SxTiming:
        t = A.SxTiming()
        self.lib.sx_last_timing(self.h, C.byref(t))
        return t

    def total_launches(self) -> int:
        return int(self.lib.sx_total_launches(self.h))

    def timer_mark(self, which: int) -> None:
        """Record a CUDA event on this context's compute stream (0 = start, 1 = stop)."""
        self._chk(self.lib.sx_timer_mark(self.h, int(which)))

    def timer_elapsed_ms(self) -> float:
        """Device time between the two marks (waits for mark 1)."""
        ms = C.c_double(0.0)
        self._chk(self.lib.sx_timer_elapsed_ms(self.h, C.byref(ms)))
        return ms.value

    def synchronize(self):
        self._chk(self.lib.sx_synchronize(self.h))

    # ---- K1
    def score_alignments(self, batch: B.AlignBatch, out: Optional[np.ndarray] = None) -> np.ndarray:
        if out is None:
            out = np.zeros(batch.n_alns, np.float64)
        self._chk(self.lib.sx_score_alignments(self.h, C.byref(batch.c), out.ctypes.data))
        return out

    def score_alignments_dev(self, db: DevAlignBatch) -> None:
        self._chk(self.lib.sx_score_alignments_dev(self.h, C.byref(db.c), db.out.ptr))

    def read_max_dev(self, db: DevAlignBatch, max_lnp: DeviceArray, max_aln: DeviceArray) -> None:
        self._chk(self.lib.sx_read_max_dev(self.h, C.byref(db.c), db.out.ptr, max_lnp.ptr, max_aln.ptr))

    # ---- K3
    def global_align(self, scores: A.SxGaScores, gb: B.GaBatch) -> Tuple[np.ndarray, np.ndarray]:
        res = np.zeros(gb.n, A.GA_RESULT_DT)
        cig = np.zeros((gb.n, gb.max_ops), np.uint32)
        self._chk(self.lib.sx_global_align(self.h, C.byref(scores), C.byref(gb.c), res.ctypes.data, cig.ctypes.data))
        return res, cig

    def global_align_dev(self, scores: A.SxGaScores, db: DevGaBatch) -> None:
        self._chk(self.lib.sx_global_align_dev(self.h, C.byref(scores), C.byref(db.c), db.res.ptr, db.cigar.ptr))

    def active_region_scores(self) -> A.SxGaScores:
        s = A.SxGaScores()
        self.lib.sx_ga_active_region_scores(C.byref(s))
        return s

    # ---- K2a
    def site_gl_germline(self, pb: B.PileupBatch, is_always_test: bool = True, out: Optional[np.ndarray] = None) -> np.ndarray:
        if out is None:
            out = np.zeros(pb.n_sites, A.DIGT_RESULT_DT)
        self._chk(self.lib.sx_site_gl_germline(self.h, C.byref(pb.c), int(is_always_test), out.ctypes.data))
        return out

    def site_gl_germline_dev(self, db: DevPileupBatch, out: DeviceArray, is_always_test: bool = True) -> None:
        self._chk(self.lib.sx_site_gl_germline_dev(self.h, C.byref(db.c), int(is_always_test), out.ptr))

    def dependent_eprob(self, pb: B.PileupBatch) -> Tuple[np.ndarray, np.ndarray]:
        off = np.zeros(pb.n_sites + 1, np.uint32)
        de = np.zeros(max(1, pb.n_calls), np.float32)
        self._chk(self.lib.sx_dependent_eprob(self.h, C.byref(pb.c), off.ctypes.data, de.ctypes.data))
        return off, de[: off[-1]]

    # ---- K2b
    def site_gl_somatic(self, npb: B.PileupBatch, tpb: B.PileupBatch, forced: Optional[np.ndarray] = None, out: Optional[np.ndarray] = None) -> np.ndarray:
        if out is None:
            out = np.zeros(npb.n_sites, A.SSNV_RESULT_DT)
        f = None if forced is None else np.ascontiguousarray(forced, np.uint8)
        self._chk(self.lib.sx_site_gl_somatic(self.h, C.byref(npb.c), C.byref(tpb.c), A.ptr(f), out.ctypes.data))
        return out

    def site_gl_somatic_dev(self, dn: DevPileupBatch, dt: DevPileupBatch, forced: Optional[DeviceArray], out: DeviceArray) -> None:
        self._chk(self.lib.sx_site_gl_somatic_dev(self.h, C.byref(dn.c), C.byref(dt.c), forced.ptr if forced else None, out.ptr))

    # ---- K5
    def indel_gl(self, ib: "B.IndelBatch", out=None) -> np.ndarray:
        if out is None:
            out = np.zeros(ib.n_loci, A.INDEL_RESULT_DT)
        self._chk(self.lib.sx_indel_gl(self.h, C.byref(ib.c), out.ctypes.data))
        return out

    # ---- K5b
    def somatic_indel(self, sb: "B.SomaticIndelBatch", opts: Optional[A.SxSindelOpts] = None, out=None) -> np.ndarray:
        """K5b: get_somatic_indel of every locus (host arrays in, sx_sindel_result records out)."""
        if out is None:
            out = np.zeros(sb.n_loci, A.SINDEL_RESULT_DT)
        o = opts or A.default_sindel_opts()
        self._chk(self.lib.sx_somatic_indel(self.h, C.byref(o), C.byref(sb.c), A.ptr(sb.err_prob), sb.err_prob.size, out.ctypes.data))
        return out

    def somatic_indel_dev(self, db: DevSomaticIndelBatch, opts: Optional[A.SxSindelOpts] = None) -> None:
        o = opts or A.default_sindel_opts()
        hb = db.host
        self._chk(self.lib.sx_somatic_indel_dev(self.h, C.byref(o), C.byref(db.c), A.ptr(hb.err_prob), hb.err_prob.size, db.out.ptr))

    # ---- K4
    def pileup_reads(self, pb: B.PileupReadsBatch):
        """K4: per-position base_call columns of a read batch (host buffers in, host columns out)."""
        out = B.PileupColumns(pb)
        self._chk(self.lib.sx_pileup_reads(self.h, C.byref(pb.c), C.byref(out.c)))
        return out.trimmed()

    # ---- K6
    def score_indels(self, sb: B.ScoreIndelsBatch, lnp: np.ndarray):
        """K6: the arg-max epilogue of scoreCandidateAlignments + score_indels (host buffers in, host records out).
        Returns (records in key order per read, n_rec[n_reads], max_aln[n_reads], eval_aln[n_reads])."""
        lnp = np.ascontiguousarray(lnp, dtype=np.float64)
        assert lnp.size >= sb.n_alns
        out = B.ScoreIndelsOut(sb)
        self._chk(self.lib.sx_score_indels(self.h, C.byref(sb.c), lnp.ctypes.data, C.byref(out.c)))
        return out.compact()

    def score_indels_dev(self, db: DevScoreIndelsBatch, lnp_dev: DeviceArray) -> None:
        self._chk(self.lib.sx_score_indels_dev(self.h, C.byref(db.c), lnp_dev.ptr, C.byref(db.out)))

    # ---- K6b
    def link_indel_reads(self, normal: B.IndelReadsSample, tumor: B.IndelReadsSample, loci: B.IndelLoci, cap_reads=None, cap_alts=None) -> B.IndelReadsOut:
        """K6b: two samples' K6 records -> K5b's per-locus read lists (host arrays in and out).  SX_ERR_CAPACITY leaves the needed sizes in
        the SxError's `totals`."""
        cr, ca = self._link_caps(normal, tumor, loci.n_loci)
        out = B.IndelReadsOut(loci.n_loci, cr if cap_reads is None else cap_reads, ca if cap_alts is None else cap_alts)
        totals = np.zeros(2, np.uint32)
        rc = self.lib.sx_link_indel_reads(self.h, C.byref(normal.c), C.byref(tumor.c), C.byref(loci.c), C.byref(out.c), totals.ctypes.data)
        self._chk_totals(rc, totals)
        return out

    @staticmethod
    def _link_caps(normal, tumor, n_loci: int) -> Tuple[int, int]:
        """Capacities no batch exceeds: an entry per record, two alternates per entry and SX_SINDEL_MAX_ALTS per locus."""
        cap_reads = sum(int(np.asarray(s.n_rec[: s.n_reads], np.int64).sum()) for s in (normal, tumor))
        return cap_reads, min(2 * cap_reads, A.SX_SINDEL_MAX_ALTS * n_loci)

    def link_indel_reads_dev(self, normal: DevIndelReadsSample, tumor: DevIndelReadsSample, loci: DevIndelLoci, cap_reads: int, cap_alts: int) -> B.IndelReadsOut:
        """K6b on device-resident inputs, into device arrays of the given capacities; returns their host copies."""
        n = loci.host.n_loci
        out = B.IndelReadsOut(n, cap_reads, cap_alts)
        d = {k: DeviceArray(self, getattr(out, k).nbytes + 64) for k in ("alt_off", "alts", "read_off", "reads", "status", "totals")}
        c = A.SxIndelReadsOut(cap_alts=cap_alts, cap_reads=cap_reads, **{k: x.ptr for k, x in d.items()})
        totals = np.zeros(2, np.uint32)
        rc = self.lib.sx_link_indel_reads_dev(self.h, C.byref(normal.c), C.byref(tumor.c), C.byref(loci.c), C.byref(c), totals.ctypes.data)
        self._chk_totals(rc, totals)
        for k in ("alt_off", "read_off", "totals"):
            getattr(out, k)[:] = d[k].download(np.uint32, getattr(out, k).size)
        out.status[:n] = d["status"].download(np.uint32, n)
        out.reads[: int(out.totals[0])] = d["reads"].download(A.SINDEL_READ_DT, int(out.totals[0]))
        out.alts[: int(out.totals[1])] = d["alts"].download(A.INDEL_KEY_DT, int(out.totals[1]))
        for x in d.values():
            x.free()
        return out

    # ---- K6g
    def link_allele_groups(self, sample: B.IndelReadsSample, groups: B.AlleleGroups, cap_reads=None, cap_lnp=None) -> B.AlleleGroupReadsOut:
        """K6g: one sample's K6 records -> K5's per-group read lists (host arrays in and out).  SX_ERR_CAPACITY leaves the needed sizes in
        the SxError's `totals`."""
        cr, cl = B.allele_group_caps(sample, groups)
        out = B.AlleleGroupReadsOut(groups.n_groups, int(groups.allele_off[-1]), cr if cap_reads is None else cap_reads, cl if cap_lnp is None else cap_lnp)
        totals = np.zeros(2, np.uint32)
        rc = self.lib.sx_link_allele_groups(self.h, C.byref(sample.c), C.byref(groups.c), C.byref(out.c), totals.ctypes.data)
        self._chk_totals(rc, totals)
        return out

    def link_allele_groups_dev(self, sample: DevIndelReadsSample, groups: DevAlleleGroups, cap_reads: int, cap_lnp: int) -> B.AlleleGroupReadsOut:
        """K6g on device-resident inputs, into device arrays of the given capacities; returns their host copies."""
        hg = groups.host
        out = B.AlleleGroupReadsOut(hg.n_groups, int(hg.allele_off[-1]), cap_reads, cap_lnp)
        d = {k: DeviceArray(self, getattr(out, k).nbytes + 64) for k in out.ARRAYS}
        c = A.SxAlleleGroupReadsOut(cap_reads=cap_reads, cap_lnp=cap_lnp, **{k: x.ptr for k, x in d.items()})
        totals = np.zeros(2, np.uint32)
        rc = self.lib.sx_link_allele_groups_dev(self.h, C.byref(sample.c), C.byref(groups.c), C.byref(c), totals.ctypes.data)
        self._chk_totals(rc, totals)
        n, r, f, a = hg.n_groups, int(totals[0]), int(totals[1]), int(hg.allele_off[-1])
        for k, cnt in (("read_off", n + 1), ("lnp_off", n + 1), ("allele_off", n + 1), ("totals", 2), ("status", n), ("ploidy", n), ("allele_del_len", a),
                       ("allele_ins_len", a), ("allele_lnp", f), ("read_length", r), ("non_ambig", r), ("is_fwd", r)):
            arr = getattr(out, k)
            arr[:cnt] = d[k].download(arr.dtype, cnt)
        for x in d.values():
            x.free()
        return out

    def _chk_totals(self, rc: int, totals: np.ndarray) -> None:
        try:
            self._chk(rc)
        except SxError as e:
            e.totals = totals.copy()
            raise

    # ---- K7
    def enumerate_alignments(self, eb: B.EnumBatch, cap_alns=None, cap_segs=None, cap_keys=None) -> B.EnumOut:
        """K7: the candidate alignments of every read (getCandidateAlignments), host buffers in, host CSR out."""
        out = B.EnumOut(eb, cap_alns, cap_segs, cap_keys)
        self._chk(self.lib.sx_enumerate_alignments(self.h, C.byref(eb.c), C.byref(out.c)))
        return out

    def enumerate_alignments_dev(self, db: DevEnumBatch) -> None:
        self._chk(self.lib.sx_enumerate_alignments_dev(self.h, C.byref(db.c), C.byref(db.out)))

    # ---- K7b
    def link_alignments(self, eb: B.EnumBatch, out: B.EnumOut, regions: np.ndarray, cap_segs=None, cap_ins=None) -> B.LinkOut:
        """K7b: K7's alignments as the alignment part of a K1 batch (host buffers).  `regions`: the K1 batch's region records."""
        n_alns = int(out.totals[0])
        lo = B.LinkOut(regions, n_alns, cap_segs if cap_segs is not None else 2 * int(out.totals[1]) + 8 * eb.n_regions + 64,
                       cap_ins if cap_ins is not None else 64 * n_alns + 16 * eb.n_regions + 64, n_enum_segs=int(out.totals[1]))
        self._chk(self.lib.sx_link_alignments(self.h, C.byref(eb.c), C.byref(out.c), n_alns, A.ptr(eb.ins_off), A.ptr(eb.ins_pool), C.byref(lo.c)))
        return lo

    # ---- K7a
    def alignment_indels(self, eb: B.EnumBatch, pools: B.AlignBatch, cap_keys=None) -> B.PrepOut:
        """K7a: the window entries every read's input alignment already contains (host buffers).  `pools`: the K1 batch holding the reads
        and reference windows (B.read_pools_of)."""
        po = B.PrepOut(eb, cap_keys)
        self._chk(self.lib.sx_alignment_indels(self.h, C.byref(eb.c), A.ptr(pools.regions), A.ptr(pools.seq4), A.ptr(pools.ref), A.ptr(eb.ins_off), A.ptr(eb.ins_pool),
                                               C.byref(po.c)))
        return po

    # ---- K9
    def choose_realignment(self, rb: B.RealignBatch, lnp: np.ndarray, cap_segs=None) -> B.RealignOut:
        """K9: rseg.realignment of every read from its candidate alignments and their scores (host buffers)."""
        lnp = np.ascontiguousarray(lnp, dtype=np.float64)
        ro = B.RealignOut(rb, cap_segs)
        self._chk(self.lib.sx_choose_realignment(self.h, C.byref(rb.c), lnp.ctypes.data, C.byref(ro.c)))
        return ro

    # ---- K7g
    def realign_gates(self, gb: B.GateBatch) -> B.GateOut:
        """K7g: which reads go into the alignment search and with which (normalized) input alignment (host buffers)."""
        go = B.GateOut(gb)
        self._chk(self.lib.sx_realign_gates(self.h, C.byref(gb.c), C.byref(go.c)))
        return go


# the name under which the test suite's host-memory context (tests/mockctx.py) takes K7's device entry
_enumerate_alignments_dev = Context.enumerate_alignments_dev


class DevSomaticIndelBatch:
    """sx_sindel_batch whose arrays live in HBM, with a device output buffer; the error-rate table stays on the host."""

    def __init__(self, ctx: "Context", hb: "B.SomaticIndelBatch"):
        self.host = hb
        self.c, self.bufs = _device_twin(ctx, hb.c, hb, 64)
        self.out = DeviceArray(ctx, max(1, hb.n_loci) * A.SINDEL_RESULT_DT.itemsize)

    def download(self) -> np.ndarray:
        return self.out.download(A.SINDEL_RESULT_DT, self.host.n_loci)


class DevScoreIndelsBatch:
    """sx_score_indels_batch whose arrays live in HBM, with device output buffers; `lnp` is usually DevAlignBatch.out."""

    def __init__(self, ctx: "Context", hb: B.ScoreIndelsBatch):
        self.host = hb
        self.c, self.bufs = _device_twin(ctx, hb.c, hb, 64)
        self.recs = DeviceArray(ctx, (hb.n_rec_slots + 1) * A.READ_INDEL_SCORE_DT.itemsize)
        self.n_rec, self.max_aln, self.eval_aln = (DeviceArray(ctx, (hb.n_reads + 1) * 4) for _ in range(3))
        self.out = A.SxScoreIndelsOut(recs=self.recs.ptr, n_rec=self.n_rec.ptr, max_aln=self.max_aln.ptr, eval_aln=self.eval_aln.ptr)

    def download(self):
        hb = self.host
        out = B.ScoreIndelsOut(hb)
        out.recs[:] = self.recs.download(A.READ_INDEL_SCORE_DT, hb.n_rec_slots + 1)
        out.n_rec[:] = self.n_rec.download(np.uint32, hb.n_reads + 1)
        out.max_aln[:] = self.max_aln.download(np.uint32, hb.n_reads + 1)
        out.eval_aln[:] = self.eval_aln.download(np.uint32, hb.n_reads + 1)
        return out.compact()


class DevIndelReadsSample:
    """sx_indel_reads_sample in HBM.  `from_score_indels` adopts a DevScoreIndelsBatch: its read arrays and the recs / n_rec arrays K6
    wrote, which that object owns -- so two samples scored on ONE context stay apart.  `from_window` does the same with a DevWindow's
    pass."""

    def __init__(self, ctx: "Context", hs: B.IndelReadsSample, adopt: Optional[dict] = None):
        self.host = hs
        self.c, self.bufs = _device_twin(ctx, hs.c, hs, 64, adopt)

    @staticmethod
    def from_score_indels(ctx: "Context", db: DevScoreIndelsBatch, key_gid, read_id=None) -> "DevIndelReadsSample":
        hb = db.host
        hs = B.IndelReadsSample(hb, np.zeros(hb.n_rec_slots + 1, A.READ_INDEL_SCORE_DT), np.zeros(hb.n_reads + 1, np.uint32), key_gid, read_id)
        adopt = {n: db.bufs[n].ptr for n in ("region_read_off", "region_key_off", "rec_off", "read_len", "non_ambig", "read_flags")}
        adopt.update(recs=db.recs.ptr, n_rec=db.n_rec.ptr)
        self = DevIndelReadsSample(ctx, hs, adopt)
        self.score = db  # (keeps the adopted buffers alive)
        return self

    @staticmethod
    def from_window(ctx: "Context", dw: "DevWindow", key_gid, read_id, non_ambig) -> "DevIndelReadsSample":
        """The sample of a DevWindow pass (keep_outputs): the window's read arrays and the recs / n_rec its pass wrote, adopted; key_gid,
        read_id and `non_ambig` (each read's count of bases that are not 'N', uint16) uploaded."""
        w = dw.w
        n = w.n_reads
        assert len(non_ambig) >= n
        sb = SimpleNamespace(n_regions=w.n_regions, n_reads=n, n_keys=w.n_keys, non_ambig=np.ascontiguousarray(non_ambig, np.uint16),
                             **{k: w.a[k] for k in ("region_read_off", "region_key_off", "rec_off", "read_len", "read_flags")})
        hs = B.IndelReadsSample(sb, np.zeros(dw.n_slots + 1, A.READ_INDEL_SCORE_DT), np.zeros(n + 1, np.uint32), key_gid, read_id)
        adopt = {k: dw.bufs[k].ptr for k in ("region_read_off", "region_key_off", "rec_off", "read_len", "read_flags")}
        adopt.update(recs=dw.obufs["recs"].ptr, n_rec=dw.obufs["n_rec"].ptr)
        self = DevIndelReadsSample(ctx, hs, adopt)
        self.window = dw  # (keeps the adopted buffers alive)
        return self


class DevIndelLoci:
    def __init__(self, ctx: "Context", hl: B.IndelLoci):
        self.host = hl
        self.c, self.bufs = _device_twin(ctx, hl.c, hl, 64)


class DevAlleleGroups:
    def __init__(self, ctx: "Context", hg: B.AlleleGroups):
        self.host = hg
        self.c, self.bufs = _device_twin(ctx, hg.c, hg, 64)


class DevGermlineIndelChain:
    """K6's records of one sample -> germline indel genotype likelihoods without a host step (sx_indel_gl_from_records_dev): the K6g link,
    then K5 on the sx_indel_batch the link left in the context's buffers.  The sample's recs / n_rec arrays are caller-owned
    (DevIndelReadsSample, from_score_indels or from_window).  `download()` returns (results, status): a group the link flagged has its
    status and an all-zero result."""

    def __init__(self, ctx: "Context", sample: DevIndelReadsSample, groups: B.AlleleGroups):
        self.ctx, self.sample, self.groups = ctx, sample, DevAlleleGroups(ctx, groups)
        n = max(1, groups.n_groups)
        self.out = DeviceArray(ctx, n * A.INDEL_RESULT_DT.itemsize)
        self.status = DeviceArray(ctx, n * 4)

    def run(self) -> None:
        ctx = self.ctx
        ctx._chk(ctx.lib.sx_indel_gl_from_records_dev(ctx.h, C.byref(self.sample.c), C.byref(self.groups.c), self.out.ptr, self.status.ptr))

    def download(self) -> Tuple[np.ndarray, np.ndarray]:
        n = self.groups.host.n_groups
        return self.out.download(A.INDEL_RESULT_DT, n), self.status.download(np.uint32, n)


class DevSomaticIndelChain:
    """K6's records of two samples -> somatic indel calls without a host step (sx_somatic_indel_from_records_dev): the link, then K5b on
    the sx_sindel_batch the link left in the context's buffers.  The samples' recs / n_rec arrays are caller-owned (DevIndelReadsSample)."""

    def __init__(self, ctx: "Context", normal: DevIndelReadsSample, tumor: DevIndelReadsSample, loci: B.IndelLoci):
        self.ctx, self.normal, self.tumor, self.loci = ctx, normal, tumor, DevIndelLoci(ctx, loci)
        self.out = DeviceArray(ctx, max(1, loci.n_loci) * A.SINDEL_RESULT_DT.itemsize)

    def run(self, opts: Optional[A.SxSindelOpts] = None) -> None:
        o = opts or A.default_sindel_opts()
        hl, ctx = self.loci.host, self.ctx
        ctx._chk(ctx.lib.sx_somatic_indel_from_records_dev(ctx.h, C.byref(o), C.byref(self.normal.c), C.byref(self.tumor.c), C.byref(self.loci.c),
                                                           A.ptr(hl.err_prob), hl.err_prob.size, self.out.ptr))

    def download(self) -> np.ndarray:
        return self.out.download(A.SINDEL_RESULT_DT, self.loci.host.n_loci)


class DevEnumBatch:
    """An sx_enum_batch and its sx_enum_out resident in device memory (for sx_enumerate_alignments_dev)."""

    def __init__(self, ctx: "Context", hb: B.EnumBatch, cap_alns=None, cap_segs=None, cap_keys=None):
        self.host = hb
        self.c, self.bufs = _device_twin(ctx, hb.c, hb, 64)
        self.shape = B.EnumOut(hb, cap_alns, cap_segs, cap_keys)  # host twin: sizes and the download target
        s = self.shape
        self.obufs = {n: DeviceArray(ctx, getattr(s, n).nbytes + 64) for n in ("totals", "aln_off", "status", "aln_pos", "aln_seg_off", "segs", "aln_key_off",
                                                                               "aln_keys", "aln_lead_key", "aln_trail_key")}
        self.out = A.SxEnumOut(cap_alns=s.cap_alns, cap_segs=s.cap_segs, cap_keys=s.cap_keys, **{n: b.ptr for n, b in self.obufs.items()})

    def download(self) -> B.EnumOut:
        s = self.shape
        for n, buf in self.obufs.items():
            a = getattr(s, n)
            a[...] = buf.download(a.dtype, a.size)
        return s


class DevRealignChain:
    """The device-resident chain of realignAndScoreRead for a batch of reads: K7a (keys of the input alignments) -> K7 (candidate
    alignments) -> K7b (K1's alignment arrays) -> K1 (scores) -> K6 (score_indels), every intermediate staying in HBM; what crosses to the
    host between the steps is the three + two totals that size the next buffers.  `pools`: the K1 batch holding the reads, qualities
    and reference windows in K7's read order (B.read_pools_of or a real one); its region records receive the alignment offsets."""

    def __init__(self, ctx: "Context", eb: B.EnumBatch, pools: B.AlignBatch, cap_alns_per_read: int = 16, read_flags=None, rec_off=None, raw: "B.GateBatch" = None):
        # bases / reference in the wide formats (K7a reads them); qualities may be dictionary-coded (qual_bits 4 selects K1's byte-entry kernel)
        assert pools.fmt == 0 and pools.qual_bits in (0, 4, 8) and pools.n_reads == eb.n_reads
        self.ctx, self.eb = ctx, eb
        self.enum = DevEnumBatch(ctx, eb, cap_alns=eb.n_reads * cap_alns_per_read + 64, cap_segs=eb.n_reads * cap_alns_per_read * 4 + 64,
                                 cap_keys=eb.n_reads * cap_alns_per_read * 2 + 64)
        self.pools = DevAlignBatch(ctx, pools)
        self.key_ins_off = DeviceArray(ctx, eb.ins_off.nbytes + 64).upload(eb.ins_off)
        self.key_ins = DeviceArray(ctx, eb.ins_pool.nbytes + 64).upload(eb.ins_pool)
        n = eb.n_reads
        self.cap_in_keys = 8 * n + 64
        self.prep = {"totals": DeviceArray(ctx, 16), "in_key_off": DeviceArray(ctx, (n + 1) * 4 + 16), "in_keys": DeviceArray(ctx, self.cap_in_keys * 2 + 16),
                     "in_lead_key": DeviceArray(ctx, n * 2 + 16), "in_trail_key": DeviceArray(ctx, n * 2 + 16)}
        p = self.prep
        self.prep_out = A.SxPrepOut(cap_keys=self.cap_in_keys, **{k: x.ptr for k, x in p.items()})
        # K7 reads what K7a writes
        c = self.enum.c
        c.in_key_off, c.in_keys, c.in_lead_key, c.in_trail_key = p["in_key_off"].ptr, p["in_keys"].ptr, p["in_lead_key"].ptr, p["in_trail_key"].ptr
        # K6's per-read inputs
        flags = read_flags if read_flags is not None else np.full(n + 1, A.SX_SIF_FWD | A.SX_SIF_TIER1, np.uint8)
        if rec_off is None:
            n_win = np.diff(eb.region_key_off.astype(np.int64))
            rec_off = np.concatenate([[0], np.cumsum(np.repeat(n_win, np.diff(eb.region_read_off.astype(np.int64))))]).astype(np.uint32)
        self.rec_off_host = rec_off
        self.read_flags = DeviceArray(ctx, flags.nbytes + 16).upload(flags)
        self.rec_off = DeviceArray(ctx, rec_off.nbytes + 16).upload(rec_off)
        self.n_slots = int(rec_off[-1])
        self.recs = DeviceArray(ctx, (self.n_slots + 1) * A.READ_INDEL_SCORE_DT.itemsize)
        self.n_rec, self.max_aln, self.eval_aln = (DeviceArray(ctx, (n + 1) * 4) for _ in range(3))
        self.link = self.lnp = None
        self.realign = None
        self.ms = {}
        # optional first step K7g: the mapper's alignments (`raw`, a B.GateBatch over the same reads) -> gate + normalized input alignment,
        # written where K7a / K7 read them; eb's own in_pos / in_segs / in_seg_off are then not used
        self.gates = None
        self.raw_host = raw
        if raw is not None:
            assert raw.eb is eb
            g = {"raw_pos": DeviceArray(ctx, raw.raw_pos.nbytes + 16).upload(raw.raw_pos), "seg_off": DeviceArray(ctx, raw.seg_off.nbytes + 16).upload(raw.seg_off),
                 "raw_segs": DeviceArray(ctx, raw.raw_segs.nbytes + 16).upload(raw.raw_segs), "gate": DeviceArray(ctx, n + 16), "in_pos": DeviceArray(ctx, n * 4 + 16),
                 "in_segs": DeviceArray(ctx, raw.raw_segs.nbytes + 16)}
            b0 = self.enum.bufs
            self.gate_batch = A.SxGateBatch(n_regions=eb.n_regions, n_reads=n, max_indel_size=eb.opts.max_indel_size,
                                            **{k: b0[k].ptr for k in ("region_read_off", "region_key_off", "keys", "realign_begin", "realign_end", "read_len")},
                                            **{k: g[k].ptr for k in ("raw_pos", "seg_off", "raw_segs")})
            self.gate_out = A.SxGateOut(gate=g["gate"].ptr, in_pos=g["in_pos"].ptr, in_segs=g["in_segs"].ptr)
            c.in_pos, c.in_seg_off, c.in_segs, c.gate = g["in_pos"].ptr, g["seg_off"].ptr, g["in_segs"].ptr, g["gate"].ptr
            self.gates = g

    def run(self):
        ctx, eb, e = self.ctx, self.eb, self.enum
        pc = self.pools.c
        if self.gates is not None:
            ctx._chk(ctx.lib.sx_realign_gates_dev(ctx.h, C.byref(self.gate_batch), C.byref(self.gate_out)))
            self.ms["k7g_realign_gates"] = ctx.timing().kernel_ms
        ctx._chk(ctx.lib.sx_alignment_indels_dev(ctx.h, C.byref(e.c), pc.regions, pc.seq4, pc.ref, self.key_ins_off.ptr, self.key_ins.ptr, C.byref(self.prep_out)))
        self.ms["k7a_alignment_indels"] = ctx.timing().kernel_ms
        ctx.enumerate_alignments_dev(e)
        self.ms["k7_enumerate"] = ctx.timing().kernel_ms
        nA, nS, nK = (int(x) for x in e.obufs["totals"].download(np.uint32, 3))
        self.totals = (nA, nS, nK)
        if self.link is None or self.link["n_alns"] < nA or self.link["n_enum_segs"] < nS:  # sized by what the enumeration produced
            max_ins = max(1, int(eb.keys["ins_len"].max(initial=0)))
            cap_segs, cap_ins = 2 * nS + 8 * eb.n_regions + 64, nS * max_ins + 16 * eb.n_regions + 64
            self.link = {"n_alns": nA, "n_enum_segs": nS, "cap_segs": cap_segs, "cap_ins": cap_ins, "totals": DeviceArray(ctx, 16),
                         "alns": DeviceArray(ctx, (nA + 1) * A.ALN_DT.itemsize + 16), "segs": DeviceArray(ctx, (cap_segs + 16) * 4 + 16),
                         "ins": DeviceArray(ctx, cap_ins + A.SX_POOL_SLACK + 16), "k6_segs": DeviceArray(ctx, (nS + 16) * 4 + 16)}
            self.lnp = DeviceArray(ctx, (nA + 1) * 8 + 16)
        L = self.link
        lo = A.SxLinkOut(cap_segs=L["cap_segs"], cap_ins=L["cap_ins"], regions=pc.regions, **{k: L[k].ptr for k in ("totals", "alns", "segs", "ins", "k6_segs")})
        ctx._chk(ctx.lib.sx_link_alignments_dev(ctx.h, C.byref(e.c), C.byref(e.out), nA, self.key_ins_off.ptr, self.key_ins.ptr, C.byref(lo)))
        self.ms["k7b_link"] = ctx.timing().kernel_ms
        n_k1_segs, ins_bytes = (int(x) for x in L["totals"].download(np.uint32, 2))
        self.k1_totals = (n_k1_segs, ins_bytes)
        k1 = A.SxAlignBatch(n_regions=eb.n_regions, n_reads=eb.n_reads, n_alns=nA, n_segs=n_k1_segs, regions=pc.regions, read_len=pc.read_len, seq4=pc.seq4, qual=pc.qual,
                            ref=pc.ref, alns=L["alns"].ptr, segs=L["segs"].ptr, ins=L["ins"].ptr, seq4_bytes=pc.seq4_bytes, qual_bytes=pc.qual_bytes, ref_bytes=pc.ref_bytes,
                            ins_bytes=ins_bytes, qual_bits=pc.qual_bits, qual_dict=pc.qual_dict)
        ctx._chk(ctx.lib.sx_score_alignments_dev(ctx.h, C.byref(k1), self.lnp.ptr))
        self.ms["k1_score_alignments"] = ctx.timing().kernel_ms
        o = e.obufs
        b = e.bufs
        k6 = A.SxScoreIndelsBatch(n_regions=eb.n_regions, n_reads=eb.n_reads, n_alns=nA, n_keys=eb.n_keys, region_read_off=b["region_read_off"].ptr,
                                  region_key_off=b["region_key_off"].ptr, keys=b["keys"].ptr, aln_off=o["aln_off"].ptr, aln_pos=o["aln_pos"].ptr,
                                  aln_seg_off=o["aln_seg_off"].ptr, segs=L["k6_segs"].ptr, aln_key_off=o["aln_key_off"].ptr, aln_keys=o["aln_keys"].ptr,
                                  read_len=b["read_len"].ptr,
                                  non_ambig=b["read_len"].ptr,  # the enum batch has no per-read count of non-N bases: every base counts
                                  read_flags=self.read_flags.ptr, rec_off=self.rec_off.ptr, opts=A.default_score_indels_opts())
        out = A.SxScoreIndelsOut(recs=self.recs.ptr, n_rec=self.n_rec.ptr, max_aln=self.max_aln.ptr, eval_aln=self.eval_aln.ptr)
        ctx._chk(ctx.lib.sx_score_indels_dev(ctx.h, C.byref(k6), self.lnp.ptr, C.byref(out)))
        self.ms["k6_score_indels"] = ctx.timing().kernel_ms
        # K9: rseg.realignment of every read, in K4's segment kinds
        n = eb.n_reads
        n_raw = int(self.raw_host.seg_off[n]) if self.gates is not None else 0
        cap = nS + 2 * n + n_raw + 64
        if self.realign is None or self.realign["cap"] < cap:
            self.realign = {"cap": cap, "totals": DeviceArray(ctx, 16), "seg_off": DeviceArray(ctx, (n + 1) * 4 + 16), "pos": DeviceArray(ctx, n * 4 + 16),
                            "n_seg": DeviceArray(ctx, n * 2 + 16), "status": DeviceArray(ctx, n + 16), "best_aln": DeviceArray(ctx, n * 4 + 16),
                            "segs": DeviceArray(ctx, cap * 4 + 16)}
        R = self.realign
        rb = A.SxRealignBatch(n_regions=eb.n_regions, n_reads=n, n_alns=nA, region_read_off=b["region_read_off"].ptr, region_key_off=b["region_key_off"].ptr,
                              keys=b["keys"].ptr, aln_off=o["aln_off"].ptr, aln_pos=o["aln_pos"].ptr, aln_seg_off=o["aln_seg_off"].ptr, segs=o["segs"].ptr,
                              aln_key_off=o["aln_key_off"].ptr, aln_keys=o["aln_keys"].ptr, read_len=b["read_len"].ptr, is_smoothed_alignments=1, k4_kinds=1,
                              smoothed_lnp_range=2.302585092994046)
        if self.gates is not None:  # the mapper's alignments are at hand: K9's output is then getBestAlignment() of every read (K4's input)
            rb.raw_pos, rb.raw_seg_off, rb.raw_segs = self.gates["raw_pos"].ptr, self.gates["seg_off"].ptr, self.gates["raw_segs"].ptr
        ro = A.SxRealignOut(cap_segs=R["cap"], **{k: R[k].ptr for k in ("totals", "seg_off", "pos", "n_seg", "status", "best_aln", "segs")})
        ctx._chk(ctx.lib.sx_choose_realignment_dev(ctx.h, C.byref(rb), self.lnp.ptr, C.byref(ro)))
        self.ms["k9_choose_realignment"] = ctx.timing().kernel_ms
        return dict(self.ms)

    def download_realignments(self):
        """(pos[n_reads], n_seg[n_reads], status[n_reads], seg_off[n_reads + 1], segs in K4's kinds)"""
        n, R = self.eb.n_reads, self.realign
        seg_off = R["seg_off"].download(np.uint32, n + 1)
        return (R["pos"].download(np.int32, n), R["n_seg"].download(np.uint16, n), R["status"].download(np.uint8, n), seg_off,
                R["segs"].download(A.ALN_SEG_DT, int(seg_off[n])))

    def download(self):
        """(EnumOut, lnp[n_alns], n_rec[n_reads], max_aln[n_reads], records of read r = recs[rec_off[r] : rec_off[r] + n_rec[r]])"""
        n = self.eb.n_reads
        return (self.enum.download(), self.lnp.download(np.float64, self.totals[0]), self.n_rec.download(np.uint32, n), self.max_aln.download(np.uint32, n),
                self.recs.download(A.READ_INDEL_SCORE_DT, self.n_slots))

    def free(self):
        bufs = list(self.enum.bufs.values()) + list(self.enum.obufs.values()) + list(self.pools.bufs.values()) + list(self.prep.values())
        bufs += [self.key_ins_off, self.key_ins, self.read_flags, self.rec_off, self.recs, self.n_rec, self.max_aln, self.eval_aln, self.pools.out]
        if self.link:
            bufs += [v for v in self.link.values() if isinstance(v, DeviceArray)] + [self.lnp]
        if self.realign:
            bufs += [v for v in self.realign.values() if isinstance(v, DeviceArray)]
        if self.gates:
            bufs += list(self.gates.values())
        for d in bufs:
            d.free()


class DevWindow:
    """sx_process_window_dev on a B.WindowBatch: every input array resident in HBM, every output array the caller may want to read
    back allocated here (tests download them; bench.py leaves them where they are)."""

    def __init__(self, ctx: "Context", w: "B.WindowBatch", keep_outputs: bool = True, cap_best_segs=None):
        self.ctx, self.w = ctx, w
        c = A.SxWindowBatch()
        ctx.lib.sx_default_window_opts(C.byref(c))
        c.n_regions, c.n_reads, c.n_keys = w.n_regions, w.n_reads, w.n_keys
        for name in B.WindowBatch.ARRAYS:  # host pointers: the twin below puts each array in device memory
            setattr(c, name, A.ptr(w.a.get(name)))
        c.n_cand_snv = int(w.a["cand_snv"].size) if w.a.get("cand_snv") is not None else 0
        c.seq4_bytes, c.qual_bytes, c.ref_bytes = w.used["seq4"], w.used["qual"], w.used["ref"]
        c.qual_bits = w.qual_bits
        c.qual_dict = (C.c_uint8 * 16)(*(w.qual_dict + [0] * (16 - len(w.qual_dict))))
        c.ref_begin, c.report_begin, c.report_end = w.ref_begin, w.report_begin, w.report_end
        c.max_read_len, c.do_site_gl = w.max_read_len, 1 if w.do_site_gl else 0
        if getattr(w, "enum_opts", None) is not None:
            keep = c.enum_opts.max_alns_per_read
            c.enum_opts = w.enum_opts
            c.enum_opts.max_alns_per_read = max(keep, w.enum_opts.max_alns_per_read)
        self.c, self.bufs = _device_twin(ctx, c, SimpleNamespace(**w.a), 80)
        self.out = A.SxWindowOut()
        self.obufs = {}
        n, ns = w.n_reads, w.n_sites
        if keep_outputs:
            n_raw = int(w.a["raw_seg_off"][n])
            self.cap_best = cap_best_segs if cap_best_segs is not None else 64 * n + n_raw + 4096
            n_slots = int(w.a["rec_off"][n])
            bases = int(np.asarray(w.a["read_len"][:n], dtype=np.int64).sum()) + 64
            sizes = {"gate": n + 16, "enum_status": n + 16, "realign_status": n + 16, "best_pos": 4 * n + 16, "best_seg_off": 4 * (n + 2), "best_n_seg": 2 * n + 16,
                     "best_segs": 4 * self.cap_best + 64, "recs": (n_slots + 1) * A.READ_INDEL_SCORE_DT.itemsize, "n_rec": 4 * n + 16, "site_off": 4 * (ns + 2),
                     "t2_off": 4 * (ns + 2), "n_spandel": 4 * (ns + 2), "n_submapped": 4 * (ns + 2), "calls": 2 * bases, "t2_calls": 2 * bases,
                     "site_gl": (ns + 1) * A.DIGT_RESULT_DT.itemsize, "totals": 64, "variant_sites": (ns // 8 + 1024) * A.SITE_CALL_DT.itemsize}
            self.obufs = {k: DeviceArray(ctx, v) for k, v in sizes.items()}
            o, b = self.out, self.obufs
            for k in ("gate", "enum_status", "realign_status", "best_pos", "best_seg_off", "best_n_seg", "best_segs", "recs", "n_rec", "site_gl", "totals"):
                setattr(o, k, b[k].ptr)
            o.cap_best_segs = self.cap_best
            if w.do_site_gl:
                o.variant_sites, o.cap_variant_sites = b["variant_sites"].ptr, ns // 8 + 1024
            o.cols = A.SxPileupColumns(calls_capacity=bases, t2_capacity=bases,
                                       **{k: b[k].ptr for k in ("site_off", "calls", "t2_off", "t2_calls", "n_spandel", "n_submapped")})
            self.n_slots = n_slots
        else:  # only the call records come out; everything else stays in the context's own buffers
            cap_v = ns // 8 + 1024
            self.obufs = {"variant_sites": DeviceArray(ctx, cap_v * A.SITE_CALL_DT.itemsize)}
            self.out.variant_sites, self.out.cap_variant_sites = self.obufs["variant_sites"].ptr, cap_v
        self.totals = np.zeros(A.SX_WIN_TOTALS, np.uint32)

    def run(self):
        """one pass; returns the per-stage device times (ms)"""
        ctx = self.ctx
        ctx._chk(ctx.lib.sx_process_window_dev(ctx.h, C.byref(self.c), C.byref(self.out), self.totals.ctypes.data))
        ms = np.zeros(A.SX_WIN_N_STAGES, np.float32)
        ctx.lib.sx_last_window_timing(ctx.h, ms.ctypes.data)
        return dict(zip(A.SX_WIN_STAGE_NAMES, (float(x) for x in ms)))

    def download(self):
        """dict of the host copies of every output (keep_outputs only)"""
        w, b = self.w, self.obufs
        n, ns = w.n_reads, w.n_sites
        d = {"gate": b["gate"].download(np.uint8, n), "enum_status": b["enum_status"].download(np.uint8, n), "realign_status": b["realign_status"].download(np.uint8, n),
             "best_pos": b["best_pos"].download(np.int32, n), "best_seg_off": b["best_seg_off"].download(np.uint32, n + 1), "best_n_seg": b["best_n_seg"].download(np.uint16, n),
             "n_rec": b["n_rec"].download(np.uint32, n), "recs": b["recs"].download(A.READ_INDEL_SCORE_DT, self.n_slots),
             "site_off": b["site_off"].download(np.uint32, ns + 1), "t2_off": b["t2_off"].download(np.uint32, ns + 1), "n_spandel": b["n_spandel"].download(np.uint32, ns),
             "n_submapped": b["n_submapped"].download(np.uint32, ns), "totals": self.totals.copy()}
        d["best_segs"] = b["best_segs"].download(A.ALN_SEG_DT, int(d["best_seg_off"][n]))
        d["calls"] = b["calls"].download(np.uint16, int(d["site_off"][ns]))
        d["t2_calls"] = b["t2_calls"].download(np.uint16, int(d["t2_off"][ns]))
        if w.do_site_gl:
            d["site_gl"] = b["site_gl"].download(A.DIGT_RESULT_DT, ns)
            d["variant_sites"] = b["variant_sites"].download(A.SITE_CALL_DT, int(self.totals[8]))
        return d

    def free(self):
        for x in list(self.bufs.values()) + list(self.obufs.values()):
            x.free()


class DevSomaticWindow:
    """sx_process_somatic_window_dev on two B.WindowBatch samples (normal, tumor) of one window of positions and the candidate loci: every
    input resident in HBM, every output allocated here.  The samples' per-read and column outputs are DevWindow's (`normal` / `tumor`).
    useTier2Evidence of the pile-up and of K5b is `use_tier2`.  records_only: only the two record lists and the totals come out; every other
    output (the samples', site_snv, indel) is left NULL, so the pass keeps it in the context's own buffers."""

    def __init__(self, ctx: "Context", normal: "B.WindowBatch", tumor: "B.WindowBatch", loci: "B.IndelLoci", key_gid, read_id=None, snv_forced=None,
                 use_tier2: bool = False, opts: Optional[A.SxSindelOpts] = None, cap_snv_calls=None, cap_indel_calls=None, records_only: bool = False):
        assert not normal.do_site_gl and not tumor.do_site_gl, "strelka2 runs no germline site model: build the samples with do_site_gl=False"
        self.ctx, self.loci = ctx, loci
        self.records_only = records_only
        self.windows = [DevWindow(ctx, w, keep_outputs=not records_only) for w in (normal, tumor)]
        self.normal, self.tumor = self.windows
        self.n_sites, n_loci = normal.n_sites, loci.n_loci
        self.opts = A.SxSindelOpts.from_buffer_copy(opts) if opts is not None else A.default_sindel_opts()
        self.opts.useTier2Evidence = int(use_tier2)
        for dw in self.windows:
            dw.c.pileup_opts.useTier2Evidence = int(use_tier2)
            dw.out.site_gl = dw.out.variant_sites = None
            dw.out.cap_variant_sites = 0
        self.dloci = DevIndelLoci(ctx, loci)
        up = lambda a, dt: None if a is None else DeviceArray(ctx, np.ascontiguousarray(a, dt).nbytes + 64).upload(np.ascontiguousarray(a, dt))
        self.inbufs = {"key_gid": [up(k, np.uint32) for k in key_gid], "read_id": [up(r, np.uint32) for r in (read_id or (None, None))],
                       "snv_forced": up(snv_forced, np.uint8)}
        self.err_prob = np.ascontiguousarray(loci.err_prob, np.float64)
        ib = self.inbufs
        self.c = A.SxSomaticWindowBatch(sample=(A.SxWindowBatch * 2)(*(dw.c for dw in self.windows)),
                                        key_gid=(C.c_void_p * 2)(*(x.ptr if x else None for x in ib["key_gid"])),
                                        read_id=(C.c_void_p * 2)(*(x.ptr if x else None for x in ib["read_id"])),
                                        snv_forced_output=ib["snv_forced"].ptr if ib["snv_forced"] else None, loci=self.dloci.c, sindel_opts=self.opts,
                                        err_prob=A.ptr(self.err_prob), n_err=self.err_prob.size)
        self.cap_snv = max(1, self.n_sites) if cap_snv_calls is None else cap_snv_calls
        self.cap_indel = max(1, n_loci) if cap_indel_calls is None else cap_indel_calls
        self.obufs = {"site_snv": DeviceArray(ctx, (self.n_sites + 1) * A.SSNV_RESULT_DT.itemsize),
                      "snv_calls": DeviceArray(ctx, (self.cap_snv + 1) * A.SOMATIC_SITE_CALL_DT.itemsize),
                      "indel": DeviceArray(ctx, (n_loci + 1) * A.SINDEL_RESULT_DT.itemsize),
                      "indel_calls": DeviceArray(ctx, (self.cap_indel + 1) * A.SOMATIC_INDEL_CALL_DT.itemsize), "totals": DeviceArray(ctx, 64)}
        if records_only:
            for k in ("site_snv", "indel"):
                self.obufs.pop(k).free()
        samples = (A.SxWindowOut * 2)() if records_only else (A.SxWindowOut * 2)(*(dw.out for dw in self.windows))
        self.out = A.SxSomaticWindowOut(sample=samples, cap_snv_calls=self.cap_snv, cap_indel_calls=self.cap_indel, **{k: b.ptr for k, b in self.obufs.items()})
        self.totals = np.zeros(A.SX_SWIN_TOTALS, np.uint32)

    def run(self):
        """one pass; returns the per-stage device times (ms).  SX_ERR_CAPACITY leaves the totals in the SxError's `totals`."""
        ctx = self.ctx
        rc = ctx.lib.sx_process_somatic_window_dev(ctx.h, C.byref(self.c), C.byref(self.out), self.totals.ctypes.data)
        ctx._chk_totals(rc, self.totals)
        ms = np.zeros(A.SX_SWIN_N_STAGES, np.float32)
        ctx.lib.sx_last_somatic_window_timing(ctx.h, ms.ctypes.data)
        return dict(zip(A.SX_SWIN_STAGE_NAMES, (float(x) for x in ms)))

    def download(self):
        """dict: each sample's DevWindow.download(), the per-position and per-locus results, the two record lists and the totals (records_only:
        the record lists and the totals)"""
        b, t = self.obufs, self.totals
        records = {"snv_calls": b["snv_calls"].download(A.SOMATIC_SITE_CALL_DT, min(int(t[0]), self.cap_snv)),
                   "indel_calls": b["indel_calls"].download(A.SOMATIC_INDEL_CALL_DT, min(int(t[1]), self.cap_indel)), "totals": t.copy()}
        if self.records_only:
            return records
        for dw in self.windows:  # (each sample's totals are where the pass wrote them)
            dw.totals[:] = dw.obufs["totals"].download(np.uint32, A.SX_WIN_TOTALS)
        return {"normal": self.normal.download(), "tumor": self.tumor.download(), "site_snv": b["site_snv"].download(A.SSNV_RESULT_DT, self.n_sites),
                "indel": b["indel"].download(A.SINDEL_RESULT_DT, self.loci.n_loci), **records}

    def free(self):
        for dw in self.windows:
            dw.free()
        bufs = list(self.obufs.values()) + list(self.dloci.bufs.values()) + [x for x in self.inbufs["key_gid"] + self.inbufs["read_id"] + [self.inbufs["snv_forced"]] if x]
        for x in bufs:
            x.free()
