"""Host-side construction of the flattened batches the C ABI consumes.

This is the Python twin of the C++ host mirror in ``strelka_b200/host`` (used by tests and bench.py): it takes
reference-shaped objects -- a candidate alignment as (pos, CIGAR path, indel keys with candidacy), a pileup as a list of
``base_call`` fields -- and produces ``sx_align_batch`` / ``sx_pileup_batch`` arrays that obey the staging rules of
``include/strelka_b200.h``.

The flattening of a candidate alignment follows the segment walk of ``scoreCandidateAlignment``
(/root/reference/src/c++/lib/starling_common/starling_read_align_score.cpp:289-499) exactly; what is resolved here is
everything that function looks up in host-only containers (``getMatchingIndelKey`` :172-224, ``getInsertSeq`` :229-256,
``IndelBuffer::isCandidateIndel`` :473-475, the leading-edge insert-sequence tail rule :334-338 / :394-398).
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import numpy as np

from . import _abi as A

# INDEL::index_t  (starling_common/indel_core.hh:57-66)
INDEL_NONE, INDEL_INDEL, INDEL_MISMATCH, INDEL_BP_LEFT, INDEL_BP_RIGHT = 0, 1, 2, 3, 4

BAM_CODE = {"=": 0, "A": 1, "C": 2, "G": 4, "T": 8, "N": 15}  # htsapi/bam_seq.hh:38-47


def codes_of(seq: str) -> np.ndarray:
    return np.array([BAM_CODE.get(c, 15) for c in seq], dtype=np.uint8)


@dataclass
class IndelKeySpec:
    """IndelKey (starling_common/IndelKey.hh:39-193) + its candidacy in the IndelBuffer."""

    pos: int
    type: int = INDEL_INDEL
    delete_length: int = 0
    insert_seq: str = ""
    is_candidate: bool = True


@dataclass
class CandidateAlignmentSpec:
    """CandidateAlignment (starling_common/CandidateAlignment.hh:36-83) for read index ``read`` of its region."""

    read: int
    pos: int
    path: List[Tuple[str, int]]  # [('M', 70), ('I', 5), ...]  ALIGNPATH types as CIGAR chars
    indels: List[IndelKeySpec] = field(default_factory=list)
    leading: int = -1  # index into indels of cal.leading_indel_key, or -1
    trailing: int = -1


@dataclass
class RegionSpec:
    ref: str
    ref_begin: int
    reads: List[Tuple[np.ndarray, np.ndarray]]  # (4-bit codes, quals) per read
    alns: List[CandidateAlignmentSpec]


def parse_cigar(s: str) -> List[Tuple[str, int]]:
    out, n = [], ""
    for ch in s:
        if ch.isdigit():
            n += ch
        else:
            out.append((ch, int(n)))
            n = ""
    return out


_ALIGN_MATCH = ("M", "=", "X")


def flatten_alignment(cal: CandidateAlignmentSpec) -> Tuple[List[Tuple[int, int, int]], bytes]:
    """-> ([(len, kind, flags)], insert bytes) following score.cpp:289-499."""
    path = cal.path
    aps = len(path)
    first = last = aps
    seen = False
    for i, (t, _) in enumerate(path):  # get_match_edge_segments, blt_util/align_path.cpp:736-752
        if t in _ALIGN_MATCH:
            if not seen:
                first = i
            seen = True
            last = i
    segs: List[Tuple[int, int, int]] = []
    ins = bytearray()
    ref_head = cal.pos
    i = 0

    def matching_key(ref_head_pos: int, dl: int, il: int, path_index: int) -> IndelKeySpec:
        if path_index < first:
            if cal.leading < 0:
                raise ValueError("leading edge indel without leading_indel_key")
            return cal.indels[cal.leading]
        if path_index > last:
            if cal.trailing < 0:
                raise ValueError("trailing edge indel without trailing_indel_key")
            return cal.indels[cal.trailing]
        for key in cal.indels:  # every key of cal.getIndels(), the edge keys included (score.cpp:203-218)
            if key.pos == ref_head_pos and key.type in (INDEL_INDEL, INDEL_MISMATCH) and key.delete_length == dl and len(key.insert_seq) == il:
                return key
        raise ValueError(f"no indel key matches path segment {path_index} at ref pos {ref_head_pos} (del {dl}, ins {il})")

    def emit_insert(key: IndelKeySpec, seg_len_for_head: int, il: int, path_index: int, flags: int) -> None:
        head = 0
        if path_index < first:
            head = len(key.insert_seq) - seg_len_for_head
        for k in range(il):
            p = head + k
            ins.append(ord(key.insert_seq[p]) if 0 <= p < len(key.insert_seq) else ord("N"))
        segs.append((il, A.SX_SEG_INSERT, flags))

    while i < aps:
        t, ln = path[i]
        # is_segment_swap_start, blt_util/align_path.cpp:868-895
        j, has_i, has_d = i, False, False
        while j < aps and path[j][0] in ("I", "D"):
            has_i |= path[j][0] == "I"
            has_d |= path[j][0] == "D"
            j += 1
        is_swap = has_i and has_d
        n_seg = 1
        if is_swap or t == "X":
            if t == "X":
                dl = il = ln
            else:
                n_seg = j - i
                il = sum(l for tt, l in path[i:j] if tt == "I")
                dl = sum(l for tt, l in path[i:j] if tt == "D")
            key = matching_key(ref_head, dl, il, i)
            fl = 0 if key.is_candidate else A.SX_SEGF_NONCANDIDATE
            emit_insert(key, ln, il, i, fl)
            segs.append((dl, A.SX_SEG_REFSKIP, 0))
            ref_head += dl
        elif t in ("M", "="):
            segs.append((ln, A.SX_SEG_MATCH, 0))
            ref_head += ln
        elif t == "I":
            key = matching_key(ref_head, 0, ln, i)
            fl = 0 if key.is_candidate else A.SX_SEGF_NONCANDIDATE
            emit_insert(key, ln, ln, i, fl)
        elif t in ("D", "N"):
            fl = 0
            if t == "D":
                key = matching_key(ref_head, ln, 0, i)
                fl = 0 if key.is_candidate else A.SX_SEGF_NONCANDIDATE
            segs.append((ln, A.SX_SEG_REFSKIP, fl))
            ref_head += ln
        elif t == "S":
            segs.append((ln, A.SX_SEG_SOFTCLIP, 0))
        elif t == "H":
            segs.append((ln, A.SX_SEG_HARDCLIP, 0))
        else:
            raise ValueError(f"Can't handle cigar code: {t}")  # blt_exception at score.cpp:461-466
        i += n_seg
    return segs, bytes(ins)


def _pad16(n: int) -> int:
    return (n + 15) & ~15


class AlignBatch:
    """Owns the numpy pools of one sx_align_batch and exposes the ctypes struct (``.c``)."""

    def __init__(self, regions, read_len, seq4, qual, ref, alns, segs, ins, used, qual_bits=8, qual_dict=None, fmt=0, n_segs=None, n_alns=None, exc_off=None, exc=None):
        self.regions, self.read_len, self.seq4, self.qual, self.ref = regions, read_len, seq4, qual, ref
        self.qual_bits = qual_bits
        self.fmt = fmt
        self.exc_off, self.exc = exc_off, exc
        self.qual_dict = (C.c_uint8 * 16)(*([int(x) for x in qual_dict] + [0] * (16 - len(qual_dict)))) if qual_dict is not None else (C.c_uint8 * 16)()
        self.alns, self.segs, self.ins = alns, segs, ins
        self.n_regions = len(regions) - 1
        self.n_reads = len(read_len)
        self.n_alns = len(alns) - 1 if n_alns is None else int(n_alns)
        self.n_segs = int(alns["seg_off"][-1]) if n_segs is None else int(n_segs)
        self.used = used
        self.c = A.SxAlignBatch(
            n_regions=self.n_regions, n_reads=self.n_reads, n_alns=self.n_alns, n_segs=self.n_segs,
            regions=A.ptr(regions), read_len=A.ptr(read_len), seq4=A.ptr(seq4), qual=A.ptr(qual), ref=A.ptr(ref), alns=A.ptr(alns), segs=A.ptr(segs), ins=A.ptr(ins),
            seq4_bytes=used["seq4"], qual_bytes=used["qual"], ref_bytes=used["ref"], ins_bytes=used["ins"], qual_bits=qual_bits, qual_dict=self.qual_dict, format=fmt,
            exc_off=A.ptr(exc_off), exc=A.ptr(exc),
        )

    def cells(self) -> int:
        """SURVEY 8a cell-update count: read bases in MATCH/INSERT segments over all alignments."""
        s = self.segs[: self.n_segs]
        if self.fmt & A.SX_FMT_SEG2:
            kind, ln = (s >> 12) & 7, s & 0xFFF
        else:
            kind, ln = s["kind"], s["len"]
        m = (kind == A.SX_SEG_MATCH) | (kind == A.SX_SEG_INSERT)
        return int(ln[m].astype(np.int64).sum())

    def algorithmic_bytes(self) -> int:
        """SURVEY 8d K1 bytes: each read once (packed bases + quals), headers, segments, inserted bases, ref windows, 8 B out/aln."""
        return int(
            self.used["seq4"] + self.used["qual"] + self.used["ref"] + self.used["ins"] + (0 if self.exc_off is None else 4 * (self.n_regions + int(self.exc_off[-1])))
            + self.n_alns * (self.alns.dtype.itemsize + 8) + self.n_segs * self.segs.dtype.itemsize
            + self.n_reads * 2 + self.n_regions * A.REGION_DT.itemsize
        )


def build_align_batch(regions: Sequence[RegionSpec], qual_bits: int = 8, compact: bool = False) -> AlignBatch:
    """qual_bits=4 sends qualities dictionary-coded, two per byte (needs <= 16 distinct values in the batch); qual_bits=2 one
    2-bit code per nibble position of the seq4 stream (<= 4 distinct values).  compact=True sends alignment headers and segments in
    the 8-byte / 2-byte wire formats (SX_FMT_ALN8 | SX_FMT_SEG2)."""
    qdict = None
    if qual_bits in (2, 4):
        vals = sorted({int(x) for r in regions for _, q in r.reads for x in np.asarray(q).tolist()})
        assert len(vals) <= (1 << qual_bits), "%d-bit quality coding needs at most %d distinct quality values" % (qual_bits, 1 << qual_bits)
        qdict = vals
        qcode = {v: i for i, v in enumerate(vals)}
    seg_align = 8 if compact else 4
    # base and quality in one nibble (SX_FMT_BASEQ): needs the 2-bit dictionary and no quality the reference would reject
    baseq = bool(compact and qual_bits == 2 and (not qdict or max(qdict) <= 70))
    exc: List[int] = []
    exc_off: List[int] = []
    reg = np.zeros(len(regions) + 1, dtype=A.REGION_DT)
    q2_codes: List[int] = []
    read_len: List[int] = []
    seq4 = bytearray()
    qual = bytearray()
    ref = bytearray()
    ins = bytearray()
    alns: List[Tuple[int, int, int, int]] = []
    segs: List[Tuple[int, int, int]] = []
    for ri, r in enumerate(regions):
        for pool in (seq4, qual, ref, ins):
            pool.extend(b"\0" * (_pad16(len(pool)) - len(pool)))
        while len(segs) % seg_align:
            segs.append((0, A.SX_SEG_HARDCLIP, 0))  # no-op pad, absorbed by the previous region's last alignment
        if qual_bits == 2 and not baseq:
            qual.extend(_pack2(q2_codes))
            qual.extend(b"\0" * (_pad16(len(qual)) - len(qual)))
            q2_codes = []
        exc_off.append(len(exc))
        region_seq0 = len(seq4)
        reg[ri] = (len(seq4), len(qual), len(ref), len(read_len), len(alns), len(segs), len(ins), r.ref_begin, len(r.ref))
        ref.extend(r.ref.encode())
        rbase = len(read_len)
        for codes, q in r.reads:
            n = len(codes)
            assert len(q) == n
            read_len.append(n)
            c = np.asarray(codes, dtype=np.uint8)
            if baseq:
                qc = np.array([qcode[int(x)] for x in np.asarray(q).tolist()], dtype=np.uint8)
                base = np.select([c == 1, c == 2, c == 4, c == 8], [0, 1, 2, 3], default=255).astype(np.uint8)
                pos0 = 2 * (len(seq4) - region_seq0)
                for i in np.nonzero(base == 255)[0].tolist():
                    exc.append(int(pos0 + i) | (int(c[i]) << 24))  # SX_EXC
                c = (np.where(base == 255, 0, base).astype(np.uint8) << 2) | qc
            if n & 1:
                c = np.concatenate([c, np.zeros(1, np.uint8)])
            seq4.extend(((c[0::2] << 4) | c[1::2]).astype(np.uint8).tobytes())
            if baseq:
                pass
            elif qual_bits == 4:
                qc = np.array([qcode[int(x)] for x in np.asarray(q).tolist()], dtype=np.uint8)
                if n & 1:
                    qc = np.concatenate([qc, np.zeros(1, np.uint8)])
                qual.extend(((qc[0::2] << 4) | qc[1::2]).astype(np.uint8).tobytes())
            elif qual_bits == 2:
                q2_codes.extend(qcode[int(x)] for x in np.asarray(q).tolist())
                if n & 1:
                    q2_codes.append(0)  # the pad nibble of an odd-length read has a (don't-care) code too
            else:
                qual.extend(np.asarray(q, dtype=np.uint8).tobytes())
        order = sorted(range(len(r.alns)), key=lambda k: r.alns[k].read)
        assert order == list(range(len(r.alns))), "alignments of a region must be sorted by read"
        for cal in r.alns:
            s, ib = flatten_alignment(cal)
            alns.append((rbase + cal.read, cal.pos, len(segs), len(ins)))
            segs.extend(s)
            ins.extend(ib)
    if qual_bits == 2 and not baseq:
        qual.extend(_pack2(q2_codes))
    exc_off.append(len(exc))
    for pool in (seq4, qual, ref, ins):
        pool.extend(b"\0" * (_pad16(len(pool)) - len(pool)))
    while len(segs) % seg_align:
        segs.append((0, A.SX_SEG_HARDCLIP, 0))
    used = {"seq4": len(seq4), "qual": len(qual), "ref": len(ref), "ins": len(ins)}
    reg[len(regions)] = (len(seq4), len(qual), len(ref), len(read_len), len(alns), len(segs), len(ins), 0, 0)
    alns.append((len(read_len), 0, len(segs), len(ins)))
    slack = b"\0" * A.SX_POOL_SLACK
    aln_arr = np.array(alns, dtype=A.ALN_DT)
    seg_arr = np.zeros(len(segs) + 16, dtype=A.ALN_SEG_DT)
    if segs:
        seg_arr[: len(segs)] = np.array(segs, dtype=A.ALN_SEG_DT)
    seg_arr["kind"][len(segs):] = A.SX_SEG_HARDCLIP
    fmt = 0
    n_segs = len(segs)
    if compact:
        # region of every alignment, then every field relative to it
        ri_of = np.searchsorted(reg["aln_begin"][1:], np.arange(len(alns) - 1), side="right")
        a8 = np.zeros(len(alns) + 2, dtype=A.ALN8_DT)  # + 16 bytes of slack: the kernels load the slice from a 16-byte boundary
        rel = {
            "read": aln_arr["read"][:-1].astype(np.int64) - reg["read_begin"][ri_of],
            "ref_pos": aln_arr["ref_pos"][:-1].astype(np.int64) - reg["ref_begin"][ri_of],
            "seg_off": aln_arr["seg_off"][:-1].astype(np.int64) - reg["seg_begin"][ri_of],
            "ins_off": aln_arr["ins_off"][:-1].astype(np.int64) - reg["ins_begin"][ri_of],
        }
        fits = all(int(v.min(initial=0)) >= (-32768 if k == "ref_pos" else 0) and int(v.max(initial=0)) <= (32767 if k == "ref_pos" else 65535) for k, v in rel.items())
        if fits:
            for k, v in rel.items():
                a8[k][: len(alns) - 1] = v
            aln_arr = a8
            fmt |= A.SX_FMT_ALN8
        if int(seg_arr["len"].max(initial=0)) <= 4095:
            seg_arr = (seg_arr["len"].astype(np.uint16) | (seg_arr["kind"].astype(np.uint16) << 12) | (seg_arr["flags"].astype(np.uint16) << 15)).astype(np.uint16)
            fmt |= A.SX_FMT_SEG2
        if baseq:
            fmt |= A.SX_FMT_BASEQ
        # reference windows as BAM 4-bit codes (SX_FMT_REF4): repack window by window at new 16-byte aligned offsets
        code_of_char = np.full(256, 15, np.uint8)
        for ch, cd in zip(b"ACGT", (1, 2, 4, 8)):
            code_of_char[ch] = cd
        ref_arr = np.frombuffer(bytes(ref), dtype=np.uint8)
        ref4 = bytearray()
        for ri in range(len(regions)):
            ref4.extend(b"\0" * (_pad16(len(ref4)) - len(ref4)))
            o, n_ref = int(reg["ref_off"][ri]), int(reg["ref_len"][ri])
            reg["ref_off"][ri] = len(ref4)
            cw = code_of_char[ref_arr[o: o + n_ref]]
            if n_ref & 1:
                cw = np.concatenate([cw, np.zeros(1, np.uint8)])
            ref4.extend(((cw[0::2] << 4) | cw[1::2]).astype(np.uint8).tobytes())
        ref4.extend(b"\0" * (_pad16(len(ref4)) - len(ref4)))
        reg["ref_off"][len(regions)] = len(ref4)
        ref = ref4
        used["ref"] = len(ref4)
        fmt |= A.SX_FMT_REF4
    return AlignBatch(
        reg,
        np.array(read_len, dtype=np.uint16),
        np.frombuffer(bytes(seq4) + slack, dtype=np.uint8).copy(),
        np.frombuffer(bytes(qual) + slack, dtype=np.uint8).copy(),
        np.frombuffer(bytes(ref) + slack, dtype=np.uint8).copy(),
        aln_arr,
        seg_arr,
        np.frombuffer(bytes(ins) + slack, dtype=np.uint8).copy(),
        used,
        qual_bits,
        qdict,
        fmt,
        n_segs,
        len(alns) - 1,
        np.array(exc_off, dtype=np.uint32) if baseq else None,
        np.array(exc + [0], dtype=np.uint32) if baseq else None,
    )


def _pack2(codes) -> bytes:
    """2-bit codes -> bytes, first code in the two high bits."""
    c = np.asarray(list(codes) + [0] * (-len(codes) % 4), dtype=np.uint8).reshape(-1, 4)
    return ((c[:, 0] << 6) | (c[:, 1] << 4) | (c[:, 2] << 2) | c[:, 3]).astype(np.uint8).tobytes()


# ------------------------------------------------------------------------------------------------------------------
# pileups
# ------------------------------------------------------------------------------------------------------------------
def pack_call(q, base_id, fwd, nbr_mm=0, filt=0, tfilt=0):
    """base_call bit layout, blt_common/snp_pos_info.hh:109-118 (works on scalars and numpy arrays)."""
    return (
        (np.asarray(q, dtype=np.uint16) & 63)
        | ((np.asarray(base_id, dtype=np.uint16) & 15) << 6)
        | ((np.asarray(fwd, dtype=np.uint16) & 1) << 10)
        | ((np.asarray(nbr_mm, dtype=np.uint16) & 1) << 11)
        | ((np.asarray(filt, dtype=np.uint16) & 1) << 12)
        | ((np.asarray(tfilt, dtype=np.uint16) & 1) << 13)
    ).astype(np.uint16)


class PileupBatch:
    def __init__(self, site_off, calls, ref_base, ploidy=None, t2_off=None, t2_calls=None):
        self.site_off = np.ascontiguousarray(site_off, dtype=np.uint32)
        self.calls = np.ascontiguousarray(calls, dtype=np.uint16)
        self.ref_base = np.ascontiguousarray(ref_base, dtype=np.uint8)
        self.ploidy = None if ploidy is None else np.ascontiguousarray(ploidy, dtype=np.uint8)
        self.t2_off = None if t2_off is None else np.ascontiguousarray(t2_off, dtype=np.uint32)
        self.t2_calls = None if t2_calls is None else np.ascontiguousarray(t2_calls, dtype=np.uint16)
        if self.calls.size == 0:
            self.calls = np.zeros(1, np.uint16)
        if self.t2_calls is not None and self.t2_calls.size == 0:
            self.t2_calls = np.zeros(1, np.uint16)
        self.n_sites = len(self.site_off) - 1
        assert len(self.ref_base) == self.n_sites
        self.c = A.SxPileupBatch(n_sites=self.n_sites, site_off=A.ptr(self.site_off), calls=A.ptr(self.calls), t2_off=A.ptr(self.t2_off), t2_calls=A.ptr(self.t2_calls),
                                 ref_base=A.ptr(self.ref_base), ploidy=A.ptr(self.ploidy))

    @property
    def n_calls(self) -> int:
        return int(self.site_off[-1])

    @staticmethod
    def from_sites(sites: Sequence[Sequence[int]], ref_bases: str, ploidy=None, t2_sites=None) -> "PileupBatch":
        off = np.zeros(len(sites) + 1, np.uint32)
        off[1:] = np.cumsum([len(s) for s in sites])
        calls = np.array([c for s in sites for c in s], dtype=np.uint16)
        t2_off = t2_calls = None
        if t2_sites is not None:
            t2_off = np.zeros(len(sites) + 1, np.uint32)
            t2_off[1:] = np.cumsum([len(s) for s in t2_sites])
            t2_calls = np.array([c for s in t2_sites for c in s], dtype=np.uint16)
        return PileupBatch(off, calls, np.frombuffer(ref_bases.encode(), dtype=np.uint8), ploidy, t2_off, t2_calls)


class ContBatch:
    """K2c's input: S PileupBatch samples over the same n_sites consecutive positions from pos_begin, and the forced-output flags (or None).
    Only sample 0's ref_base is read."""

    def __init__(self, samples: Sequence[PileupBatch], pos_begin: int = 0, forced_output=None):
        assert 1 <= len(samples) <= A.SX_CONT_MAX_SAMPLES
        self.samples = list(samples)
        self.n_sites = self.samples[0].n_sites
        assert all(p.n_sites == self.n_sites for p in self.samples)
        self.n_samples = len(self.samples)
        self.pos_begin = int(pos_begin)
        self.forced_output = None if forced_output is None else np.ascontiguousarray(forced_output, dtype=np.uint8)
        assert self.forced_output is None or self.forced_output.size == self.n_sites
        self.c = A.SxContBatch(n_sites=self.n_sites, n_samples=self.n_samples, pos_begin=self.pos_begin, forced_output=A.ptr(self.forced_output))
        for k, p in enumerate(self.samples):
            self.c.sample[k] = p.c


class ContOut:
    """K2c's output arrays (host): records, their (record, sample) entries, per-site record offsets and the total."""

    def __init__(self, n_sites: int, n_samples: int, cap_loci: int):
        self.n_samples, self.cap_loci = n_samples, int(cap_loci)
        self.loci = np.zeros(max(1, self.cap_loci), A.CONT_LOCUS_DT)
        self.samples = np.zeros(max(1, self.cap_loci * n_samples), A.CONT_SAMPLE_DT)
        self.site_rec_off = np.zeros(n_sites + 1, np.uint32)
        self.totals = np.zeros(1, np.uint32)
        self.c = A.SxContOut(loci=A.ptr(self.loci), samples=A.ptr(self.samples), site_rec_off=A.ptr(self.site_rec_off), cap_loci=self.cap_loci)

    def trimmed(self):
        """(records, entries [records, n_samples], site_rec_off)"""
        n = int(self.totals[0])
        return self.loci[:n], self.samples[: n * self.n_samples].reshape(n, self.n_samples), self.site_rec_off


def cont_cap(b: ContBatch) -> int:
    """an upper bound of K2c's record count: four per site (an 'N' reference's forced site)"""
    return 4 * b.n_sites


class GaBatch:
    def __init__(self, queries: Sequence[str], refs: Sequence[str], max_ops: int = 64):
        assert len(queries) == len(refs)
        self.n = len(queries)
        self.query = np.frombuffer(("".join(queries) + "\0" * 16).encode(), dtype=np.uint8).copy()
        self.ref = np.frombuffer(("".join(refs) + "\0" * 16).encode(), dtype=np.uint8).copy()
        self.query_off = np.zeros(self.n + 1, np.uint32)
        self.query_off[1:] = np.cumsum([len(q) for q in queries])
        self.ref_off = np.zeros(self.n + 1, np.uint32)
        self.ref_off[1:] = np.cumsum([len(r) for r in refs])
        self.max_ops = max_ops
        self.c = A.SxGaBatch(n=self.n, query=A.ptr(self.query), ref=A.ptr(self.ref), query_off=A.ptr(self.query_off), ref_off=A.ptr(self.ref_off), max_ops=max_ops)

    def cells(self) -> int:
        q = np.diff(self.query_off).astype(np.int64)
        r = np.diff(self.ref_off).astype(np.int64)
        return int((q * r).sum()) * 3


def cigar_string(ops: np.ndarray) -> str:
    return "".join(f"{int(o) >> 4}{'MIDNSHP=X'[int(o) & 15]}" for o in ops)


class IndelBatch:
    """sx_indel_batch: per locus an orthogonal allele group (A non-ref indel alleles) and, per supporting read, the flat allele
    log-likelihood vector {ref, alt1..altA} (ReadPathScores floats), read_length, nonAmbiguousBasesInRead, strand."""

    def __init__(self, loci):
        """loci: list of dicts {ploidy, alleles: [(del_len, ins_len)], reads: [(lnp[A+1], read_length, non_ambig, is_fwd)]}"""
        n = len(loci)
        self.n_loci = n
        self.read_off = np.zeros(n + 1, np.uint32)
        self.lnp_off = np.zeros(n + 1, np.uint32)
        self.allele_off = np.zeros(n + 1, np.uint32)
        self.ploidy = np.array([l["ploidy"] for l in loci], np.uint8)
        dl, il, lnp, rl, na, fw = [], [], [], [], [], []
        for i, l in enumerate(loci):
            A_ = len(l["alleles"])
            self.read_off[i + 1] = self.read_off[i] + len(l["reads"])
            self.lnp_off[i + 1] = self.lnp_off[i] + len(l["reads"]) * (A_ + 1)
            self.allele_off[i + 1] = self.allele_off[i] + A_
            for d, ins in l["alleles"]:
                dl.append(d)
                il.append(ins)
            for v, rlen, nonamb, fwd in l["reads"]:
                assert len(v) == A_ + 1
                lnp.extend(v)
                rl.append(rlen)
                na.append(nonamb)
                fw.append(fwd)
        pad = lambda a, dt: np.array(a if len(a) else [0], dtype=dt)
        self.allele_del_len, self.allele_ins_len = pad(dl, np.uint16), pad(il, np.uint16)
        self.allele_lnp, self.read_length, self.non_ambig, self.is_fwd = pad(lnp, np.float32), pad(rl, np.uint16), pad(na, np.uint16), pad(fw, np.uint8)
        if self.ploidy.size == 0:
            self.ploidy = np.zeros(1, np.uint8)
        self.c = A.SxIndelBatch(n_loci=n, read_off=A.ptr(self.read_off), lnp_off=A.ptr(self.lnp_off), allele_off=A.ptr(self.allele_off), ploidy=A.ptr(self.ploidy),
                                allele_del_len=A.ptr(self.allele_del_len), allele_ins_len=A.ptr(self.allele_ins_len), allele_lnp=A.ptr(self.allele_lnp),
                                read_length=A.ptr(self.read_length), non_ambig=A.ptr(self.non_ambig), is_fwd=A.ptr(self.is_fwd))

    @staticmethod
    def from_arrays(read_off, lnp_off, allele_off, ploidy, allele_del_len, allele_ins_len, allele_lnp, read_length, non_ambig, is_fwd) -> "IndelBatch":
        """An IndelBatch over flat arrays (the K6g link's output)."""
        ib = IndelBatch.__new__(IndelBatch)
        ib.n_loci = int(np.asarray(read_off).size - 1)
        for k, v, dt in (("read_off", read_off, np.uint32), ("lnp_off", lnp_off, np.uint32), ("allele_off", allele_off, np.uint32), ("ploidy", ploidy, np.uint8),
                         ("allele_del_len", allele_del_len, np.uint16), ("allele_ins_len", allele_ins_len, np.uint16), ("allele_lnp", allele_lnp, np.float32),
                         ("read_length", read_length, np.uint16), ("non_ambig", non_ambig, np.uint16), ("is_fwd", is_fwd, np.uint8)):
            a = np.ascontiguousarray(v, dt)
            setattr(ib, k, a if a.size else np.zeros(1, dt))
        ib.c = A.SxIndelBatch(n_loci=ib.n_loci, **{k: A.ptr(getattr(ib, k)) for k in ("read_off", "lnp_off", "allele_off", "ploidy", "allele_del_len", "allele_ins_len",
                                                                                       "allele_lnp", "read_length", "non_ambig", "is_fwd")})
        return ib


# ------------------------------------------------------------------------------------------------------------------
# K5b somatic_indel
# ------------------------------------------------------------------------------------------------------------------
class SomaticIndelBatch:
    """sx_sindel_batch plus its host error-rate table.  Built from flat arrays (`SomaticIndelBatch(...)`) or from per-locus dicts
    (`SomaticIndelBatch.from_loci`)."""

    def __init__(self, key, is_forced_output, err_idx, err_prob, alt_off, alts, read_off, reads):
        self.key = np.ascontiguousarray(key, A.INDEL_KEY_DT)
        self.n_loci = n = self.key.size
        self.is_forced_output = np.ascontiguousarray(is_forced_output, np.uint8)
        self.err_idx = np.ascontiguousarray(err_idx, np.uint32)
        self.err_prob = np.ascontiguousarray(err_prob, np.float64)
        self.alt_off = np.ascontiguousarray(alt_off, np.uint32)
        self.alts = np.ascontiguousarray(alts, A.INDEL_KEY_DT)
        self.read_off = np.ascontiguousarray(read_off, np.uint32)
        self.reads = np.ascontiguousarray(reads, A.SINDEL_READ_DT)
        assert self.is_forced_output.size == n and self.err_idx.size == n and self.alt_off.size == n + 1 and self.read_off.size == 2 * n + 1
        assert self.alt_off[-1] == self.alts.size and self.read_off[-1] == self.reads.size
        self._keep = [a if a.size else np.zeros(1, a.dtype) for a in (self.key, self.is_forced_output, self.err_idx, self.alts, self.reads)]
        k, f, e, al, rd = self._keep
        self.c = A.SxSindelBatch(n_loci=n, key=A.ptr(k), is_forced_output=A.ptr(f), err_idx=A.ptr(e), alt_off=A.ptr(self.alt_off), alts=A.ptr(al), read_off=A.ptr(self.read_off),
                                 reads=A.ptr(rd))

    @staticmethod
    def from_loci(loci) -> "SomaticIndelBatch":
        """loci: dicts {key: (pos, del_len, ins_len), forced, err_prob, alts: [(pos, del_len, ins_len, ins_id)] (distinct keys),
        reads: ([normal reads], [tumor reads])}, a read being (ref, indel, read_length, non_ambig, is_tier1, [(alt index, lnp)] <= 2),
        in read_path_lnp order.  Equal error probabilities share one table entry."""
        n = len(loci)
        key = np.zeros(n, A.INDEL_KEY_DT)
        forced = np.zeros(n, np.uint8)
        err_idx = np.zeros(n, np.uint32)
        table: dict = {}
        alt_off = np.zeros(n + 1, np.uint32)
        read_off = np.zeros(2 * n + 1, np.uint32)
        alts, reads = [], []
        for i, l in enumerate(loci):
            key[i]["pos"], key[i]["del_len"], key[i]["ins_len"] = l["key"]
            forced[i] = 1 if l.get("forced") else 0
            err_idx[i] = table.setdefault(float(l["err_prob"]), len(table))
            alts.extend(l["alts"])
            alt_off[i + 1] = alt_off[i] + len(l["alts"])
            for s in range(2):
                reads.extend(l["reads"][s])
                read_off[2 * i + s + 1] = read_off[2 * i + s] + len(l["reads"][s])
        ak = np.zeros(len(alts), A.INDEL_KEY_DT)
        for j, (pos, dl, il, ins_id) in enumerate(alts):
            ak[j]["pos"], ak[j]["del_len"], ak[j]["ins_len"], ak[j]["ins_id"] = pos, dl, il, ins_id
        rd = np.zeros(len(reads), A.SINDEL_READ_DT)
        for j, (ref, indel, rlen, nonamb, t1, ra) in enumerate(reads):
            r = rd[j]
            r["ref"], r["indel"], r["read_length"], r["non_ambig"], r["is_tier1"], r["n_alt"] = ref, indel, rlen, nonamb, 1 if t1 else 0, len(ra)
            for k, (a, lnp) in enumerate(ra[:2]):
                r["alt"][k], r["alt_lnp"][k] = a, lnp
        err = np.array(sorted(table, key=table.get), np.float64)
        return SomaticIndelBatch(key, forced, err_idx, err, alt_off, ak, read_off, rd)


# ------------------------------------------------------------------------------------------------------------------
# K6b indel_reads
# ------------------------------------------------------------------------------------------------------------------
class IndelReadsSample:
    """One sample's side of sx_link_indel_reads: the K6 batch's read arrays, K6's output as it left the device (record slots at rec_off,
    n_rec of them used per read), the batch-wide id of every window entry and the reads' ids (None: the read's index)."""

    def __init__(self, sb, recs, n_rec, key_gid, read_id=None):
        n = sb.n_reads
        self.n_regions, self.n_reads, self.n_keys = sb.n_regions, n, sb.n_keys
        self.region_read_off, self.region_key_off, self.rec_off = sb.region_read_off, sb.region_key_off, sb.rec_off
        self.read_len, self.non_ambig, self.read_flags = sb.read_len, sb.non_ambig, sb.read_flags
        self.recs = np.ascontiguousarray(recs, A.READ_INDEL_SCORE_DT)
        self.n_rec = np.ascontiguousarray(n_rec, np.uint32)
        self.key_gid = np.ascontiguousarray(key_gid, np.uint32)
        self.read_id = None if read_id is None else np.ascontiguousarray(read_id, np.uint32)
        assert self.recs.size >= int(sb.rec_off[n]) and self.n_rec.size >= n and self.key_gid.size >= sb.n_keys
        assert self.read_id is None or self.read_id.size >= n
        self._keep = [a if a.size else np.zeros(1, a.dtype) for a in (self.recs, self.n_rec, self.key_gid)]
        rc, nr, kg = self._keep
        self.c = A.SxIndelReadsSample(n_regions=self.n_regions, n_reads=n, n_keys=self.n_keys, region_read_off=A.ptr(self.region_read_off),
                                      region_key_off=A.ptr(self.region_key_off), key_gid=A.ptr(kg), rec_off=A.ptr(self.rec_off), recs=A.ptr(rc), n_rec=A.ptr(nr),
                                      read_len=A.ptr(self.read_len), non_ambig=A.ptr(self.non_ambig), read_flags=A.ptr(self.read_flags), read_id=A.ptr(self.read_id))


class IndelLoci:
    """sx_indel_loci: the candidates to call (ascending id) and the table of every id's entry; err_prob is K5b's host error-rate table."""

    def __init__(self, gid, key, is_forced_output, err_idx, gid_key, err_prob):
        self.gid = np.ascontiguousarray(gid, np.uint32)
        self.n_loci = n = self.gid.size
        self.key = np.ascontiguousarray(key, A.INDEL_KEY_DT)
        self.is_forced_output = np.ascontiguousarray(is_forced_output, np.uint8)
        self.err_idx = np.ascontiguousarray(err_idx, np.uint32)
        self.gid_key = np.ascontiguousarray(gid_key, A.INDEL_KEY_DT)
        self.n_gid = self.gid_key.size
        self.err_prob = np.ascontiguousarray(err_prob, np.float64)
        assert self.key.size == n and self.is_forced_output.size == n and self.err_idx.size == n
        self._keep = [a if a.size else np.zeros(1, a.dtype) for a in (self.gid, self.key, self.is_forced_output, self.err_idx, self.gid_key)]
        g, k, f, e, gk = self._keep
        self.c = A.SxIndelLoci(n_loci=n, n_gid=self.n_gid, gid=A.ptr(g), key=A.ptr(k), is_forced_output=A.ptr(f), err_idx=A.ptr(e), gid_key=A.ptr(gk))


class IndelReadsOut:
    """sx_indel_reads_out with capacities; `batch(loci)` is the sx_sindel_batch it forms with the loci."""

    def __init__(self, n_loci, cap_reads, cap_alts):
        self.n_loci = n_loci
        self.alt_off = np.zeros(n_loci + 1, np.uint32)
        self.alts = np.zeros(max(1, cap_alts), A.INDEL_KEY_DT)
        self.read_off = np.zeros(2 * n_loci + 1, np.uint32)
        self.reads = np.zeros(max(1, cap_reads), A.SINDEL_READ_DT)
        self.status = np.zeros(max(1, n_loci), np.uint32)
        self.totals = np.zeros(2, np.uint32)
        self.c = A.SxIndelReadsOut(alt_off=A.ptr(self.alt_off), alts=A.ptr(self.alts), read_off=A.ptr(self.read_off), reads=A.ptr(self.reads), status=A.ptr(self.status),
                                   totals=A.ptr(self.totals), cap_alts=cap_alts, cap_reads=cap_reads)

    def trimmed(self):
        """(alt_off, alts, read_off, reads, status, totals) without the unused capacity."""
        return (self.alt_off, self.alts[: int(self.totals[1])], self.read_off, self.reads[: int(self.totals[0])], self.status[: self.n_loci], self.totals)

    def batch(self, loci: IndelLoci) -> SomaticIndelBatch:
        alt_off, alts, read_off, reads, _, _ = self.trimmed()
        return SomaticIndelBatch(loci.key, loci.is_forced_output, loci.err_idx, loci.err_prob, alt_off, alts, read_off, reads)


def link_indel_reads(normal: IndelReadsSample, tumor: IndelReadsSample, loci: IndelLoci) -> IndelReadsOut:
    """Host restatement of sx_link_indel_reads with dicts, the way the reference's containers do it: read_path_lnp[read id] = entry per
    (locus, sample), walked in key order.  A second check beside the oracle; not a fast path."""
    locus_of = {int(g): l for l, g in enumerate(loci.gid)}
    lists = [({}, {}) for _ in range(loci.n_loci)]
    dup = np.zeros(loci.n_loci, bool)
    for s, sm in enumerate((normal, tumor)):
        region = np.repeat(np.arange(sm.n_regions), np.diff(sm.region_read_off[: sm.n_regions + 1]).astype(np.int64))
        for r in range(sm.n_reads):
            k0 = int(sm.region_key_off[region[r]]) if sm.n_rec[r] else 0
            rid = r if sm.read_id is None else int(sm.read_id[r])
            for rec in sm.recs[int(sm.rec_off[r]) : int(sm.rec_off[r]) + int(sm.n_rec[r])]:
                if not rec["flags"] & A.SX_RIS_SCORED:
                    continue
                l = locus_of.get(int(sm.key_gid[k0 + int(rec["key"])]))
                if l is None:
                    continue
                dup[l] |= rid in lists[l][s]
                n_alt = int(rec["n_alt"])
                lists[l][s][rid] = (rec, r, [int(sm.key_gid[k0 + int(rec["alt_key"][a])]) for a in range(n_alt)])
    alts_of = [sorted({g for d in ls for _, _, ids in d.values() for g in ids}) for ls in lists]
    status = np.array([(A.SX_INDEL_READS_ST_DUP_READ if dup[l] else 0) | (A.SX_SINDEL_ST_CAP if len(alts_of[l]) > A.SX_SINDEL_MAX_ALTS else 0)
                       for l in range(loci.n_loci)], np.uint32)
    n_reads = sum(len(d) for l, ls in enumerate(lists) if not status[l] for d in ls)
    n_alts = sum(len(a) for l, a in enumerate(alts_of) if not status[l])
    out = IndelReadsOut(loci.n_loci, n_reads, n_alts)
    out.status[: loci.n_loci] = status
    out.totals[:] = (n_reads, n_alts)
    at = aa = 0
    for l, ls in enumerate(lists):
        out.alt_off[l] = aa
        for s, (sm, d) in enumerate(zip((normal, tumor), ls)):
            out.read_off[2 * l + s] = at
            if status[l]:
                continue
            for rid in sorted(d):
                rec, r, ids = d[rid]
                e = out.reads[at]
                e["ref"], e["indel"], e["read_length"], e["non_ambig"] = rec["ref_lnp"], rec["indel_lnp"], sm.read_len[r], sm.non_ambig[r]
                e["is_tier1"], e["n_alt"] = 1 if sm.read_flags[r] & A.SX_SIF_TIER1 else 0, len(ids)
                for a, g in enumerate(ids):
                    e["alt"][a], e["alt_lnp"][a] = alts_of[l].index(g), rec["alt_lnp"][a]
                at += 1
        if not status[l]:
            out.alts[aa : aa + len(alts_of[l])] = loci.gid_key[alts_of[l]]
            aa += len(alts_of[l])
    out.alt_off[loci.n_loci], out.read_off[2 * loci.n_loci] = aa, at
    return out


# ------------------------------------------------------------------------------------------------------------------
# K6g allele_groups
# ------------------------------------------------------------------------------------------------------------------
class AlleleGroups:
    """sx_allele_groups: per group its non-reference alleles and contrast alleles as batch-wide ids, and its ploidy; gid_key is the entry of
    every id.  `from_lists` takes one list of ids per group."""

    def __init__(self, allele_off, allele_gid, contrast_off, contrast_gid, ploidy, gid_key):
        self.allele_off = np.ascontiguousarray(allele_off, np.uint32)
        self.allele_gid = np.ascontiguousarray(allele_gid, np.uint32)
        self.contrast_off = np.ascontiguousarray(contrast_off, np.uint32)
        self.contrast_gid = np.ascontiguousarray(contrast_gid, np.uint32)
        self.ploidy = np.ascontiguousarray(ploidy, np.uint8)
        self.gid_key = np.ascontiguousarray(gid_key, A.INDEL_KEY_DT)
        self.n_groups = n = self.ploidy.size
        self.n_gid = self.gid_key.size
        assert self.allele_off.size == n + 1 and self.contrast_off.size == n + 1
        self._keep = [a if a.size else np.zeros(1, a.dtype) for a in (self.allele_gid, self.contrast_gid, self.ploidy, self.gid_key)]
        ag, cg, pl, gk = self._keep
        self.c = A.SxAlleleGroups(n_groups=n, n_gid=self.n_gid, allele_off=A.ptr(self.allele_off), allele_gid=A.ptr(ag), contrast_off=A.ptr(self.contrast_off),
                                  contrast_gid=A.ptr(cg), ploidy=A.ptr(pl), gid_key=A.ptr(gk))

    @staticmethod
    def from_lists(alleles, contrasts, ploidy, gid_key) -> "AlleleGroups":
        off = lambda ls: np.concatenate([[0], np.cumsum([len(x) for x in ls], dtype=np.int64)]).astype(np.uint32)
        flat = lambda ls: np.array([g for x in ls for g in x], np.uint32)
        return AlleleGroups(off(alleles), flat(alleles), off(contrasts), flat(contrasts), ploidy, gid_key)

    def group(self, g: int):
        """(alleles, contrasts, ploidy) of group g"""
        a = self.allele_gid[self.allele_off[g] : self.allele_off[g + 1]]
        c = self.contrast_gid[self.contrast_off[g] : self.contrast_off[g + 1]]
        return [int(x) for x in a], [int(x) for x in c], int(self.ploidy[g])


class AlleleGroupReadsOut:
    """sx_allele_group_reads_out with capacities; `batch()` is the sx_indel_batch (IndelBatch) its arrays form."""

    ARRAYS = ("read_off", "lnp_off", "allele_off", "ploidy", "allele_del_len", "allele_ins_len", "allele_lnp", "read_length", "non_ambig", "is_fwd", "status", "totals")

    def __init__(self, n_groups: int, n_alleles: int, cap_reads: int, cap_lnp: int):
        self.n_groups, self.n_alleles = n_groups, n_alleles
        self.read_off, self.lnp_off, self.allele_off = (np.zeros(n_groups + 1, np.uint32) for _ in range(3))
        self.ploidy = np.zeros(max(1, n_groups), np.uint8)
        self.allele_del_len, self.allele_ins_len = (np.zeros(max(1, n_alleles), np.uint16) for _ in range(2))
        self.allele_lnp = np.zeros(max(1, cap_lnp), np.float32)
        self.read_length, self.non_ambig = (np.zeros(max(1, cap_reads), np.uint16) for _ in range(2))
        self.is_fwd = np.zeros(max(1, cap_reads), np.uint8)
        self.status = np.zeros(max(1, n_groups), np.uint32)
        self.totals = np.zeros(2, np.uint32)
        self.c = A.SxAlleleGroupReadsOut(cap_reads=cap_reads, cap_lnp=cap_lnp, **{k: A.ptr(getattr(self, k)) for k in self.ARRAYS})

    def trimmed(self):
        """Every output array without the unused capacity, in ARRAYS order."""
        n, r, f, a = self.n_groups, int(self.totals[0]), int(self.totals[1]), self.n_alleles
        return (self.read_off, self.lnp_off, self.allele_off, self.ploidy[:n], self.allele_del_len[:a], self.allele_ins_len[:a], self.allele_lnp[:f], self.read_length[:r],
                self.non_ambig[:r], self.is_fwd[:r], self.status[:n], self.totals)

    def batch(self) -> IndelBatch:
        return IndelBatch.from_arrays(*self.trimmed()[:10])


def allele_group_caps(sample: IndelReadsSample, groups: AlleleGroups):
    """Capacities no call exceeds: every scored entry of each group's first allele supports it."""
    n = sample.n_rec[: sample.n_reads].astype(np.int64)
    read_of = np.repeat(np.arange(sample.n_reads), n)
    at = sample.rec_off[read_of].astype(np.int64) + np.arange(read_of.size) - np.repeat(np.cumsum(n) - n, n)
    region = np.repeat(np.arange(sample.n_regions), np.diff(sample.region_read_off[: sample.n_regions + 1]).astype(np.int64))
    scored = (sample.recs["flags"][at] & A.SX_RIS_SCORED) != 0
    key = sample.region_key_off[region[read_of[scored]]].astype(np.int64) + sample.recs["key"][at[scored]]
    cnt = np.bincount(sample.key_gid[np.minimum(key, max(0, sample.key_gid.size - 1))], minlength=groups.n_gid) if key.size else np.zeros(groups.n_gid, np.int64)
    first = groups.allele_gid[groups.allele_off[:-1]] if groups.n_groups else np.zeros(0, np.uint32)
    per = cnt[np.minimum(first, max(0, cnt.size - 1))] if cnt.size else np.zeros(first.size, np.int64)
    return int(per.sum()), int((per * np.diff(groups.allele_off.astype(np.int64)) + per).sum())


def link_allele_groups(sample: IndelReadsSample, groups: AlleleGroups) -> AlleleGroupReadsOut:
    """Host restatement of sx_link_allele_groups with dicts: read_path_lnp[read id] = entry per id, then per group the supporting reads in
    ascending id and their allele log-likelihoods with the contrast fold.  A third check beside the oracle and the kernel body; not a fast
    path.  Raises ValueError where the library refuses the call."""
    named = set(groups.allele_gid.tolist()) | set(groups.contrast_gid.tolist())
    for g in range(groups.n_groups):
        al, co, pl = groups.group(g)
        if not 1 <= len(al) <= A.SX_INDEL_MAX_ALLELES or pl not in (1, 2) or any(x >= groups.n_gid for x in al + co):
            raise ValueError(f"group {g} is outside the link's domain")
    maps = {x: {} for x in named}
    dup = set()
    region = np.repeat(np.arange(sample.n_regions), np.diff(sample.region_read_off[: sample.n_regions + 1]).astype(np.int64))
    for r in range(sample.n_reads):
        k0 = int(sample.region_key_off[region[r]]) if sample.n_rec[r] else 0
        rid = r if sample.read_id is None else int(sample.read_id[r])
        for rec in sample.recs[int(sample.rec_off[r]) : int(sample.rec_off[r]) + int(sample.n_rec[r])]:
            if not rec["flags"] & A.SX_RIS_SCORED:
                continue
            if int(rec["key"]) >= int(sample.region_key_off[region[r] + 1]) - k0 or int(sample.key_gid[k0 + int(rec["key"])]) >= groups.n_gid:
                raise ValueError(f"read {r}: a window index outside its region's window, or an id at or past n_gid")
            m = maps.get(int(sample.key_gid[k0 + int(rec["key"])]))
            if m is None:
                continue
            if rid in m:
                dup.add(int(sample.key_gid[k0 + int(rec["key"])]))
            m[rid] = (float(rec["ref_lnp"]), float(rec["indel_lnp"]), r)
    n_al = int(groups.allele_off[-1])
    rows = []
    status = np.zeros(groups.n_groups, np.uint32)
    for g in range(groups.n_groups):
        al, co, _ = groups.group(g)
        if any(x in dup for x in al + co):
            status[g] = A.SX_INDEL_READS_ST_DUP_READ
            rows.append([])
            continue
        tier1 = lambda rid: sample.read_flags[maps[al[0]][rid][2]] & A.SX_SIF_TIER1
        sup = sorted(rid for rid in maps[al[0]] if tier1(rid) and all(rid in maps[x] for x in al[1:]))
        rows.append([])
        for rid in sup:
            lnp = np.zeros(len(al) + 1, np.float32)
            l0 = None
            for a, x in enumerate(al):
                ref, indel, _ = maps[x][rid]
                l0 = np.float32(ref) if l0 is None else max(l0, np.float32(ref))
                lnp[1 + a] = indel
            for x in co:
                if rid in maps[x]:
                    l0 = max(l0, np.float32(maps[x][rid][0]))
            uncovered = l0
            for x in co:
                v = np.float32(maps[x][rid][1]) if rid in maps[x] else uncovered
                if v > l0:
                    l0 = v
            lnp[0] = l0
            rows[g].append((lnp, maps[al[0]][rid][2]))
    n_reads = sum(len(x) for x in rows)
    n_lnp = sum(len(x) * (len(groups.group(g)[0]) + 1) for g, x in enumerate(rows))
    out = AlleleGroupReadsOut(groups.n_groups, n_al, n_reads, n_lnp)
    out.totals[:] = (n_reads, n_lnp)
    out.status[: groups.n_groups] = status
    out.ploidy[: groups.n_groups] = groups.ploidy
    out.allele_off[:] = groups.allele_off
    out.allele_del_len[:n_al] = groups.gid_key["del_len"][groups.allele_gid]
    out.allele_ins_len[:n_al] = groups.gid_key["ins_len"][groups.allele_gid]
    at = f = 0
    for g, x in enumerate(rows):
        out.read_off[g], out.lnp_off[g] = at, f
        for lnp, r in x:
            out.allele_lnp[f : f + lnp.size] = lnp
            out.read_length[at], out.non_ambig[at] = sample.read_len[r], sample.non_ambig[r]
            out.is_fwd[at] = 1 if sample.read_flags[r] & A.SX_SIF_FWD else 0
            at, f = at + 1, f + lnp.size
    out.read_off[groups.n_groups], out.lnp_off[groups.n_groups] = at, f
    return out


# ------------------------------------------------------------------------------------------------------------------
# K4 pileup_reads
# ------------------------------------------------------------------------------------------------------------------
_PILEUP_KIND = {"M": A.SX_SEG_MATCH, "I": A.SX_SEG_INSERT, "D": A.SX_SEG_DELETE, "N": A.SX_SEG_SKIP, "S": A.SX_SEG_SOFTCLIP, "H": A.SX_SEG_HARDCLIP}


class PileupReadSpec:
    """One read with its best alignment, as pileup_read_segment sees it."""

    def __init__(self, codes, quals, pos, path, fwd=True, mapq=60, tier=1, pins=(False, False)):
        self.codes, self.quals, self.pos, self.path, self.fwd, self.mapq, self.tier, self.pins = codes, quals, pos, path, fwd, mapq, tier, pins


class PileupReadsBatch:
    """Owns the pools of one sx_pileup_reads_batch (reads must be given in pile-up order: ascending position)."""

    def __init__(self, reads: Sequence[PileupReadSpec], ref: str, ref_begin: int, report_begin: int, report_end: int, cand_snv=(), opts=None, buffer_pos=None,
                 qual_dict=None):
        """buffer_pos: the read-buffer position of every read (ascending) when the reads' best alignments are not themselves in pile-up
        order (realigned reads); qual_dict: send the qualities dictionary-coded, two per byte (every quality must be in the dictionary)."""
        self.n_reads = len(reads)
        hdr = np.zeros(len(reads) + 1, dtype=A.PILEUP_READ_DT)
        seq4, qual, segs = bytearray(), bytearray(), []
        span = 1
        for i, r in enumerate(reads):
            n = len(r.codes)
            assert len(r.quals) == n
            flags = (A.SX_PRF_FWD if r.fwd else 0) | (A.SX_PRF_TIER1 if r.tier == 1 else 0) | (A.SX_PRF_TIER1OR2 if r.tier in (1, 2) else 0)
            flags |= (A.SX_PRF_PIN_FIRST if r.pins[0] else 0) | (A.SX_PRF_PIN_SECOND if r.pins[1] else 0)
            hdr[i] = (len(seq4), len(qual), len(segs), r.pos, n, r.mapq, flags)
            c = np.asarray(r.codes, dtype=np.uint8)
            if n & 1:
                c = np.concatenate([c, np.zeros(1, np.uint8)])
            seq4.extend(((c[0::2] << 4) | c[1::2]).astype(np.uint8).tobytes())
            if qual_dict is None:
                qual.extend(np.asarray(r.quals, dtype=np.uint8).tobytes())
            else:
                qc = np.array([qual_dict.index(int(q)) for q in r.quals] + ([0] if n & 1 else []), dtype=np.uint8)
                qual.extend(((qc[0::2] << 4) | qc[1::2]).astype(np.uint8).tobytes())
            segs.extend((ln, _PILEUP_KIND[k], 0) for k, ln in r.path)
            span = max(span, sum(ln for k, ln in r.path if k in "MDN"))
        hdr[len(reads)] = (len(seq4), len(qual), len(segs), 0, 0, 0, 0)
        self.reads = hdr
        self.total_bases = int(hdr["len"].astype(np.int64).sum())
        self.seq4 = np.frombuffer(bytes(seq4) + b"\0" * 64, dtype=np.uint8).copy()
        self.qual = np.frombuffer(bytes(qual) + b"\0" * 64, dtype=np.uint8).copy()
        self.segs = np.zeros(len(segs) + 16, dtype=A.ALN_SEG_DT)
        if segs:
            self.segs[: len(segs)] = np.array(segs, dtype=A.ALN_SEG_DT)
        self.ref = np.frombuffer(ref.encode() + b"\0" * 64, dtype=np.uint8).copy()
        keys = sorted(((p - report_begin) << 2) | b for p, b in cand_snv if report_begin <= p < report_end)
        self.cand_snv = np.array(keys + [0], dtype=np.uint32)
        self.n_sites = report_end - report_begin
        self.opts = opts or A.default_pileup_opts()
        self.c = A.SxPileupReadsBatch(
            n_reads=len(reads), n_segs=len(segs), reads=A.ptr(self.reads), seq4=A.ptr(self.seq4), qual=A.ptr(self.qual), segs=A.ptr(self.segs), ref=A.ptr(self.ref),
            ref_begin=ref_begin, ref_len=len(ref), report_begin=report_begin, report_end=report_end, cand_snv=A.ptr(self.cand_snv), n_cand_snv=len(keys), max_ref_span=span,
            max_read_len=int(hdr["len"].max(initial=1)), opts=self.opts,
        )
        self.buffer_pos = None
        if buffer_pos is not None:
            self.buffer_pos = np.ascontiguousarray(list(buffer_pos) + [0], dtype=np.int32)
            self.c.buffer_pos = A.ptr(self.buffer_pos)
            self.c.max_pos_shift = int(np.abs(self.buffer_pos[: len(reads)].astype(np.int64) - hdr["pos"][: len(reads)].astype(np.int64)).max(initial=0))
        if qual_dict is not None:
            self.c.qual_bits = 4
            self.c.qual_dict = (C.c_uint8 * 16)(*(list(qual_dict) + [0] * (16 - len(qual_dict))))


class PileupColumns:
    """Host buffers for sx_pileup_columns sized for a batch (capacity = total read bases, always enough)."""

    def __init__(self, pb: PileupReadsBatch):
        n, cap = pb.n_sites, pb.total_bases + 16
        self.site_off, self.t2_off = np.zeros(n + 1, np.uint32), np.zeros(n + 1, np.uint32)
        self.calls, self.t2_calls = np.zeros(cap, np.uint16), np.zeros(cap, np.uint16)
        self.n_spandel, self.n_submapped = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
        self.c = A.SxPileupColumns(site_off=A.ptr(self.site_off), calls=A.ptr(self.calls), t2_off=A.ptr(self.t2_off), t2_calls=A.ptr(self.t2_calls),
                                   n_spandel=A.ptr(self.n_spandel), n_submapped=A.ptr(self.n_submapped), calls_capacity=cap, t2_capacity=cap)

    def trimmed(self):
        return (self.site_off, self.calls[: int(self.site_off[-1])], self.t2_off, self.t2_calls[: int(self.t2_off[-1])], self.n_spandel, self.n_submapped)


# ---------------------------------------------------------------------------------------------------------------------------
# K6 score_indels
# ---------------------------------------------------------------------------------------------------------------------------
class WindowKeySpec:
    """One IndelBuffer entry of a region's window (IndelKey + the per-sample facts score_indels reads)."""

    def __init__(self, pos, del_len=0, ins="", mismatch=False, candidate=True, ref_to_indel_lnp=-11.5, indel_to_ref_lnp=-11.5):
        self.pos, self.del_len, self.ins, self.mismatch, self.candidate = pos, del_len, ins, mismatch, candidate
        self.ref_to_indel_lnp, self.indel_to_ref_lnp = ref_to_indel_lnp, indel_to_ref_lnp

    def order(self):
        """IndelKey::operator< (IndelKey.hh:53-76): pos, type, insert length, delete length, insert sequence."""
        return (self.pos, 2 if self.mismatch else 1, len(self.ins), self.del_len, self.ins)


class ScoredReadSpec:
    """A read segment with its candidate alignments: alns = [(pos, [(kind, len)...], [window index...])] in std::set order."""

    def __init__(self, length, alns, fwd=True, tier1=True, non_ambig=None, incomplete=False):
        self.length, self.alns, self.fwd, self.tier1, self.incomplete = length, alns, fwd, tier1, incomplete
        self.non_ambig = length if non_ambig is None else non_ambig


class ScoreIndelsBatch:
    """Owns the arrays of one sx_score_indels_batch.  regions = [(window keys in IndelKey order, reads)]."""

    def __init__(self, regions, opts=None):
        keys, ins_pool, ins_off = [], bytearray(), [0]
        region_read_off, region_key_off = [0], [0]
        aln_off, aln_pos, aln_seg_off, segs, aln_key_off, aln_keys = [0], [], [0], [], [0], []
        read_len, non_ambig, read_flags, rec_off = [], [], [], [0]
        for win, reads in regions:
            assert len(win) <= 65535
            assert all(win[i].order() < win[i + 1].order() for i in range(len(win) - 1)), "window must be in IndelKey order"
            intern = {"": 0}
            for k in win:
                iid = intern.setdefault(k.ins, len(intern))
                keys.append((k.pos, k.del_len, len(k.ins), iid, A.SX_INDEL_TYPE_MISMATCH if k.mismatch else A.SX_INDEL_TYPE_INDEL,
                             A.SX_IKF_CANDIDATE if k.candidate else 0, 0, k.ref_to_indel_lnp, k.indel_to_ref_lnp))
                ins_pool.extend(k.ins.encode())
                ins_off.append(len(ins_pool))
            for r in reads:
                for pos, path, kidx in r.alns:
                    aln_pos.append(pos)
                    segs.extend((ln, _PILEUP_KIND[k], 0) for k, ln in path)
                    aln_seg_off.append(len(segs))
                    assert list(kidx) == sorted(set(kidx)) and all(0 <= i < len(win) for i in kidx)
                    aln_keys.extend(kidx)
                    aln_key_off.append(len(aln_keys))
                aln_off.append(len(aln_pos))
                read_len.append(r.length)
                non_ambig.append(r.non_ambig)
                read_flags.append((A.SX_SIF_FWD if r.fwd else 0) | (A.SX_SIF_TIER1 if r.tier1 else 0) | (A.SX_SIF_INCOMPLETE if r.incomplete else 0))
                rec_off.append(rec_off[-1] + len(win))
            region_read_off.append(len(read_len))
            region_key_off.append(len(keys))
        u32 = lambda x: np.array(x, dtype=np.uint32)  # noqa: E731  (every list starts with its leading 0)
        self.n_regions, self.n_reads, self.n_alns, self.n_keys = len(regions), len(read_len), len(aln_pos), len(keys)
        self.region_read_off, self.region_key_off = u32(region_read_off), u32(region_key_off)
        self.keys = np.zeros(len(keys) + 1, dtype=A.INDEL_KEY_DT)
        if keys:
            self.keys[: len(keys)] = np.array(keys, dtype=A.INDEL_KEY_DT)
        self.aln_off, self.aln_seg_off, self.aln_key_off, self.rec_off = u32(aln_off), u32(aln_seg_off), u32(aln_key_off), u32(rec_off)
        self.aln_pos = np.array(aln_pos + [0], dtype=np.int32)
        self.segs = np.zeros(len(segs) + 16, dtype=A.ALN_SEG_DT)
        if segs:
            self.segs[: len(segs)] = np.array(segs, dtype=A.ALN_SEG_DT)
        self.aln_keys = np.array(aln_keys + [0], dtype=np.uint16)
        self.read_len = np.array(read_len + [0], dtype=np.uint16)
        self.non_ambig = np.array(non_ambig + [0], dtype=np.uint16)
        self.read_flags = np.array(read_flags + [0], dtype=np.uint8)
        self.n_segs, self.n_aln_keys, self.n_rec_slots = len(segs), len(aln_keys), rec_off[-1]
        # test-only: the insert sequences behind ins_id (the reference harness rebuilds IndelKeys from them)
        self.ins_pool = np.frombuffer(bytes(ins_pool) + b"\0", dtype=np.uint8).copy()
        self.ins_off = u32(ins_off)
        self.opts = opts or A.default_score_indels_opts()
        self.c = self._struct()

    def _struct(self) -> A.SxScoreIndelsBatch:
        return A.SxScoreIndelsBatch(
            n_regions=self.n_regions, n_reads=self.n_reads, n_alns=self.n_alns, n_keys=self.n_keys, region_read_off=A.ptr(self.region_read_off),
            region_key_off=A.ptr(self.region_key_off), keys=A.ptr(self.keys), aln_off=A.ptr(self.aln_off), aln_pos=A.ptr(self.aln_pos), aln_seg_off=A.ptr(self.aln_seg_off),
            segs=A.ptr(self.segs), aln_key_off=A.ptr(self.aln_key_off), aln_keys=A.ptr(self.aln_keys), read_len=A.ptr(self.read_len), non_ambig=A.ptr(self.non_ambig),
            read_flags=A.ptr(self.read_flags), rec_off=A.ptr(self.rec_off), opts=self.opts,
        )

    @classmethod
    def from_arrays(cls, arrays: dict, opts=None) -> "ScoreIndelsBatch":
        """Wrap ready-made flat arrays (tools/synth.cpp synth_k6_fill): keys are the sx_score_indels_batch field names."""
        self = cls.__new__(cls)
        for k, v in arrays.items():
            setattr(self, k, v)
        self.n_regions, self.n_reads = len(self.region_read_off) - 1, len(self.aln_off) - 1
        self.n_alns, self.n_keys = int(self.aln_off[-1]), int(self.region_key_off[-1])
        self.n_segs, self.n_aln_keys, self.n_rec_slots = int(self.aln_seg_off[self.n_alns]), int(self.aln_key_off[self.n_alns]), int(self.rec_off[-1])
        self.ins_pool = self.ins_off = None
        self.opts = opts or A.default_score_indels_opts()
        self.c = self._struct()
        return self

    def algorithmic_bytes(self) -> int:
        """bytes one pass must move: every input array once + the scores + one record slot header per read."""
        return (self.n_keys * 32 + self.n_alns * (8 + 4 + 4 + 4) + self.n_segs * 4 + self.n_aln_keys * 2 + self.n_reads * (4 + 2 + 2 + 1 + 4 + 12))


class ScoreIndelsOut:
    """Host buffers for sx_score_indels_out."""

    def __init__(self, sb: ScoreIndelsBatch):
        self.recs = np.zeros(sb.n_rec_slots + 1, dtype=A.READ_INDEL_SCORE_DT)
        self.n_rec = np.zeros(sb.n_reads + 1, np.uint32)
        self.max_aln = np.zeros(sb.n_reads + 1, np.uint32)
        self.eval_aln = np.zeros(sb.n_reads + 1, np.uint32)
        self.c = A.SxScoreIndelsOut(recs=A.ptr(self.recs), n_rec=A.ptr(self.n_rec), max_aln=A.ptr(self.max_aln), eval_aln=A.ptr(self.eval_aln))
        self._sb = sb

    def compact(self):
        """(per-read record lists concatenated, n_rec, max_aln, eval_aln) with the unused slots dropped."""
        sb = self._sb
        parts = [self.recs[int(sb.rec_off[r]) : int(sb.rec_off[r]) + int(self.n_rec[r])] for r in range(sb.n_reads)]
        recs = np.concatenate(parts) if parts else self.recs[:0]
        return recs, self.n_rec[: sb.n_reads].copy(), self.max_aln[: sb.n_reads].copy(), self.eval_aln[: sb.n_reads].copy()


def score_indels_batch_from_regions(regions: Sequence[RegionSpec], fwd=True, ref_to_indel_lnp=-9.903487552536127, indel_to_ref_lnp=-9.903487552536127,
                                    opts=None) -> ScoreIndelsBatch:
    """The K6 view of the regions a K1 batch was built from (same alignment order, so K1's lnp[a] is K6's score of alignment a):
    per region the window = the distinct IndelKeys of its alignments' indel sets (edge keys are not part of cal.getIndels()) in
    IndelKey order; '=' / 'X' path segments are sent as MATCH.  Every alignment of a region must belong to consecutive reads."""
    out = []
    for rg in regions:
        keyspecs = {}
        for cal in rg.alns:
            for i, k in enumerate(cal.indels):
                if i in (cal.leading, cal.trailing):
                    continue
                w = WindowKeySpec(k.pos, k.delete_length, k.insert_seq, k.type == INDEL_MISMATCH, k.is_candidate, ref_to_indel_lnp, indel_to_ref_lnp)
                keyspecs.setdefault(w.order(), w)
        order = sorted(keyspecs)
        index_of = {o: i for i, o in enumerate(order)}
        reads = [ScoredReadSpec(len(codes), [], fwd=fwd, non_ambig=int((np.asarray(codes) != 15).sum())) for codes, _q in rg.reads]
        last = -1
        for cal in rg.alns:
            assert cal.read >= last, "alignments must be grouped by read"
            last = cal.read
            kidx = sorted({index_of[WindowKeySpec(k.pos, k.delete_length, k.insert_seq, k.type == INDEL_MISMATCH).order()]
                           for i, k in enumerate(cal.indels) if i not in (cal.leading, cal.trailing)})
            path = [("M" if t in _ALIGN_MATCH else t, ln) for t, ln in cal.path]
            reads[cal.read].alns.append((cal.pos, path, kidx))
        out.append(([keyspecs[o] for o in order], reads))
    return ScoreIndelsBatch(out, opts)


# ------------------------------------------------------------------------------------------------------------------------------
# K7 enumerate_alignments
# ------------------------------------------------------------------------------------------------------------------------------
_AP_OF = {"M": A.SX_AP_MATCH, "I": A.SX_AP_INSERT, "D": A.SX_AP_DELETE, "N": A.SX_AP_SKIP, "S": A.SX_AP_SOFT_CLIP, "H": A.SX_AP_HARD_CLIP, "=": A.SX_AP_SEQ_MATCH,
          "X": A.SX_AP_SEQ_MISMATCH}
AP_CHAR = {v: k for k, v in _AP_OF.items()}


class EnumKeySpec(WindowKeySpec):
    """A window entry with what the alignment search reads of its IndelData (IndelData.hh:270-273,374,382,387)."""

    def __init__(self, pos, del_len=0, ins="", mismatch=False, candidate=True, not_discovered=False, forced=False, active_region=-1, hap_ids=(0, 0, 0, 0), bypass=0):
        super().__init__(pos, del_len, ins, mismatch, candidate)
        self.not_discovered, self.forced, self.active_region, self.hap_ids, self.bypass = not_discovered, forced, active_region, tuple(hap_ids), bypass


class EnumReadSpec:
    """One read of a K7 batch: bases (ASCII), the normalized input alignment (pos, [(cigar char, len)...]) and the window indices of
    the non-candidate entries the read is an observation of."""

    def __init__(self, seq, pos, path, use_keys=()):
        self.seq, self.pos, self.path, self.use_keys = seq, pos, list(path), sorted(set(use_keys))


_COMPLEMENT_FREE_CODES = {"A": 1, "C": 2, "G": 4, "T": 8}


def alignment_indels(read: EnumReadSpec, ref: str, ref_begin: int, win: Sequence[WindowKeySpec], max_indel_size: int = 49, strict: bool = True):
    """Host side of K7's input (what K7a, sx_alignment_indels, computes on the device): getAlignmentIndels(cal, ref, rseg, maxIndelSize,
    includeMismatches=true) (CandidateAlignment.cpp:58-173) and the edge keys of getCandidateAlignment (starling_read_align.cpp:1481-1522),
    as window indices.  Returns (in_keys, lead, trail).  An indel of the alignment that is not a window entry: KeyError (the reference
    throws, starling_read_align.cpp:1866-1872), or with strict=False the index SX_NO_KEY, which makes K7 answer SX_ENUM_ST_EXCEPTION."""
    index_of = {k.order(): i for i, k in enumerate(win)}

    def find(k):
        w = index_of.get(k.order())
        if w is None:
            if strict:
                raise KeyError(k.order())
            return A.SX_NO_KEY
        return w

    path = read.path
    match_idx = [i for i, (t, _l) in enumerate(path) if t in "M=X"]
    first, last = (match_idx[0], match_idx[-1]) if match_idx else (len(path), len(path))
    keys, lead, trail, has_lead, has_trail = set(), A.SX_NO_KEY, A.SX_NO_KEY, False, False
    read_off, ref_pos = 0, read.pos
    i = 0
    while i < len(path):
        t, ln = path[i]
        edge = i < first or i > last
        # a swap = a run of adjacent insert / delete segments holding BOTH kinds (is_segment_swap_start, align_path.cpp:868-895)
        j, ins_len, del_len = i, 0, 0
        while j < len(path) and path[j][0] in "ID":
            if path[j][0] == "I":
                ins_len += path[j][1]
            else:
                del_len += path[j][1]
            j += 1
        swap = ins_len > 0 and del_len > 0
        step = 1
        if edge:
            if t in "ID":  # getCandidateAlignment sets the edge key for every edge indel segment, the last one wins; it is inserted once
                w = find(WindowKeySpec(ref_pos, ln if t == "D" else 0, read.seq[read_off : read_off + ln] if t == "I" else ""))
                if i < first:
                    lead, has_lead = w, True
                else:
                    trail, has_trail = w, True
        elif swap:
            step = j - i
            keys.add(find(WindowKeySpec(ref_pos, del_len, read.seq[read_off : read_off + ins_len])) if max(ins_len, del_len) <= max_indel_size else A.SX_NO_KEY)
        elif t in "ID":
            keys.add(find(WindowKeySpec(ref_pos, ln if t == "D" else 0, read.seq[read_off : read_off + ln] if t == "I" else "")) if ln <= max_indel_size else A.SX_NO_KEY)
        elif t in "M=X":
            for b in range(ln):
                base = read.seq[read_off + b]
                if base in "=N":  # BAM_BASE::REF and ANY are skipped; every other IUPAC code reads back as 'N' and never equals the reference code
                    continue
                if base not in "ACGT":
                    base = "N"
                rp = ref_pos + b
                rb = ref[rp - ref_begin] if 0 <= rp - ref_begin < len(ref) else "N"
                if base == rb:
                    continue
                w = index_of.get(WindowKeySpec(rp, 1, base, mismatch=True).order())
                if w is not None:  # a mismatch that is no window entry is dropped (starling_read_align.cpp:1865)
                    keys.add(w)
        for s in range(i, i + step):
            st, sl = path[s]
            if st in "MIS=X":
                read_off += sl
            if st in "MDN=X":
                ref_pos += sl
        i += step
    if has_lead:
        keys.add(lead)
    if has_trail:
        keys.add(trail)
    return sorted(keys), lead, trail


class EnumBatch:
    """Owns the arrays of one sx_enum_batch.  regions = [(ref, ref_begin, (realign_begin, realign_end), window keys in IndelKey order, reads)]."""

    def __init__(self, regions, opts=None, strict=True):
        self.opts = opts or A.default_enum_opts()
        keys, hap, ins_pool, ins_off = [], [], bytearray(), [0]
        region_read_off, region_key_off, rb, re_ = [0], [0], [], []
        in_pos, in_seg_off, in_segs, in_key_off, in_keys, use_key_off, use_keys, lead, trail, read_len = [], [0], [], [0], [], [0], [], [], [], []
        ref_pool, ref_off, ref_begin, read_pool, read_off = bytearray(), [0], [], bytearray(), [0]
        any_hap = False
        for ref, rbeg, (ra, rz), win, reads in regions:
            assert all(win[i].order() < win[i + 1].order() for i in range(len(win) - 1)), "window must be in IndelKey order"
            intern = {"": 0}
            for k in win:
                iid = intern.setdefault(k.ins, len(intern))
                flags = (A.SX_IKF_CANDIDATE if k.candidate else 0) | (A.SX_IKF_NOT_DISCOVERED if getattr(k, "not_discovered", False) else 0) | (
                    A.SX_IKF_FORCED_OUTPUT if getattr(k, "forced", False) else 0)
                keys.append((k.pos, k.del_len, len(k.ins), iid, A.SX_INDEL_TYPE_MISMATCH if k.mismatch else A.SX_INDEL_TYPE_INDEL, flags, 0, 0.0, 0.0))
                ar = getattr(k, "active_region", -1)
                any_hap = any_hap or ar >= 0
                hap.append((ar, tuple(getattr(k, "hap_ids", (0, 0, 0, 0))), getattr(k, "bypass", 0), (0, 0, 0)))
                ins_pool.extend(k.ins.encode())
                ins_off.append(len(ins_pool))
            for r in reads:
                ik, ld, tr = alignment_indels(r, ref, rbeg, win, self.opts.max_indel_size, strict)
                in_pos.append(r.pos)
                in_segs.extend((ln, _AP_OF[t], 0) for t, ln in r.path)
                in_seg_off.append(len(in_segs))
                in_keys.extend(ik)
                in_key_off.append(len(in_keys))
                use_keys.extend(r.use_keys)
                use_key_off.append(len(use_keys))
                lead.append(ld)
                trail.append(tr)
                read_len.append(len(r.seq))
                read_pool.extend(r.seq.encode())
                read_off.append(len(read_pool))
            region_read_off.append(len(read_len))
            region_key_off.append(len(keys))
            rb.append(ra)
            re_.append(rz)
            ref_pool.extend(ref.encode())
            ref_off.append(len(ref_pool))
            ref_begin.append(rbeg)
        u32 = lambda x: np.array(x, dtype=np.uint32)  # noqa: E731
        u16 = lambda x: np.array(list(x) + [0], dtype=np.uint16)  # noqa: E731
        self.n_regions, self.n_reads, self.n_keys = len(regions), len(read_len), len(keys)
        self.region_read_off, self.region_key_off = u32(region_read_off), u32(region_key_off)
        self.keys = np.zeros(len(keys) + 1, dtype=A.INDEL_KEY_DT)
        if keys:
            self.keys[: len(keys)] = np.array(keys, dtype=A.INDEL_KEY_DT)
        self.key_hap = np.zeros(len(keys) + 1, dtype=A.KEY_HAP_DT)
        if hap:
            self.key_hap[: len(hap)] = np.array(hap, dtype=A.KEY_HAP_DT)
        self.has_hap = any_hap
        self.realign_begin, self.realign_end = np.array(rb + [0], np.int32), np.array(re_ + [0], np.int32)
        self.in_pos = np.array(in_pos + [0], np.int32)
        self.in_seg_off, self.in_key_off, self.use_key_off = u32(in_seg_off), u32(in_key_off), u32(use_key_off)
        self.in_segs = np.zeros(len(in_segs) + 4, dtype=A.ALN_SEG_DT)
        if in_segs:
            self.in_segs[: len(in_segs)] = np.array(in_segs, dtype=A.ALN_SEG_DT)
        self.in_keys, self.use_keys, self.in_lead_key, self.in_trail_key, self.read_len = u16(in_keys), u16(use_keys), u16(lead), u16(trail), u16(read_len)
        # test-only: what the reference harness needs to rebuild the reference's objects
        self.ins_pool = np.frombuffer(bytes(ins_pool) + b"\0", dtype=np.uint8).copy()
        self.ins_off = u32(ins_off)
        self.ref_pool = np.frombuffer(bytes(ref_pool) + b"\0", dtype=np.uint8).copy()
        self.ref_off, self.ref_begin = u32(ref_off), np.array(ref_begin + [0], np.int32)
        self.read_pool = np.frombuffer(bytes(read_pool) + b"\0", dtype=np.uint8).copy()
        self.read_off = u32(read_off)
        self.c = A.SxEnumBatch(
            n_regions=self.n_regions, n_reads=self.n_reads, n_keys=self.n_keys, region_read_off=A.ptr(self.region_read_off), region_key_off=A.ptr(self.region_key_off),
            keys=A.ptr(self.keys), key_hap=A.ptr(self.key_hap) if any_hap else None, realign_begin=A.ptr(self.realign_begin), realign_end=A.ptr(self.realign_end),
            in_pos=A.ptr(self.in_pos), in_seg_off=A.ptr(self.in_seg_off), in_segs=A.ptr(self.in_segs), in_key_off=A.ptr(self.in_key_off), in_keys=A.ptr(self.in_keys),
            use_key_off=A.ptr(self.use_key_off), use_keys=A.ptr(self.use_keys), in_lead_key=A.ptr(self.in_lead_key), in_trail_key=A.ptr(self.in_trail_key),
            read_len=A.ptr(self.read_len), opts=self.opts,
        )

    def set_gate(self, gate: Optional[np.ndarray]):
        """K7g's per-read gate bytes (or None): reads whose SX_GATE_REALIGN bit is clear get no alignments."""
        self.gate = None if gate is None else np.ascontiguousarray(gate, dtype=np.uint8)
        self.c.gate = A.ptr(self.gate)

    def algorithmic_bytes(self, n_alns: int, n_segs: int, n_keys: int) -> int:
        """bytes one enumeration must move: every input array once + the CSR it writes."""
        n_in_segs, n_in_keys, n_use = int(self.in_seg_off[-1]), int(self.in_key_off[-1]), int(self.use_key_off[-1])
        inp = self.n_keys * (32 + (12 if self.has_hap else 0)) + self.n_regions * 16 + self.n_reads * (4 + 4 + 4 + 4 + 2 + 2 + 2) + n_in_segs * 4 + (n_in_keys + n_use) * 2
        out = self.n_reads * (4 + 1) + n_alns * (4 + 4 + 4 + 2 + 2) + n_segs * 4 + n_keys * 2
        return inp + out


class EnumOut:
    """Host buffers for sx_enum_out."""

    def __init__(self, eb: EnumBatch, cap_alns=None, cap_segs=None, cap_keys=None):
        self.cap_alns = cap_alns if cap_alns is not None else max(64, eb.n_reads * 64)
        self.cap_segs = cap_segs if cap_segs is not None else self.cap_alns * 16
        self.cap_keys = cap_keys if cap_keys is not None else self.cap_alns * 8
        self.totals = np.zeros(4, np.uint32)
        self.aln_off = np.zeros(eb.n_reads + 1, np.uint32)
        self.status = np.zeros(eb.n_reads + 1, np.uint8)
        self.aln_pos = np.zeros(self.cap_alns + 1, np.int32)
        self.aln_seg_off = np.zeros(self.cap_alns + 2, np.uint32)
        self.segs = np.zeros(self.cap_segs + 1, dtype=A.ALN_SEG_DT)
        self.aln_key_off = np.zeros(self.cap_alns + 2, np.uint32)
        self.aln_keys = np.zeros(self.cap_keys + 1, np.uint16)
        self.aln_lead_key = np.zeros(self.cap_alns + 1, np.uint16)
        self.aln_trail_key = np.zeros(self.cap_alns + 1, np.uint16)
        self.c = A.SxEnumOut(cap_alns=self.cap_alns, cap_segs=self.cap_segs, cap_keys=self.cap_keys, totals=A.ptr(self.totals), aln_off=A.ptr(self.aln_off),
                             status=A.ptr(self.status), aln_pos=A.ptr(self.aln_pos), aln_seg_off=A.ptr(self.aln_seg_off), segs=A.ptr(self.segs),
                             aln_key_off=A.ptr(self.aln_key_off), aln_keys=A.ptr(self.aln_keys), aln_lead_key=A.ptr(self.aln_lead_key), aln_trail_key=A.ptr(self.aln_trail_key))
        self._n_reads = eb.n_reads

    def trimmed(self):
        """(aln_off, status, aln_pos, aln_seg_off, segs, aln_key_off, aln_keys, lead, trail) cut to the produced sizes."""
        nA, nS, nK = (int(x) for x in self.totals[:3])
        return (self.aln_off[: self._n_reads + 1].copy(), self.status[: self._n_reads].copy(), self.aln_pos[:nA].copy(), self.aln_seg_off[: nA + 1].copy(),
                self.segs[:nS].copy(), self.aln_key_off[: nA + 1].copy(), self.aln_keys[:nK].copy(), self.aln_lead_key[:nA].copy(), self.aln_trail_key[:nA].copy())

    def alignments_of(self, r: int):
        """read r's candidate alignments as [(pos, cigar string, [keys], lead, trail)] (debugging aid)."""
        out = []
        for a in range(int(self.aln_off[r]), int(self.aln_off[r + 1])):
            cig = "".join(f"{int(s['len'])}{AP_CHAR[int(s['kind'])]}" for s in self.segs[int(self.aln_seg_off[a]) : int(self.aln_seg_off[a + 1])])
            out.append((int(self.aln_pos[a]), cig, [int(k) for k in self.aln_keys[int(self.aln_key_off[a]) : int(self.aln_key_off[a + 1])]],
                        int(self.aln_lead_key[a]), int(self.aln_trail_key[a])))
        return out


# ------------------------------------------------------------------------------------------------------------------------------
# K7b link_alignments: K7's output -> the alignment part of K1's batch
# ------------------------------------------------------------------------------------------------------------------------------
class LinkOut:
    """Host buffers for sx_link_out.  `regions` = the region records of the K1 batch the alignments will join (a copy is taken: the
    call fills aln_begin / seg_begin / ins_begin)."""

    def __init__(self, regions: np.ndarray, n_alns: int, cap_segs: int, cap_ins: int, n_enum_segs: int = 0):
        self.cap_segs, self.cap_ins, self.n_alns = int(cap_segs), int(cap_ins), int(n_alns)
        self.totals = np.zeros(2, np.uint32)
        self.regions = regions.copy()
        self.alns = np.zeros(n_alns + 1, dtype=A.ALN_DT)
        self.segs = np.zeros(self.cap_segs + 16, dtype=A.ALN_SEG_DT)
        self.segs["kind"][:] = A.SX_SEG_HARDCLIP
        self.ins = np.zeros(self.cap_ins + A.SX_POOL_SLACK + 16, np.uint8)
        self.k6_segs = np.zeros(n_enum_segs + 16, dtype=A.ALN_SEG_DT) if n_enum_segs else None  # K7's segments with K6's kinds
        self.c = A.SxLinkOut(cap_segs=self.cap_segs, cap_ins=self.cap_ins, totals=A.ptr(self.totals), regions=A.ptr(self.regions), alns=A.ptr(self.alns),
                             segs=A.ptr(self.segs), ins=A.ptr(self.ins), k6_segs=A.ptr(self.k6_segs))

    def align_batch(self, reads_of: "AlignBatch") -> "AlignBatch":
        """the K1 batch made of `reads_of`'s read / quality / reference pools and the linked alignments."""
        used = dict(reads_of.used)
        used["ins"] = int(self.totals[1])
        assert reads_of.fmt == 0 and reads_of.qual_bits in (0, 8), "the linked alignment arrays are in the wide formats"
        return AlignBatch(self.regions, reads_of.read_len, reads_of.seq4, reads_of.qual, reads_of.ref, self.alns, self.segs, self.ins, used, qual_bits=reads_of.qual_bits,
                          n_segs=int(self.totals[0]), n_alns=self.n_alns)


def regions_from_enumeration(eb: EnumBatch, out: "EnumOut", quals_of=None) -> List[RegionSpec]:
    """The enumerated alignments as reference-shaped objects (RegionSpec / CandidateAlignmentSpec with IndelKeySpecs): what the host
    path (build_align_batch, the reference harness ref_score_region) consumes.  quals_of(read index, length) -> qualities."""
    regions = []
    for g in range(eb.n_regions):
        k0 = int(eb.region_key_off[g])
        ref = bytes(eb.ref_pool[int(eb.ref_off[g]) : int(eb.ref_off[g + 1])]).decode()
        reads, alns = [], []
        r0, r1 = int(eb.region_read_off[g]), int(eb.region_read_off[g + 1])
        for r in range(r0, r1):
            seq = bytes(eb.read_pool[int(eb.read_off[r]) : int(eb.read_off[r + 1])]).decode()
            q = quals_of(r, len(seq)) if quals_of else np.full(len(seq), 30, np.uint8)
            reads.append((codes_of(seq), np.asarray(q, np.uint8)))
            for a in range(int(out.aln_off[r]), int(out.aln_off[r + 1])):
                kidx = [int(x) for x in out.aln_keys[int(out.aln_key_off[a]) : int(out.aln_key_off[a + 1])]]
                keys = []
                for w in kidx:
                    k = eb.keys[k0 + w]
                    ins = bytes(eb.ins_pool[int(eb.ins_off[k0 + w]) : int(eb.ins_off[k0 + w + 1])]).decode()
                    keys.append(IndelKeySpec(int(k["pos"]), INDEL_MISMATCH if int(k["type"]) == A.SX_INDEL_TYPE_MISMATCH else INDEL_INDEL, int(k["del_len"]), ins,
                                             bool(int(k["flags"]) & A.SX_IKF_CANDIDATE)))
                lead, trail = int(out.aln_lead_key[a]), int(out.aln_trail_key[a])
                path = [(AP_CHAR[int(s["kind"])], int(s["len"])) for s in out.segs[int(out.aln_seg_off[a]) : int(out.aln_seg_off[a + 1])]]
                alns.append(CandidateAlignmentSpec(r - r0, int(out.aln_pos[a]), path, keys, kidx.index(lead) if lead != A.SX_NO_KEY else -1,
                                                   kidx.index(trail) if trail != A.SX_NO_KEY else -1))
        regions.append(RegionSpec(ref, int(eb.ref_begin[g]), reads, alns))
    return regions


class PrepOut:
    """Host buffers for sx_prep_out (K7a)."""

    def __init__(self, eb: EnumBatch, cap_keys=None):
        self.cap_keys = cap_keys if cap_keys is not None else 8 * eb.n_reads + 64
        self.totals = np.zeros(2, np.uint32)
        self.in_key_off = np.zeros(eb.n_reads + 1, np.uint32)
        self.in_keys = np.zeros(self.cap_keys + 1, np.uint16)
        self.in_lead_key = np.zeros(eb.n_reads + 1, np.uint16)
        self.in_trail_key = np.zeros(eb.n_reads + 1, np.uint16)
        self.c = A.SxPrepOut(cap_keys=self.cap_keys, totals=A.ptr(self.totals), in_key_off=A.ptr(self.in_key_off), in_keys=A.ptr(self.in_keys),
                             in_lead_key=A.ptr(self.in_lead_key), in_trail_key=A.ptr(self.in_trail_key))
        self._n = eb.n_reads

    def trimmed(self):
        return self.in_key_off[: self._n + 1].copy(), self.in_keys[: int(self.totals[0])].copy(), self.in_lead_key[: self._n].copy(), self.in_trail_key[: self._n].copy()


def read_pools_of(eb: EnumBatch) -> AlignBatch:
    """The reads and reference windows of an EnumBatch where K1 keeps them (an AlignBatch without alignments): K7a's other input."""
    regions = []
    for g in range(eb.n_regions):
        ref = bytes(eb.ref_pool[int(eb.ref_off[g]) : int(eb.ref_off[g + 1])]).decode()
        reads = []
        for r in range(int(eb.region_read_off[g]), int(eb.region_read_off[g + 1])):
            seq = bytes(eb.read_pool[int(eb.read_off[r]) : int(eb.read_off[r + 1])]).decode()
            reads.append((codes_of(seq), np.full(len(seq), 30, np.uint8)))
        regions.append(RegionSpec(ref, int(eb.ref_begin[g]), reads, []))
    return build_align_batch(regions)


# ------------------------------------------------------------------------------------------------------------------------------
# K9 choose_realignment
# ------------------------------------------------------------------------------------------------------------------------------
class RealignBatch:
    """sx_realign_batch over K7's output (host arrays): the candidate alignments of EnumBatch `eb` as enumerated into `out`."""

    def __init__(self, eb: EnumBatch, out: "EnumOut", is_smoothed=True, smoothed_lnp_range=2.302585092994046, k4_kinds=False, pin_flags=None, raw: "GateBatch" = None):
        self.eb, self.enum_out = eb, out
        self.n_alns = int(out.totals[0])
        self.pin_flags = pin_flags
        self.raw = raw  # the mapper's alignments: with them the output is getBestAlignment() of every read
        self.c = A.SxRealignBatch(n_regions=eb.n_regions, n_reads=eb.n_reads, n_alns=self.n_alns, region_read_off=A.ptr(eb.region_read_off),
                                  region_key_off=A.ptr(eb.region_key_off), keys=A.ptr(eb.keys), aln_off=A.ptr(out.aln_off), aln_pos=A.ptr(out.aln_pos),
                                  aln_seg_off=A.ptr(out.aln_seg_off), segs=A.ptr(out.segs), aln_key_off=A.ptr(out.aln_key_off), aln_keys=A.ptr(out.aln_keys),
                                  read_len=A.ptr(eb.read_len), pin_flags=A.ptr(pin_flags), is_smoothed_alignments=1 if is_smoothed else 0, k4_kinds=1 if k4_kinds else 0,
                                  smoothed_lnp_range=smoothed_lnp_range)
        if raw is not None:
            self.c.raw_pos, self.c.raw_seg_off, self.c.raw_segs = A.ptr(raw.raw_pos), A.ptr(raw.seg_off), A.ptr(raw.raw_segs)


class RealignOut:
    """Host buffers for sx_realign_out."""

    def __init__(self, rb: RealignBatch, cap_segs=None):
        n = rb.eb.n_reads
        n_raw = int(rb.raw.seg_off[n]) if getattr(rb, "raw", None) is not None else 0
        self.cap_segs = cap_segs if cap_segs is not None else int(rb.enum_out.totals[1]) + 2 * n + n_raw + 64
        self.totals = np.zeros(2, np.uint32)
        self.seg_off = np.zeros(n + 1, np.uint32)
        self.pos = np.zeros(n + 1, np.int32)
        self.n_seg = np.zeros(n + 1, np.uint16)
        self.status = np.zeros(n + 1, np.uint8)
        self.best_aln = np.zeros(n + 1, np.uint32)
        self.segs = np.zeros(self.cap_segs + 1, dtype=A.ALN_SEG_DT)
        self.c = A.SxRealignOut(cap_segs=self.cap_segs, totals=A.ptr(self.totals), seg_off=A.ptr(self.seg_off), pos=A.ptr(self.pos), n_seg=A.ptr(self.n_seg),
                                status=A.ptr(self.status), best_aln=A.ptr(self.best_aln), segs=A.ptr(self.segs))
        self._n = n

    def realignment_of(self, r: int):
        """(pos, cigar string) of read r, or None when it was not realigned."""
        if not (int(self.status[r]) & A.SX_REALIGN_ST_REALIGNED):
            return None
        s0 = int(self.seg_off[r])
        return int(self.pos[r]), "".join(f"{int(s['len'])}{AP_CHAR[int(s['kind'])]}" for s in self.segs[s0 : s0 + int(self.n_seg[r])])


# ------------------------------------------------------------------------------------------------------------------------------
# K7g realign_gates
# ------------------------------------------------------------------------------------------------------------------------------
class GateBatch:
    """sx_gate_batch: the mapper's alignments of an EnumBatch's reads (raw = [(pos, [(cigar char, len)...])] per read, batch order) with the
    batch's window and realignment ranges."""

    def __init__(self, eb: EnumBatch, raw, max_indel_size=49, pin_flags=None):
        assert len(raw) == eb.n_reads
        self.eb = eb
        segs, seg_off, pos = [], [0], []
        for p, path in raw:
            pos.append(p)
            segs.extend((ln, _AP_OF[t], 0) for t, ln in path)
            seg_off.append(len(segs))
        self.raw_pos = np.array(pos + [0], np.int32)
        self.seg_off = np.array(seg_off, np.uint32)
        self.raw_segs = np.zeros(len(segs) + 4, dtype=A.ALN_SEG_DT)
        if segs:
            self.raw_segs[: len(segs)] = np.array(segs, dtype=A.ALN_SEG_DT)
        self.n_segs = len(segs)
        self.pin_flags = pin_flags
        self.c = A.SxGateBatch(n_regions=eb.n_regions, n_reads=eb.n_reads, region_read_off=A.ptr(eb.region_read_off), region_key_off=A.ptr(eb.region_key_off),
                               keys=A.ptr(eb.keys), realign_begin=A.ptr(eb.realign_begin), realign_end=A.ptr(eb.realign_end), raw_pos=A.ptr(self.raw_pos),
                               seg_off=A.ptr(self.seg_off), raw_segs=A.ptr(self.raw_segs), read_len=A.ptr(eb.read_len), pin_flags=A.ptr(pin_flags), max_indel_size=max_indel_size)


class GateOut:
    def __init__(self, gb: GateBatch):
        n = gb.eb.n_reads
        self.gate = np.zeros(n + 1, np.uint8)
        self.in_pos = np.zeros(n + 1, np.int32)
        self.in_segs = np.zeros(gb.n_segs + 4, dtype=A.ALN_SEG_DT)
        self.c = A.SxGateOut(gate=A.ptr(self.gate), in_pos=A.ptr(self.in_pos), in_segs=A.ptr(self.in_segs))
        self._gb = gb

    def alignment_of(self, r: int):
        """(pos, cigar) of the normalized alignment (pads dropped), or None when the read does not go into the search."""
        if not (int(self.gate[r]) & A.SX_GATE_REALIGN):
            return None
        s0, s1 = int(self._gb.seg_off[r]), int(self._gb.seg_off[r + 1])
        return int(self.in_pos[r]), "".join(f"{int(s['len'])}{AP_CHAR[int(s['kind'])]}" for s in self.in_segs[s0:s1] if not (int(s["kind"]) == A.SX_AP_HARD_CLIP and int(s["len"]) == 0))


# ------------------------------------------------------------------------------------------------------------------------------
# process_window (sx_process_window_dev): one description of a window of reads for the whole device-resident pass
# ------------------------------------------------------------------------------------------------------------------------------
class WindowBatch:
    """Host arrays of an sx_window_batch.  `a` maps the struct's array fields to numpy arrays; scalars are attributes.  Two ways in:
    from_enum (a test batch: EnumBatch + the mapper's alignments + its K1 pools, one contig segment) and from_arrays (a generator's output)."""

    ARRAYS = ("region_read_off", "region_key_off", "keys", "key_hap", "key_ins_off", "key_ins", "realign_begin", "realign_end", "raw_pos", "raw_seg_off", "raw_segs",
              "read_len", "read_flags", "mapq", "use_key_off", "use_keys", "rec_off", "regions", "seq4", "qual", "ref", "cand_snv")

    def __init__(self, a: dict, n_regions: int, n_reads: int, n_keys: int, ref_begin: int, report_begin: int, report_end: int, qual_bits: int = 8, qual_dict=None,
                 max_read_len: int = 0, do_site_gl: bool = True, used=None):
        self.a = a
        self.n_regions, self.n_reads, self.n_keys = n_regions, n_reads, n_keys
        self.ref_begin, self.report_begin, self.report_end = ref_begin, report_begin, report_end
        self.qual_bits, self.qual_dict = qual_bits, list(qual_dict or [])
        self.max_read_len, self.do_site_gl = max_read_len, do_site_gl
        self.used = used or {"seq4": int(a["seq4"].nbytes), "qual": int(a["qual"].nbytes), "ref": int(a["ref"].nbytes)}
        self.n_sites = report_end - report_begin

    @classmethod
    def from_enum(cls, eb: "EnumBatch", gb: "GateBatch", pools: AlignBatch, read_flags=None, mapq=None, report=None, do_site_gl=True):
        """eb's regions must lie on one contig segment in ascending order with reads in read-buffer order (a single region always does)."""
        assert pools.fmt == 0 and pools.qual_bits in (0, 4, 8) and pools.n_reads == eb.n_reads and gb.eb is eb
        n = eb.n_reads
        reg = pools.regions.copy()
        ref0, rb0 = int(reg["ref_off"][0]), int(reg["ref_begin"][0])
        # the pools' reference windows as views of ONE array: window g must start (ref_begin[g] - ref_begin[0]) bytes after window 0
        for g in range(eb.n_regions):
            assert int(reg["ref_off"][g]) - ref0 == int(reg["ref_begin"][g]) - rb0, "the regions' reference windows are not views of one contig segment"
        reg["ref_off"] -= ref0
        ref = pools.ref[ref0:]
        n_win = np.diff(eb.region_key_off.astype(np.int64))
        rec_off = np.concatenate([[0], np.cumsum(np.repeat(n_win, np.diff(eb.region_read_off.astype(np.int64))))]).astype(np.uint32)
        flags = np.full(n + 1, A.SX_PRF_FWD | A.SX_PRF_TIER1 | A.SX_PRF_TIER1OR2, np.uint8) if read_flags is None else np.ascontiguousarray(read_flags, np.uint8)
        mq = np.full(n + 1, 60, np.uint8) if mapq is None else np.ascontiguousarray(mapq, np.uint8)
        a = {"region_read_off": eb.region_read_off, "region_key_off": eb.region_key_off, "keys": eb.keys, "key_hap": eb.key_hap if eb.has_hap else None,
             "key_ins_off": eb.ins_off, "key_ins": eb.ins_pool, "realign_begin": eb.realign_begin, "realign_end": eb.realign_end, "raw_pos": gb.raw_pos,
             "raw_seg_off": gb.seg_off, "raw_segs": gb.raw_segs, "read_len": eb.read_len, "read_flags": flags, "mapq": mq, "use_key_off": eb.use_key_off,
             "use_keys": eb.use_keys, "rec_off": rec_off, "regions": reg, "seq4": pools.seq4, "qual": pools.qual, "ref": ref, "cand_snv": None}
        if report is None:
            last = eb.n_regions - 1
            report = (rb0, int(reg["ref_begin"][last]) + int(reg["ref_len"][last]))
        w = cls(a, eb.n_regions, n, eb.n_keys, rb0, report[0], report[1], 4 if pools.qual_bits == 4 else 8, pools.qual_dict, int(eb.read_len[:n].max(initial=1)), do_site_gl,
                {"seq4": pools.used["seq4"], "qual": pools.used["qual"], "ref": int(reg["ref_off"][eb.n_regions - 1]) + int(reg["ref_len"][eb.n_regions - 1])})
        w.enum_opts = eb.opts
        return w


# ---- somatic callable regions (sx_somatic_callable_regions_dev's host builder)
def somatic_callable_regions(site_snv: np.ndarray, pos_begin: int):
    """SomaticCallableProcessor + RegionProcessor on sx_ssnv_result records of consecutive positions pos_begin, pos_begin + 1, ...: a
    position is callable unless both qphred < 15 and nonsomatic_qphred < 15; returns the half-open intervals of consecutive callable
    positions as (begin, end) int32 arrays"""
    c = ~((site_snv["qphred"] < 15) & (site_snv["nonsomatic_qphred"] < 15))
    d = np.diff(np.concatenate([[0], c.astype(np.int8), [0]]))
    return (np.nonzero(d == 1)[0] + pos_begin).astype(np.int32), (np.nonzero(d == -1)[0] + pos_begin).astype(np.int32)


# ---------------------------------------------------------------------------------------------------------------------------
# K4m pileup_metrics
# ---------------------------------------------------------------------------------------------------------------------------
def _mapped_qscore_table() -> np.ndarray:
    """qphred_cache::mappedq[mapq 0..90][basecall q 0..70] (blt_util/qscore_cache.cpp:44-47)"""
    t = np.zeros((91, 71), np.uint8)
    for j in range(91):
        me = math.pow(10.0, -float(j) / 10.0)
        for i in range(71):
            be = math.pow(10.0, -float(i) / 10.0)
            p = ((1.0 - me) * be) + (me * 0.75)
            t[j, i] = int(math.floor(-10.0 * max(-307.0, math.log10(p)) + 0.5))
    return t


def _z_stat(vals: np.ndarray, is_ref: np.ndarray):
    """fastRanksum::get_z_stat of (is_ref, value) observations in closed form: (z, overflow, N2, sum of the category-2 values)"""
    n1, n2 = int(is_ref.sum()), int((~is_ref).sum())
    if n1 + n2 == 0:
        return 0.0, False, 0, 0
    uniq, inv, cnt = np.unique(vals.astype(np.int64), return_inverse=True, return_counts=True)
    before = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    wx2 = 2 * before[inv] + cnt[inv] + 1  # twice the mean rank of each observation's value
    R1, R2 = int(wx2[is_ref].sum()) * 0.5, int(wx2[~is_ref].sum()) * 0.5
    a, b, w1 = (n2, n1, R2) if R1 > R2 else (n1, n2, R1)
    prod = a * (a + b + 1)
    if prod > 2147483647:
        return 0.0, True, n2, int(vals[~is_ref].astype(np.int64).sum())
    mean = float(prod) / 2.0
    var = math.sqrt(float(b) * mean / 6.0)
    z = 0.0 if abs(var) < 0.0001 else (w1 - mean) / var
    return z, False, n2, int(vals[~is_ref].astype(np.int64).sum())


def pileup_metrics(pb: PileupReadsBatch, mode: int, full_len=None, full_off=None, observations: Optional[list] = None) -> np.ndarray:
    """The host restatement of K4m (sx_pileup_metrics) in numpy: every visited base's observation, then each position's statistics in closed
    form.  full_len / full_off: rseg.full_read_size() / full_read_offset() of every read (None: its own length / 0).  observations: a list
    that receives, per position, the (mapq, qscore, is_ref, submapped, somatic, edge, cycle, read_pos, read_size) tuples of its bases."""
    assert mode in (A.SX_PM_MAPQ, A.SX_PM_GERMLINE, A.SX_PM_SOMATIC)
    o = pb.opts
    rb, re = int(pb.c.report_begin), int(pb.c.report_end)
    ref_begin, ref = int(pb.c.ref_begin), bytes(pb.ref[: int(pb.c.ref_len)])
    ref_at = lambda pos: chr(ref[pos - ref_begin]) if 0 <= pos - ref_begin < len(ref) else "N"
    mq = _mapped_qscore_table()
    cand = set(int(k) for k in pb.cand_snv[: int(pb.c.n_cand_snv)])
    qual_bits = int(pb.c.qual_bits)
    qdict = list(pb.c.qual_dict)
    chars = "=AC" + "N" + "G" + "NNN" + "T" + "N" * 7
    ids = [4, 0, 1, 5, 2, 5, 5, 5, 3, 5, 5, 5, 5, 5, 5, 4]
    obs = [[] for _ in range(re - rb)]  # per site: (mapq, qscore, is_ref, submapped, somatic, edge, cycle, read_pos, read_size)
    reads, segs = pb.reads, pb.segs
    for r in range(pb.n_reads):
        rd = reads[r]
        flags, n, pos0, mapq = int(rd["flags"]), int(rd["len"]), int(rd["pos"]), int(rd["mapq"])
        if flags & A.SX_PRF_SKIP:
            continue
        path = [(int(s["kind"]), int(s["len"])) for s in segs[int(rd["seg_off"]): int(reads[r + 1]["seg_off"])]]
        so = int(rd["seq_off"])
        code = lambda i: (int(pb.seq4[so + (i >> 1)]) >> (4 if i % 2 == 0 else 0)) & 15
        qo = int(rd["qual_off"])
        qual = (lambda i: qdict[(int(pb.qual[qo + (i >> 1)]) >> (4 if i % 2 == 0 else 0)) & 15]) if qual_bits == 4 else (lambda i: int(pb.qual[qo + i]))
        span = sum(ln for k, ln in path if k in (A.SX_SEG_MATCH, A.SX_SEG_DELETE, A.SX_SEG_SKIP))
        if pos0 >= re or pos0 + span <= rb:
            continue
        fwd = bool(flags & A.SX_PRF_FWD)
        amb = 0
        if fwd:
            while amb < n and code(n - 1 - amb) == 15:
                amb += 1
        else:
            while amb < n and code(amb) == 15:
                amb += 1
        b, e = (0, n - amb) if fwd else (amb, n)
        if o.minDistanceFromReadEdge > 0:
            b += o.minDistanceFromReadEdge
            e = e - o.minDistanceFromReadEdge if o.minDistanceFromReadEdge <= e else 0
            if e <= b:
                continue
        submapped, tier1 = not (flags & A.SX_PRF_TIER1OR2), bool(flags & A.SX_PRF_TIER1)
        amq = max(5, mapq)
        adjust = o.isBasecallQualAdjustedForMapq and amq <= 80
        fo = 0 if full_off is None else int(full_off[r])
        fl = n if full_len is None else int(full_len[r])
        matches = [i for i, (k, _) in enumerate(path) if k == A.SX_SEG_MATCH]
        first, last = (matches[0], matches[-1]) if matches else (len(path), len(path))
        filt = None
        if mode == A.SX_PM_SOMATIC and tier1 and not submapped and o.mismatchDensityFilterFlankSize > 0:
            fs = o.mismatchDensityFilterFlankSize
            ds = max(1 + 2 * fs, n) - 2 * fs
            delta = np.zeros(ds + 1, np.int64)

            def inc(start, length):
                delta[max(2 * fs, start) - 2 * fs] += 1
                if start + length < ds:
                    delta[start + length] -= 1

            rp, fp = 0, pos0
            for i, (k, ln) in enumerate(path):
                edge = i < first or i > last
                if k == A.SX_SEG_INSERT and not edge:
                    inc(rp, ln)
                elif k == A.SX_SEG_DELETE and not edge:
                    inc(rp, 0)
                elif k == A.SX_SEG_MATCH:
                    for p in range(max(rp, b), min(rp + ln, e)):
                        c = code(p)
                        if chars[c] == ref_at(fp + p - rp):
                            continue
                        rel = fp + p - rp - rb
                        if ids[c] < 4 and 0 <= rel < (1 << 30) and ((rel << 2) | ids[c]) in cand:
                            continue
                        inc(p, 1)
                if k in (A.SX_SEG_MATCH, A.SX_SEG_INSERT, A.SX_SEG_SOFTCLIP):
                    rp += ln
                if k in (A.SX_SEG_MATCH, A.SX_SEG_DELETE, A.SX_SEG_SKIP):
                    fp += ln
            tot = np.cumsum(delta[:ds])
            filt = lambda p: int(o.mismatchDensityFilterMaxMismatchCount) < int(tot[min(ds - 1, max(fs, p) - fs)])
        rp, fp = 0, pos0
        for k, ln in path:
            if k == A.SX_SEG_MATCH:
                for p in range(max(rp, b), min(rp + ln, e)):
                    pos = fp + p - rp
                    if pos < rb or pos >= re:
                        continue
                    c = code(p)
                    cid = ids[c]
                    if cid > 4:
                        raise ValueError("unknown base code")
                    q = qual(p)
                    if adjust:
                        if q > 70:
                            raise ValueError("qscore above 70")
                        q = int(mq[min(amq, 90), q])
                    is_ref = ref_at(pos) == "ACGTN"[cid]
                    som = False
                    if mode == A.SX_PM_SOMATIC and tier1 and not submapped:
                        f = c == 15 or q < o.minBasecallErrorPhredProb
                        if not f and filt is not None:
                            f = filt(p)
                        som = not f
                    fpos = p + fo
                    d = min(fpos, (fl - (fpos + 1)) & 0xFFFFFFFF)
                    obs[pos - rb].append((mapq, q, is_ref, submapped, som, min(20, d), p if fwd else n - (p + 1), p, n))
            if k in (A.SX_SEG_MATCH, A.SX_SEG_INSERT, A.SX_SEG_SOFTCLIP):
                rp += ln
            if k in (A.SX_SEG_MATCH, A.SX_SEG_DELETE, A.SX_SEG_SKIP):
                fp += ln
    if observations is not None:
        observations.extend(obs)
    out = np.zeros(re - rb, A.PILEUP_METRICS_DT)
    for s, ob in enumerate(obs):
        rec = out[s]
        if not ob:
            continue
        a = np.array(ob, dtype=np.int64)
        mapq, q, isr, sub, som, edge, cyc, rpos, rsize = (a[:, i] for i in range(9))
        isr, sub, som = isr.astype(bool), sub.astype(bool), som.astype(bool)
        rec["mapq_count"], rec["mapq_zero"], rec["mapq_sum_sq"] = len(ob), int((mapq == 0).sum()), float(int((mapq * mapq).sum()))
        st = 0
        if mode == A.SX_PM_GERMLINE:
            z, ov, _, _ = _z_stat(mapq, isr)
            rec["mq_ranksum"], st = z, st | (A.SX_PM_ST_MQ_OVERFLOW if ov else 0)
            m = ~sub
            z, ov, n2, s2 = _z_stat(q[m], isr[m])
            rec["baseq_ranksum"], rec["raw_baseq"], st = z, (s2 / float(n2) if n2 else 0.0), st | (A.SX_PM_ST_BASEQ_OVERFLOW if ov else 0)
            z, ov, n2, s2 = _z_stat(cyc[m], isr[m])
            rec["read_pos_ranksum"], rec["raw_pos"], st = z, (s2 / float(n2) if n2 else 0.0), st | (A.SX_PM_ST_READ_POS_OVERFLOW if ov else 0)
            alt = m & ~isr
            rec["mean_edge_distance"] = int(edge[alt].sum()) / float(int(alt.sum())) if alt.any() else 0.0
        elif mode == A.SX_PM_SOMATIC:
            z, ov, _, _ = _z_stat(rpos[som], isr[som])
            rec["read_pos_ranksum"], st = z, st | (A.SX_PM_ST_READ_POS_OVERFLOW if ov else 0)
            alt = som & ~isr
            na = int(alt.sum())
            rec["n_alt_read_pos"] = na
            if na:
                p = np.sort(rpos[alt])
                pm, lm = int(p[na // 2]), int(np.sort(rsize[alt] - rpos[alt])[na // 2])
                rec["median_read_pos"] = min(pm, lm)
                if na >= 3:
                    rec["median_read_pos_var"] = int(np.sort(np.abs(p - pm))[na // 2])
        rec["status"] = st
    return out
