"""Read batches for K4m (pileup metrics): seeded random pile-ups under several option sets, and the edge batches -- a site deeper than the
reduce kernel's shared-memory tile, a site whose rank-sum product overflows the reference's int, 'N' reference positions and calls, alt
lists of every small size, MAPQ 0 and 255, clipped and trimmed reads across both report edges."""
from __future__ import annotations

import numpy as np

import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

MODES = (A.SX_PM_MAPQ, A.SX_PM_GERMLINE, A.SX_PM_SOMATIC)


def opts(density=True, tier2=False, adjust=True, min_edge=0):
    o = A.default_pileup_opts()
    o.mismatchDensityFilterFlankSize = 20 if density else 0
    o.useTier2Evidence = int(tier2)
    o.isBasecallQualAdjustedForMapq = int(adjust)
    o.minDistanceFromReadEdge = min_edge
    return o


OPTION_SETS = {"default": opts(), "no_density": opts(density=False), "tier2": opts(tier2=True), "no_adjust": opts(adjust=False), "min_edge": opts(min_edge=3)}


def random_batch(seed: int, o=None, n_reads=300, ref_len=1500, qual_dict=False):
    rng = np.random.default_rng(seed)
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=n_reads, ref_len=ref_len)
    for r in reads:  # MAPQ 0 and 255 as well as the generator's range
        x = rng.random()
        r.mapq = 0 if x < 0.05 else 255 if x < 0.08 else r.mapq
        if qual_dict:
            r.quals = [min(q, 40) // 10 * 10 + 2 for q in r.quals]
    qd = [2, 12, 22, 32, 42] if qual_dict else None
    return B.PileupReadsBatch(reads, ref, ref_begin, ref_begin + 50, ref_begin + len(ref) - 50, cand, opts=o, qual_dict=qd)


def full_read_arrays(pb: B.PileupReadsBatch, seed: int):
    """full_read_size / full_read_offset of a read taken as a segment of a longer read (RNA segments)"""
    rng = np.random.default_rng(seed)
    n = pb.n_reads
    off = rng.integers(0, 30, size=n).astype(np.uint16) * (rng.random(n) < 0.3)
    full = (pb.reads["len"][:n].astype(np.int64) + off + rng.integers(0, 30, size=n) * (rng.random(n) < 0.3)).astype(np.uint16)
    return full, off.astype(np.uint16)


def edge_batch():
    """hand-made reads over 'N' reference positions, alt lists of sizes 0..6, both strands, trimmed and clipped ends, filtered calls"""
    ref = "ACGTACGTNNACGTACGTACGTACGTACGTACGTACGTACGT" * 3
    reads = []
    C = {"A": 1, "C": 2, "G": 4, "T": 8, "N": 15}
    for k in range(7):  # k alt reads at site 20 + 9 k, and as many reference reads
        site = 20 + 9 * k
        for j in range(2 * k):
            seq = list(ref[site - 4 - j: site + 20 - j])
            if j < k:
                seq[4 + j] = "A" if ref[site] != "A" else "C"
            reads.append(B.PileupReadSpec([C[b] for b in seq], [30 + j] * len(seq), site - 4 - j, [("M", len(seq))], fwd=j % 2 == 0))
    for j in range(3):  # 'N' calls at 'N' reference positions, a low quality, an N run at each end
        seq = list(ref[4 + j: 28 + j])
        seq[0] = "N"
        seq[-1] = "N"
        reads.append(B.PileupReadSpec([C[b] for b in seq], [5 if i == 10 else 35 for i in range(len(seq))], 4 + j,
                                      [("H", 3), ("S", 2), ("M", len(seq) - 4), ("S", 2)], fwd=j != 1, mapq=[0, 255, 17][j], tier=[1, 2, 0][j]))
    reads.sort(key=lambda r: r.pos)
    return B.PileupReadsBatch(reads, ref, 0, 6, len(ref) - 10, [], opts=opts())


def deep_batch(depth: int, seed: int = 7, alt_frac: float = 0.3):
    """`depth` short reads over one site (past the reduce kernel's 512-word tile), mixed categories and mapping qualities"""
    rng = np.random.default_rng(seed)
    ref = "ACGT" * 20
    reads = []
    C = {"A": 1, "C": 2, "G": 4, "T": 8}
    for i in range(depth):
        start = int(rng.integers(30, 41))
        seq = list(ref[start: start + 20])
        if rng.random() < alt_frac:
            seq[40 - start] = "A" if ref[40] != "A" else "G"
        reads.append(B.PileupReadSpec([C[b] for b in seq], [int(rng.integers(15, 41)) for _ in seq], start, [("M", 20)], fwd=bool(rng.random() < 0.5),
                                      mapq=int(rng.choice([0, 20, 40, 60, 255])), tier=1 if rng.random() < 0.9 else int(rng.choice([0, 2]))))
    reads.sort(key=lambda r: r.pos)
    return B.PileupReadsBatch(reads, ref, 0, 10, 70, [], opts=opts())


def overflow_batch(depth: int = 66000):
    """one-base reads at one site, half reference and half alternate with the same MAPQ: mq_ranksum's n1 (n1 + n2 + 1) passes 2^31 - 1"""
    reads = [B.PileupReadSpec([1 if i % 2 == 0 else 2], [30], 5, [("M", 1)], mapq=60) for i in range(depth)]
    return B.PileupReadsBatch(reads, "CCCCCACCCC", 0, 0, 10, [], opts=opts())


# ---------------------------------------------------------------------------------------------------------------------------------------
# the reference's own answers: oracle/ref_harness_pileup_metrics.cpp (oracle/_ref, where build() could compile it), else the frozen ones
# ---------------------------------------------------------------------------------------------------------------------------------------
import ctypes as _C  # noqa: E402
import os as _os  # noqa: E402

_ROOT = _os.path.dirname(_os.path.dirname(_os.path.abspath(__file__)))
REF_SO = _os.path.join(_ROOT, "oracle", "_ref", "libstrelka_ref_pileup_metrics.so")
GOLDEN = _os.path.join(_ROOT, "tests", "golden", "pileup_metrics_ref.npz")
_ref = None


def have_ref() -> bool:
    return _os.path.exists(REF_SO)


def ref_metrics(pb: B.PileupReadsBatch, mode: int) -> np.ndarray:
    """the reference's pileup_read_segment with the metrics on, read back through its own accessors"""
    global _ref
    if _ref is None:
        _ref = _C.CDLL(REF_SO)
        _ref.ref_pileup_metrics.argtypes = [_C.POINTER(A.SxPileupReadsBatch), _C.c_uint32, _C.c_void_p, _C.c_char_p, _C.c_int]
    out = np.zeros(pb.n_sites, A.PILEUP_METRICS_DT)
    err = _C.create_string_buffer(512)
    if _ref.ref_pileup_metrics(_C.byref(pb.c), mode, out.ctypes.data, err, 512) != 0:
        raise RuntimeError(err.value.decode(errors="replace"))
    return out


def golden_cases():
    """(key, batch, mode) of every frozen case: the seeded batches under each option set, the edge batch and a deep site (the overflow site is
    left out: the reference's value there is undefined)"""
    for name in sorted(OPTION_SETS):
        for seed in (1, 2):
            pb = random_batch(seed, OPTION_SETS[name], qual_dict=seed == 2)
            for mode in MODES:
                yield f"{name}_{seed}_{mode}", pb, mode
    for mode in MODES:
        yield f"edge_{mode}", edge_batch(), mode
        yield f"deep_{mode}", deep_batch(1200), mode


def golden():
    return np.load(GOLDEN)


# ---------------------------------------------------------------------------------------------------------------------------------------
# the window passes' own pile-up batch, rebuilt on the host
# ---------------------------------------------------------------------------------------------------------------------------------------
def window_pileup_batch(w: B.WindowBatch, d: dict, max_indel_size: int):
    """the sx_pileup_reads_batch sx_process_window_dev builds for K4 (sx_pipeline.cu, sxp_pileup_reads_kernel) from a DevWindow download `d`:
    the best alignments, the read pools, the reference and cand_snv, with SX_PRF_SKIP on a read that was not realigned and whose only alignment
    has an indel over max_indel_size.  (The metrics are order-free: the buffer order is not needed.)"""
    import types

    import somatic_window_leg as SW

    n = w.n_reads
    seq_off, qual_off, packed, per_q = SW.read_offsets(w)
    reads = np.zeros(n + 1, A.PILEUP_READ_DT)
    flags = w.a["read_flags"][:n] & (A.SX_PRF_FWD | A.SX_PRF_TIER1 | A.SX_PRF_TIER1OR2 | A.SX_PRF_PIN_FIRST | A.SX_PRF_PIN_SECOND)
    raw_off, raw = w.a["raw_seg_off"], w.a["raw_segs"]
    for r in range(n):
        if not (int(d["realign_status"][r]) & A.SX_REALIGN_ST_REALIGNED):
            inner = raw[int(raw_off[r]) + 1: max(int(raw_off[r]) + 1, int(raw_off[r + 1]) - 1)]
            if any(int(s["kind"]) in (A.SX_AP_INSERT, A.SX_AP_DELETE) and int(s["len"]) > max_indel_size for s in inner):
                flags[r] |= A.SX_PRF_SKIP
    reads["seq_off"][:n], reads["qual_off"][:n] = seq_off, qual_off
    reads["seq_off"][n] = int(seq_off[-1] + packed[-1]) if n else 0
    reads["qual_off"][n] = int(qual_off[-1] + per_q[-1]) if n else 0
    reads["seg_off"] = d["best_seg_off"][: n + 1]
    reads["pos"][:n], reads["len"][:n], reads["mapq"][:n], reads["flags"][:n] = d["best_pos"], w.a["read_len"][:n], w.a["mapq"][:n], flags
    pb = types.SimpleNamespace(n_reads=n, n_sites=w.n_sites, reads=reads, segs=np.concatenate([d["best_segs"], np.zeros(16, A.ALN_SEG_DT)]),
                               seq4=w.a["seq4"], qual=w.a["qual"], ref=w.a["ref"], opts=A.default_pileup_opts())
    cand = w.a.get("cand_snv")
    pb.cand_snv = cand if cand is not None else np.zeros(1, np.uint32)
    span = 1
    pb.c = A.SxPileupReadsBatch(n_reads=n, n_segs=int(d["best_seg_off"][n]), reads=A.ptr(reads), seq4=A.ptr(pb.seq4), qual=A.ptr(pb.qual), segs=A.ptr(pb.segs),
                                ref=A.ptr(pb.ref), ref_begin=w.ref_begin, ref_len=int(w.used["ref"]), report_begin=w.report_begin, report_end=w.report_end,
                                cand_snv=A.ptr(pb.cand_snv), n_cand_snv=int(cand.size) if cand is not None else 0, max_ref_span=span,
                                max_read_len=int(w.max_read_len), opts=pb.opts, qual_bits=4 if w.qual_bits == 4 else 8)
    pb.c.qual_dict = (_C.c_uint8 * 16)(*(list(w.qual_dict) + [0] * (16 - len(w.qual_dict))))
    return pb
