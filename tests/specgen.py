"""Seeded generators of reference-shaped test inputs (candidate alignments, pileups, haplotype/reference pairs)."""
from __future__ import annotations

from typing import List, Tuple

import numpy as np

from strelka_b200 import _abi as A
from strelka_b200 import batch as B

BASES = "ACGT"
CODE_OF = {"A": 1, "C": 2, "G": 4, "T": 8, "N": 15, "=": 0}
QUALS = np.array([0, 2, 3, 11, 17, 25, 30, 37, 40, 41, 60, 70], dtype=np.uint8)
QUAL_P = np.array([0.01, 0.02, 0.02, 0.05, 0.05, 0.1, 0.1, 0.45, 0.1, 0.05, 0.03, 0.02])


def rand_seq(rng: np.random.Generator, n: int, n_frac: float = 0.0) -> str:
    s = rng.integers(0, 4, n)
    out = np.array(list(BASES))[s]
    if n_frac > 0:
        out[rng.random(n) < n_frac] = "N"
    return "".join(out)


def random_region(rng: np.random.Generator, n_reads: int = 6, alns_per_read: Tuple[int, int] = (1, 4), read_len: Tuple[int, int] = (30, 150),
                  ref_len: int = 400, ref_begin: int = 1000, weird: bool = True) -> B.RegionSpec:
    """One region with randomly shaped candidate alignments: plain matches, internal insertions / deletions / swaps /
    SEQ_MISMATCH blocks, leading- and trailing-edge insertions with longer key sequences, soft/hard clips, skips, N and '='
    read codes, alignments hanging off either end of the held reference, candidate and non-candidate indels."""
    ref = rand_seq(rng, ref_len, 0.01 if weird else 0.0)
    reads = []
    alns: List[B.CandidateAlignmentSpec] = []
    # candidacy must be a function of the indel key within a region (one IndelBuffer)
    cand_of = {}

    def candidacy(pos, typ, dl, ins):
        k = (pos, typ, dl, ins)
        if k not in cand_of:
            cand_of[k] = bool(rng.random() < 0.7)
        return cand_of[k]

    for r in range(n_reads):
        L = int(rng.integers(read_len[0], read_len[1] + 1))
        na = int(rng.integers(alns_per_read[0], alns_per_read[1] + 1))
        read_bases: List[str] = ["A"] * L
        first = True
        for _ in range(na):
            # build a path consuming exactly L read bases
            remaining = L
            path: List[Tuple[str, int]] = []
            indels: List[B.IndelKeySpec] = []
            leading = trailing = -1
            pos = int(rng.integers(ref_begin - 20, ref_begin + ref_len - L // 2))
            ref_head = pos
            expected: List[str] = []  # the base each read position is compared against ('?' = none)

            def ref_at(p):
                q = p - ref_begin
                return ref[q] if 0 <= q < ref_len else "N"

            if weird and rng.random() < 0.1:
                path.append(("H", int(rng.integers(1, 5))))
            if weird and rng.random() < 0.2 and remaining > 20:
                n = int(rng.integers(1, 8))
                path.append(("S", n))
                expected += ["?"] * n
                remaining -= n
            if weird and rng.random() < 0.15 and remaining > 20:
                n = int(rng.integers(1, 6))
                full = rand_seq(rng, n + int(rng.integers(0, 4)))  # key sequence may be longer than the observed tail
                indels.append(B.IndelKeySpec(ref_head, B.INDEL_INDEL, 0, full, candidacy(ref_head, 1, 0, full)))
                leading = len(indels) - 1
                path.append(("I", n))
                expected += list(full[len(full) - n:])
                remaining -= n
            tail_budget = 0
            want_trailing_ins = weird and rng.random() < 0.15 and remaining > 30
            want_trailing_clip = weird and rng.random() < 0.2 and remaining > 30
            if want_trailing_ins:
                tail_budget += 5
            if want_trailing_clip:
                tail_budget += 7
            # internal structure: M (event M)*
            n_events = int(rng.integers(0, 4)) if remaining > 40 else 0
            body = remaining - tail_budget
            for e in range(n_events + 1):
                last_block = e == n_events
                m = body if last_block else int(rng.integers(3, max(4, body // (n_events + 1 - e))))
                m = max(1, min(m, body))
                mt = "=" if (weird and rng.random() < 0.1) else "M"
                path.append((mt, m))
                expected += [ref_at(ref_head + k) for k in range(m)]
                ref_head += m
                body -= m
                if last_block or body < 8:
                    if not last_block:
                        # fold what is left into a final match block
                        path.append(("M", body))
                        expected += [ref_at(ref_head + k) for k in range(body)]
                        ref_head += body
                        body = 0
                    break
                ev = rng.random()
                if ev < 0.3:  # insertion
                    n = int(rng.integers(1, min(6, body - 3) + 1))
                    s = rand_seq(rng, n)
                    indels.append(B.IndelKeySpec(ref_head, B.INDEL_INDEL, 0, s, candidacy(ref_head, 1, 0, s)))
                    path.append(("I", n))
                    expected += list(s)
                    body -= n
                elif ev < 0.6:  # deletion
                    n = int(rng.integers(1, 12))
                    indels.append(B.IndelKeySpec(ref_head, B.INDEL_INDEL, n, "", candidacy(ref_head, 1, n, "")))
                    path.append(("D", n))
                    ref_head += n
                elif ev < 0.75:  # swap, either order
                    ni = int(rng.integers(1, min(5, body - 3) + 1))
                    nd = int(rng.integers(1, 8))
                    s = rand_seq(rng, ni)
                    # complex (insert+delete) alleles are never candidates: IndelBuffer.cpp:118-129 sets doNotGenotype
                    indels.append(B.IndelKeySpec(ref_head, B.INDEL_INDEL, nd, s, False))
                    if rng.random() < 0.5:
                        path += [("I", ni), ("D", nd)]
                    else:
                        path += [("D", nd), ("I", ni)]
                    expected += list(s)
                    ref_head += nd
                    body -= ni
                elif ev < 0.9 and weird:  # SEQ_MISMATCH block with a MISMATCH key
                    n = int(rng.integers(1, min(4, body - 3) + 1))
                    s = rand_seq(rng, n)
                    indels.append(B.IndelKeySpec(ref_head, B.INDEL_MISMATCH, n, s, candidacy(ref_head, 2, n, s)))
                    path.append(("X", n))
                    expected += list(s)
                    ref_head += n
                    body -= n
                else:  # skip
                    n = int(rng.integers(1, 30))
                    path.append(("N", n))
                    ref_head += n
            remaining = tail_budget
            if want_trailing_ins:
                n = int(rng.integers(1, 6))
                full = rand_seq(rng, n + int(rng.integers(0, 4)))
                indels.append(B.IndelKeySpec(ref_head, B.INDEL_INDEL, 0, full, candidacy(ref_head, 1, 0, full)))
                trailing = len(indels) - 1
                path.append(("I", n))
                expected += list(full[:n])
                remaining -= n
            if remaining > 0:
                if want_trailing_clip:
                    path.append(("S", remaining))
                    expected += ["?"] * remaining
                else:
                    # give the spare bases back to the last match block is awkward after a trailing insert: soft-clip them
                    path.append(("S", remaining))
                    expected += ["?"] * remaining
                remaining = 0
            if weird and rng.random() < 0.05:
                path.append(("H", 3))
            assert len(expected) == L, (len(expected), L, path)
            if first:
                # derive the read from the first alignment's expectation, with sequencing noise
                for k in range(L):
                    e = expected[k]
                    b = e if e in BASES else BASES[int(rng.integers(0, 4))]
                    if rng.random() < 0.05:
                        b = BASES[int(rng.integers(0, 4))]
                    read_bases[k] = b
                first = False
            # merge adjacent same-type segments the generator may have produced
            merged: List[Tuple[str, int]] = []
            for t, l in path:
                if merged and merged[-1][0] == t and t in ("M", "=", "S"):
                    merged[-1] = (t, merged[-1][1] + l)
                else:
                    merged.append((t, l))
            alns.append(B.CandidateAlignmentSpec(r, pos, merged, indels, leading, trailing))
        codes = np.array([CODE_OF[b] for b in read_bases], dtype=np.uint8)
        if weird:
            z = rng.random(L)
            codes[z < 0.02] = 15  # N
            codes[(z >= 0.02) & (z < 0.03)] = 0  # '='
            codes[(z >= 0.03) & (z < 0.035)] = 3  # an IUPAC ambiguity nibble: matches nothing
        quals = rng.choice(QUALS, size=L, p=QUAL_P).astype(np.uint8)
        reads.append((codes, quals))
    return B.RegionSpec(ref, ref_begin, reads, alns)


def simple_region(rng: np.random.Generator, n_reads: int = 30, n_haps: int = 4, read_len: int = 150, ref_len: int = 420, ref_begin: int = 100000) -> B.RegionSpec:
    """A cfg2-shaped candidate locus: `n_haps` haplotypes (reference + alt indel alleles at one locus), every read scored
    against every haplotype."""
    ref = rand_seq(rng, ref_len)
    locus = ref_begin + ref_len // 2
    haps = [None]
    for _ in range(n_haps - 1):
        if rng.random() < 0.5:
            n = int(min(20, rng.geometric(0.4)))
            haps.append(("I", rand_seq(rng, n)))
        else:
            haps.append(("D", int(min(20, rng.geometric(0.4)))))
    reads, alns = [], []
    for r in range(n_reads):
        start = int(rng.integers(locus - read_len + 10, locus - 10))
        h = haps[int(rng.integers(0, n_haps))]
        # read sequence from haplotype h
        left = locus - start
        if h is None:
            s = ref[start - ref_begin: start - ref_begin + read_len]
        elif h[0] == "I":
            s = (ref[start - ref_begin: locus - ref_begin] + h[1] + ref[locus - ref_begin:])[:read_len]
        else:
            s = (ref[start - ref_begin: locus - ref_begin] + ref[locus - ref_begin + h[1]:])[:read_len]
        s = s.ljust(read_len, "A")
        q = rng.choice(np.array([11, 25, 37], np.uint8), size=read_len, p=[0.03, 0.07, 0.90])
        bases = np.array(list(s))
        err = rng.random(read_len) < 10.0 ** (-q.astype(np.float64) / 10.0)  # (uint8 would wrap under the minus sign)
        bases[err] = np.array(list(BASES))[rng.integers(0, 4, int(err.sum()))]
        reads.append((np.array([CODE_OF[b] for b in bases], np.uint8), q.astype(np.uint8)))
        for hh in haps:
            if hh is None:
                alns.append(B.CandidateAlignmentSpec(r, start, [("M", read_len)], []))
            elif hh[0] == "I":
                n = min(len(hh[1]), read_len - left)
                rest = read_len - left - n
                key = B.IndelKeySpec(locus, B.INDEL_INDEL, 0, hh[1], True)
                if rest > 0:
                    alns.append(B.CandidateAlignmentSpec(r, start, [("M", left), ("I", n), ("M", rest)], [key]))
                else:
                    alns.append(B.CandidateAlignmentSpec(r, start, [("M", left), ("I", n)], [key], trailing=0))
            else:
                key = B.IndelKeySpec(locus, B.INDEL_INDEL, hh[1], "", True)
                alns.append(B.CandidateAlignmentSpec(r, start, [("M", left), ("D", hh[1]), ("M", read_len - left)], [key]))
    return B.RegionSpec(ref, ref_begin, reads, alns)


# ------------------------------------------------------------------------------------------------------------------
# pileups
# ------------------------------------------------------------------------------------------------------------------
def random_pileups(rng: np.random.Generator, n_sites: int, depth: float = 30.0, alt_frac_choices=(0.0, 0.0, 0.0, 0.02, 0.1, 0.25, 0.5, 1.0),
                   filt_frac: float = 0.05, with_tier2: bool = False, n_ref_frac: float = 0.01, max_depth: int = 250):
    """-> PileupBatch.  Each site: Poisson depth, a minor allele at a random fraction, strand split, phred mix, a few filtered calls."""
    sites, t2, refs = [], [], []
    for _ in range(n_sites):
        n = int(min(max_depth, rng.poisson(depth)))
        ref_id = int(rng.integers(0, 4))
        alt_id = (ref_id + int(rng.integers(1, 4))) % 4
        af = float(rng.choice(alt_frac_choices))
        q = rng.choice(np.array([2, 3, 11, 17, 25, 30, 37, 40, 41, 60], np.uint8), size=n, p=[0.01, 0.01, 0.04, 0.04, 0.1, 0.1, 0.5, 0.1, 0.07, 0.03])
        base = np.where(rng.random(n) < af, alt_id, ref_id)
        err = rng.random(n) < 0.01
        base[err] = rng.integers(0, 4, int(err.sum()))
        fwd = rng.random(n) < 0.5
        nbr = rng.random(n) < 0.1
        filt = rng.random(n) < filt_frac
        tfilt = filt & (rng.random(n) < 0.5)
        sites.append(list(B.pack_call(q, base, fwd, nbr, filt, tfilt)))
        refs.append("N" if rng.random() < n_ref_frac else BASES[ref_id])
        if with_tier2:
            m = int(rng.poisson(depth * 0.1))
            q2 = rng.choice(np.array([11, 25, 37], np.uint8), size=m)
            b2 = np.where(rng.random(m) < af, alt_id, ref_id)
            t2.append(list(B.pack_call(q2, b2, rng.random(m) < 0.5, 0, rng.random(m) < 0.3, 0)))
    return B.PileupBatch.from_sites(sites, "".join(refs), None, t2 if with_tier2 else None)


def random_ga_problems(rng: np.random.Generator, n: int, qlen=(5, 120), rlen=(5, 150), n_frac=0.0):
    qs, rs = [], []
    for _ in range(n):
        R = int(rng.integers(rlen[0], rlen[1] + 1))
        r = rand_seq(rng, R, n_frac)
        mode = rng.random()
        if mode < 0.7:
            # haplotype-like query: the reference with a few edits
            q = list(r)
            for _ in range(int(rng.integers(0, 5))):
                if not q:
                    break
                p = int(rng.integers(0, len(q)))
                e = rng.random()
                if e < 0.4:
                    q[p] = BASES[int(rng.integers(0, 4))]
                elif e < 0.7:
                    del q[p: p + int(rng.integers(1, 8))]
                else:
                    q[p:p] = list(rand_seq(rng, int(rng.integers(1, 8))))
            q = "".join(q)
            if rng.random() < 0.2:
                q = rand_seq(rng, int(rng.integers(1, 6))) + q
            if rng.random() < 0.2:
                q = q + rand_seq(rng, int(rng.integers(1, 6)))
            if not q:
                q = "A"
        else:
            q = rand_seq(rng, int(rng.integers(qlen[0], qlen[1] + 1)), n_frac)
        qs.append(q)
        rs.append(r)
    return qs, rs


def random_indel_loci(rng: np.random.Generator, n_loci: int, depth=(5, 60)):
    """Orthogonal allele groups with 1..4 non-ref indel alleles; per read a ref-path score and one score per allele, shaped like
    the max-path scores score_indels leaves in ReadPathScores (a read supports one allele strongly, the rest weakly)."""
    loci = []
    for _ in range(n_loci):
        A_ = int(rng.choice([1, 1, 1, 2, 2, 3, 4]))
        alleles = []
        for _a in range(A_):
            if rng.random() < 0.5:
                alleles.append((int(min(49, rng.geometric(0.3))), 0))
            elif rng.random() < 0.8:
                alleles.append((0, int(min(49, rng.geometric(0.3)))))
            else:
                alleles.append((int(rng.integers(1, 10)), int(rng.integers(1, 10))))
        n = int(rng.integers(depth[0], depth[1]))
        reads = []
        for _r in range(n):
            rl = int(rng.choice([75, 100, 150, 151, 8]))
            supp = int(rng.integers(0, A_ + 1))
            v = rng.normal(-60.0, 15.0, A_ + 1)
            v[supp] = rng.normal(-8.0, 4.0)
            if rng.random() < 0.1:
                v[:] = v[supp]  # uninformative read
            reads.append(([float(np.float32(min(x, -0.01))) for x in v], rl, int(rng.integers(max(1, rl - 10), rl + 1)), int(rng.random() < 0.5)))
        loci.append({"ploidy": int(rng.choice([2, 2, 2, 1])), "alleles": alleles, "reads": reads})
    return loci


def random_pileup_reads(rng: np.random.Generator, n_reads: int = 200, ref_len: int = 1200, ref_begin: int = 5000, read_len=(40, 151), n_frac: float = 0.02,
                        snv_rate: float = 0.01, allow_skip: bool = False):
    """Reads piled over one contig segment, in pile-up order: plain matches, internal and edge insertions / deletions, soft and hard
    clips, N runs at either end, mismatches (some of them registered as candidate SNVs), all three mapping tiers, both strands,
    low mapping qualities (the mapq adjustment), reads hanging off the report range."""
    ref = rand_seq(rng, ref_len)
    alt = {}  # position -> alt base of a "true" SNV (registered as candidate for about half of them)
    for p in rng.choice(ref_len, size=max(1, int(snv_rate * ref_len)), replace=False).tolist():
        alt[p] = BASES[(BASES.index(ref[p]) + 1 + int(rng.integers(0, 3))) % 4]
    cand = [(ref_begin + p, BASES.index(b)) for p, b in alt.items() if rng.random() < 0.5]
    reads = []
    starts = np.sort(rng.integers(-60, ref_len - 20, size=n_reads))
    for s0 in starts.tolist():
        L = int(rng.integers(read_len[0], read_len[1]))
        path, bases = [], []
        remaining, rp = L, s0
        if rng.random() < 0.1:
            path.append(("H", int(rng.integers(1, 6))))
        if rng.random() < 0.15 and remaining > 30:
            n = int(rng.integers(1, 9))
            path.append(("S", n))
            bases += list(rand_seq(rng, n))
            remaining -= n
        if rng.random() < 0.08 and remaining > 30:  # leading-edge insertion
            n = int(rng.integers(1, 5))
            path.append(("I", n))
            bases += list(rand_seq(rng, n))
            remaining -= n
        if rng.random() < 0.05:  # leading-edge deletion
            n = int(rng.integers(1, 5))
            path.append(("D", n))
            rp += n
        tail_clip = int(rng.integers(1, 9)) if (rng.random() < 0.15 and remaining > 30) else 0
        remaining -= tail_clip
        n_ev = int(rng.choice([0, 0, 0, 1, 1, 2]))
        while remaining > 0:
            m = remaining if n_ev == 0 else int(rng.integers(1, max(2, remaining - 2 * n_ev)))
            path.append(("M", m))
            for k in range(m):
                q = rp + k
                b = ref[q] if 0 <= q < ref_len else "A"
                if q in alt and rng.random() < 0.5:
                    b = alt[q]
                elif rng.random() < 0.02:
                    b = BASES[int(rng.integers(0, 4))]
                bases.append(b)
            rp += m
            remaining -= m
            if remaining <= 0 or n_ev == 0:
                continue
            n_ev -= 1
            u = rng.random()
            if u < 0.4:
                n = int(min(remaining - 1, rng.integers(1, 6))) if remaining > 1 else 0
                if n > 0:
                    path.append(("I", n))
                    bases += list(rand_seq(rng, n))
                    remaining -= n
            elif u < 0.9 or not allow_skip:
                n = int(rng.integers(1, 8))
                path.append(("D", n))
                rp += n
            else:
                n = int(rng.integers(20, 60))
                path.append(("N", n))
                rp += n
        if rng.random() < 0.04:  # trailing-edge deletion
            path.append(("D", int(rng.integers(1, 4))))
        if tail_clip:
            path.append(("S", tail_clip))
            bases += list(rand_seq(rng, tail_clip))
        # merge adjacent equal kinds (a path never repeats a kind back to back)
        merged = []
        for k, n in path:
            if merged and merged[-1][0] == k:
                merged[-1] = (k, merged[-1][1] + n)
            else:
                merged.append((k, n))
        bases = np.array(bases)
        assert len(bases) == L
        codes = np.array([CODE_OF[b] for b in bases], np.uint8)
        if rng.random() < n_frac * 5:  # N run at an end (ambiguous end trimming), N inside
            n = int(rng.integers(1, 6))
            if rng.random() < 0.5:
                codes[:n] = 15
            else:
                codes[-n:] = 15
        codes[rng.random(L) < n_frac * 0.2] = 15
        quals = rng.choice(QUALS, size=L, p=QUAL_P).astype(np.uint8)
        tier = int(rng.choice([1, 1, 1, 1, 2, 0]))
        reads.append(B.PileupReadSpec(codes, quals, ref_begin + s0, merged, fwd=bool(rng.random() < 0.5), mapq=int(rng.choice([0, 3, 12, 30, 60, 60, 60, 255])), tier=tier))
    return reads, ref, ref_begin, cand


_PATH_ENUM = {"M": 1, "I": 2, "D": 3, "N": 4, "S": 5, "H": 6}  # ALIGNPATH::align_t (blt_util/align_path.hh:36-48)


def _alignment_order_key(aln, fwd):
    """CandidateAlignment::operator< (CandidateAlignment.hh:37-47): alignment (pos, strand, path size, segments), then the indel set."""
    pos, path, kidx = aln
    return (pos, int(fwd), len(path), [(_PATH_ENUM[k], ln) for k, ln in path], list(kidx))


def random_score_indels_regions(rng: np.random.Generator, n_regions: int = 8, reads_per_region=(1, 6), alns_per_read=(1, 7), tie_rate: float = 0.5):
    """Regions for K6: per region a window of IndelBuffer entries (deletions, insertions, swaps, a few mismatch entries; candidates
    and non-candidates; shifted copies of the same deletion / insertion so that late_indel_normalization_filter finds equivalent
    alignments) and reads whose candidate alignments carry consistent paths over subsets of the window.  Returns (regions, lnp)."""
    regions, lnp = [], []
    for _ in range(n_regions):
        base = int(rng.integers(1000, 100000))
        # ---- window
        specs = {}
        n_keys = int(rng.integers(1, 8))
        while len(specs) < n_keys:
            pos = base + int(rng.integers(20, 140))
            t = rng.random()
            if t < 0.45:
                k = B.WindowKeySpec(pos, del_len=int(rng.integers(1, 12)))
            elif t < 0.8:
                k = B.WindowKeySpec(pos, ins=rand_seq(rng, int(rng.integers(1, 5))))
            elif t < 0.92:
                k = B.WindowKeySpec(pos, del_len=int(rng.integers(1, 5)), ins=rand_seq(rng, int(rng.integers(1, 4))))
            else:
                k = B.WindowKeySpec(pos, del_len=1, ins=rand_seq(rng, 1), mismatch=True)
            specs[k.order()] = k
            if not k.mismatch and rng.random() < 0.35:  # the same event one or two bases over: an "equivalent" indel
                k2 = B.WindowKeySpec(pos + int(rng.integers(1, 3)), del_len=k.del_len, ins=k.ins)
                specs[k2.order()] = k2
        win = [specs[o] for o in sorted(specs)]
        for k in win:
            k.candidate = bool(rng.random() < 0.8)
            k.ref_to_indel_lnp = float(np.log(rng.choice([1e-4, 5e-5, 2e-5, 1e-3]) * (1 + 0.01 * rng.integers(0, 3))))
            k.indel_to_ref_lnp = float(np.log(rng.choice([1e-4, 5e-5, 2e-5, 1e-3]) * (1 + 0.01 * rng.integers(0, 3))))
        # ---- reads
        reads = []
        for _r in range(int(rng.integers(reads_per_region[0], reads_per_region[1] + 1))):
            L = int(rng.integers(30, 151))
            fwd = bool(rng.random() < 0.5)
            start0 = base + int(rng.integers(-40, 120))
            alns = {}
            for _a in range(int(rng.integers(alns_per_read[0], alns_per_read[1] + 1))):
                start = start0 + int(rng.integers(-3, 4)) * int(rng.random() < 0.3)
                lead_clip = int(rng.integers(1, 8)) if rng.random() < 0.15 else 0
                trail_clip = int(rng.integers(1, 8)) if rng.random() < 0.15 else 0
                lead_ins = int(rng.integers(1, 6)) if rng.random() < 0.08 else 0
                path, kidx = [], []
                if rng.random() < 0.05:
                    path.append(("H", int(rng.integers(1, 5))))
                if lead_clip:
                    path.append(("S", lead_clip))
                remaining = L - lead_clip - trail_clip
                if lead_ins and lead_ins < remaining - 2:
                    path.append(("I", lead_ins))
                    remaining -= lead_ins
                ref_head = start
                take_p = rng.choice([0.0, 0.3, 0.6, 0.9])
                for i, k in enumerate(win):
                    if k.mismatch:
                        if ref_head <= k.pos and rng.random() < 0.3:
                            kidx.append(i)  # no trace in the path (a SEQ_MISMATCH block is sent as MATCH)
                        continue
                    if k.pos <= ref_head or rng.random() >= take_p:
                        continue
                    m = k.pos - ref_head
                    if m + len(k.ins) >= remaining - 1:
                        break
                    path.append(("M", m))
                    remaining -= m
                    if k.ins:
                        path.append(("I", len(k.ins)))
                        remaining -= len(k.ins)
                    if k.del_len:
                        path.append(("D", k.del_len))
                    ref_head = k.pos + k.del_len
                    kidx.append(i)
                if remaining <= 0:
                    continue
                trail_ins = int(rng.integers(1, 6)) if (rng.random() < 0.08 and remaining > 8) else 0
                path.append(("M", remaining - trail_ins))
                if trail_ins:
                    path.append(("I", trail_ins))
                if trail_clip:
                    path.append(("S", trail_clip))
                # merge adjacent equal kinds (M after M when a key was skipped cannot happen, but keep paths canonical)
                aln = (start, tuple(path), tuple(sorted(kidx)))
                alns[(start, tuple(path), tuple(sorted(kidx)))] = aln
            ordered = sorted(alns.values(), key=lambda a: _alignment_order_key(a, fwd))
            if not ordered:
                continue
            reads.append(B.ScoredReadSpec(L, [(a[0], list(a[1]), list(a[2])) for a in ordered], fwd=fwd, tier1=bool(rng.random() < 0.7),
                                          non_ambig=L - int(rng.integers(0, 3)), incomplete=bool(rng.random() < 0.2)))
            top = -float(rng.integers(8, 40))
            for _a in ordered:
                if rng.random() < tie_rate:
                    lnp.append(top - float(rng.choice([0.0, 0.0, 0.5, 2.0, 2.5])))
                else:
                    lnp.append(top - float(rng.random() * 12))
        regions.append((win, reads))
    return regions, np.array(lnp + [0.0], dtype=np.float64)


SCORE_INDELS_GOLDEN_CASES = 8


def score_indels_case(case: int):
    """The seeded K6 batch number `case` (tests/golden/score_indels_ref.npz holds the reference's output for cases 0..7; the
    option set cycles through oligo anchors, smoothing off, small maxIndelSize / large flank)."""
    from strelka_b200 import _abi as A

    rng = np.random.default_rng(1000 + case)
    regions, lnp = random_score_indels_regions(rng, 8, tie_rate=float(rng.choice([0.2, 0.5, 0.9])))
    opts = A.default_score_indels_opts()
    if case % 4 == 1:
        opts.upstream_oligo_size = int(rng.integers(1, 12))
    if case % 4 == 2:
        opts.is_smoothed_alignments = 0
    if case % 4 == 3:
        opts.max_indel_size = int(rng.integers(1, 20))
        opts.min_read_bp_flank = int(rng.integers(1, 40))
    return B.ScoreIndelsBatch(regions, opts), lnp


# ------------------------------------------------------------------------------------------------------------------------------
# K7 enumerate_alignments: regions with a reference, an IndelBuffer window and reads whose input alignments use some of its entries
# ------------------------------------------------------------------------------------------------------------------------------
def _keys_conflict(a, b) -> bool:
    """is_indel_conflict (indel_util.cpp:29-45)."""
    margin = 0 if (a.mismatch or b.mismatch) else 1
    return (b.pos + b.del_len + margin > a.pos) and (b.pos < a.pos + a.del_len + margin)


def random_enum_region(rng: np.random.Generator, n_reads: int = 6, ref_len: int = 420, ref_begin: int = 1000, n_keys=(1, 8), read_len=(30, 120), hap: bool = False,
                       n_samples: int = 1, cluster: bool = False, clip_rate: float = 0.1):
    ref = rand_seq(rng, ref_len)
    keys = {}
    centre = ref_begin + int(rng.integers(120, ref_len - 120))
    for _ in range(int(rng.integers(n_keys[0], n_keys[1] + 1))):
        pos = int(centre + rng.integers(-25, 26)) if cluster else ref_begin + int(rng.integers(70, ref_len - 90))
        u = rng.random()
        common = dict(candidate=bool(rng.random() < 0.8), not_discovered=bool(rng.random() < 0.12))
        if hap:
            common.update(active_region=int(rng.choice([-1, 0, 0, 1])), hap_ids=tuple(int(x) for x in rng.integers(0, 4, 4)), bypass=int(rng.integers(0, 4)) if rng.random() < 0.3 else 0,
                          forced=bool(rng.random() < 0.1))
        if u < 0.33:
            k = B.EnumKeySpec(pos, int(rng.integers(1, 13)), "", **common)
        elif u < 0.66:
            k = B.EnumKeySpec(pos, 0, rand_seq(rng, int(rng.integers(1, 11))), **common)
        elif u < 0.78:
            d = int(rng.integers(1, 7))
            common["candidate"] = False  # a complex allele is never a candidate (IndelBuffer.cpp:119-128, :218: doNotGenotype)
            k = B.EnumKeySpec(pos, d, rand_seq(rng, d if rng.random() < 0.4 else int(rng.integers(1, 7))), **common)
        else:
            rb = ref[pos - ref_begin]
            base = str(rng.choice([c for c in "ACGT" if c != rb]))
            if hap and common["active_region"] < 0:
                common["active_region"] = 0
            k = B.EnumKeySpec(pos, 1, base, mismatch=True, **common)
        keys.setdefault(k.order(), k)
    win = [keys[o] for o in sorted(keys)]
    mm_at = {k.pos: k for k in win if k.mismatch}
    reads = []
    for _ in range(n_reads):
        rl = int(rng.integers(read_len[0], read_len[1] + 1))
        u = rng.random()
        anchor = win[int(rng.integers(0, len(win)))]
        if u < 0.25:
            start = anchor.pos - int(rng.integers(1, 12))
        elif u < 0.5:
            start = anchor.pos - rl + int(rng.integers(-3, 10))
        else:
            start = anchor.pos - int(rng.integers(0, rl))
        start = max(ref_begin + 20, min(start, ref_begin + ref_len - rl - 40))
        # the indels the mapper's alignment already contains: a non-conflicting subset, spaced so that each is flanked by matches
        chosen = []
        for k in win:
            if k.mismatch or rng.random() > 0.35:
                continue
            if any(_keys_conflict(k, c) for c in chosen):
                continue
            chosen.append(k)
        path, seq, ref_pos, remaining = [], [], start, rl
        used = []

        def match(n):
            nonlocal ref_pos
            for _i in range(n):
                rb = ref[ref_pos - ref_begin]
                mk = mm_at.get(ref_pos)
                v = rng.random()
                if mk is not None and v < 0.5:
                    seq.append(mk.ins)
                elif v < 0.03:
                    seq.append(str(rng.choice(list("ACGT"))))
                elif v < 0.04:
                    seq.append("N")
                else:
                    seq.append(rb)
                ref_pos += 1

        for k in chosen:
            m = k.pos - ref_pos
            if m < 1 or m + len(k.ins) + 1 > remaining:
                continue
            match(m)
            path.append(("M", m))
            remaining -= m
            if k.del_len:
                path.append(("D", k.del_len))
                ref_pos += k.del_len
            if k.ins:
                path.append(("I", len(k.ins)))
                seq.append(k.ins)
                remaining -= len(k.ins)
            used.append(k)
        match(remaining)
        if path and path[-1][0] == "M":
            path[-1] = ("M", path[-1][1] + remaining)
        else:
            path.append(("M", remaining))
        seq = "".join(seq)
        assert len(seq) == rl
        if rng.random() < clip_rate:  # hard clips (not part of read_size()).  Soft clips never reach getCandidateAlignments: its caller
            # matchifies them first (starling_read_align.cpp:2051-2057), and the reference asserts (:466) on some soft-clipped inputs
            if rng.random() < 0.6:
                path.insert(0, ("H", int(rng.integers(1, 20))))
            if rng.random() < 0.6:
                path.append(("H", int(rng.integers(1, 20))))
        index_of = {k.order(): i for i, k in enumerate(win)}
        use = [index_of[k.order()] for k in used if not k.candidate and rng.random() > 0.03]
        use += [i for i, k in enumerate(win) if not k.candidate and rng.random() < 0.3]
        reads.append(B.EnumReadSpec(seq, start, path, use))
    if rng.random() < 0.15 and reads:
        r = reads[int(rng.integers(0, len(reads)))]
        span = sum(ln for t, ln in r.path if t in "MD=X")
        realign = (r.pos - int(rng.integers(0, 15)), r.pos + span + int(rng.integers(0, 15)))
    else:
        realign = (ref_begin + 5, ref_begin + ref_len - 5)
    return ref, ref_begin, realign, win, reads


def enum_case(case: int, n_regions: int = 6):
    """Seeded K7 batches: plain windows, clustered (conflicting) windows, phased active-region windows with two samples, dense windows
    (the density and max-toggle limits), tight toggle budgets."""
    rng = np.random.default_rng(7000 + case)
    mode = case % 6
    opts = A.default_enum_opts()
    kw = {}
    if mode == 1:
        kw = dict(cluster=True, n_keys=(2, 9))
    elif mode == 2:
        kw = dict(hap=True, cluster=bool(case & 8), n_keys=(2, 8))
        opts.is_haplotyping_enabled = 1
        opts.n_samples = 2
        opts.sample_id = (case // 6) % 2
    elif mode == 3:
        kw = dict(cluster=True, n_keys=(8, 16), read_len=(30, 60))
    elif mode == 4:
        opts.max_read_indel_toggle = int(rng.integers(0, 4))
        kw = dict(cluster=bool(case & 8))
    elif mode == 5:
        kw = dict(hap=True, n_keys=(1, 6), clip_rate=0.4)
        opts.is_haplotyping_enabled = int(case & 8 != 0)
    regions = [random_enum_region(rng, n_reads=int(rng.integers(1, 7)), **kw) for _ in range(n_regions)]
    return B.EnumBatch(regions, opts)


ENUM_GOLDEN_CASES = 12


def score_indels_batch_from_enumeration(eb: "B.EnumBatch", out: "B.EnumOut", ref_to_indel_lnp=-9.9, indel_to_ref_lnp=-9.9, k6_segs=None) -> "B.ScoreIndelsBatch":
    """K7's output as K6's input: the same alignments in the same (std::set) order with the same key lists; only the segment kinds
    are relabelled ('=' / 'X' are MATCH for score_indels, DELETE keeps its own kind) and the per-read fields K6 needs are added."""
    kind = np.zeros(16, np.uint8)
    kind[[A.SX_AP_MATCH, A.SX_AP_SEQ_MATCH, A.SX_AP_SEQ_MISMATCH]] = A.SX_SEG_MATCH
    kind[A.SX_AP_INSERT], kind[A.SX_AP_DELETE], kind[A.SX_AP_SOFT_CLIP], kind[A.SX_AP_HARD_CLIP] = A.SX_SEG_INSERT, 5, A.SX_SEG_SOFTCLIP, A.SX_SEG_HARDCLIP
    aln_off, _st, aln_pos, aln_seg_off, segs, aln_key_off, aln_keys, _lead, _trail = out.trimmed()
    segs2 = np.zeros(len(segs) + 16, dtype=A.ALN_SEG_DT)
    segs2["len"][: len(segs)] = segs["len"]
    segs2["kind"][: len(segs)] = kind[segs["kind"]]
    if k6_segs is not None:  # the relabelled copy K7b wrote (sx_link_out.k6_segs): must be this array
        assert k6_segs[: len(segs)].tobytes() == segs2[: len(segs)].tobytes()
    keys = eb.keys.copy()
    keys["ref_to_indel_lnp"], keys["indel_to_ref_lnp"] = ref_to_indel_lnp, indel_to_ref_lnp
    n_win = np.diff(eb.region_key_off.astype(np.int64))
    read_region = np.repeat(np.arange(eb.n_regions), np.diff(eb.region_read_off.astype(np.int64)))
    rec_off = np.concatenate([[0], np.cumsum(n_win[read_region])]).astype(np.uint32)
    arrays = dict(region_read_off=eb.region_read_off, region_key_off=eb.region_key_off, keys=keys, aln_off=aln_off, aln_pos=np.concatenate([aln_pos, [0]]).astype(np.int32),
                  aln_seg_off=aln_seg_off, segs=segs2, aln_key_off=aln_key_off, aln_keys=np.concatenate([aln_keys, [0]]).astype(np.uint16), read_len=eb.read_len,
                  non_ambig=eb.read_len.copy(), read_flags=np.full(eb.n_reads + 1, A.SX_SIF_FWD | A.SX_SIF_TIER1, np.uint8), rec_off=rec_off)
    return B.ScoreIndelsBatch.from_arrays(arrays)


def enum_edge_case(case: int, n_regions: int = 5):
    """K7a / K7 inputs outside the tidy ones enum_case makes: input alignments with leading / trailing edge insertions and deletions
    (RNA-style pinned edges), indels that are no window entries (private indels: SX_NO_KEY, the reference throws), adjacent
    insert + delete runs in both orders, read bases '=' and non-ACGT letters."""
    rng = np.random.default_rng(9000 + case)
    regions = []
    for _ in range(n_regions):
        ref, ref_begin, realign, win, reads = random_enum_region(rng, n_reads=int(rng.integers(2, 7)), cluster=bool(case & 1), n_keys=(2, 8), clip_rate=0.2)
        extra = {}
        out_reads = []
        for r in reads:
            path, seq, pos = list(r.path), r.seq, r.pos
            body = [i for i, (t, _l) in enumerate(path) if t != "H"]
            u = rng.random()
            if u < 0.3 and path[body[0]][0] == "M" and path[body[0]][1] > 8:  # leading edge insertion (+ sometimes a deletion behind it)
                n = int(rng.integers(1, 5))
                i0 = body[0]
                path[i0] = ("M", path[i0][1] - n)
                ins = [("I", n)]  # (an insertion + deletion at the leading edge makes the reference assert, starling_read_align.cpp:461)
                path[i0:i0] = ins
                pos += n  # the first n read bases are inserted: the match now starts n reference bases further on
                if rng.random() < 0.7:  # make the edge key(s) window entries
                    rp = pos
                    for t, ln in ins:
                        k = B.EnumKeySpec(rp, ln if t == "D" else 0, seq[:n] if t == "I" else "", candidate=bool(rng.random() < 0.5))
                        extra.setdefault(k.order(), k)
                        rp += ln if t == "D" else 0
            elif u < 0.55 and path[body[-1]][0] == "M" and path[body[-1]][1] > 8:  # trailing edge insertion / deletion
                i1 = body[-1]
                if rng.random() < 0.5:
                    n = int(rng.integers(1, 5))
                    path[i1] = ("M", path[i1][1] - n)
                    path.insert(i1 + 1, ("I", n))
                    end = pos + sum(ln for t, ln in path if t in "MD=X")
                    if rng.random() < 0.7:
                        k = B.EnumKeySpec(end, 0, seq[len(seq) - n:], candidate=True)
                        extra.setdefault(k.order(), k)
                else:
                    d = int(rng.integers(1, 6))
                    end = pos + sum(ln for t, ln in path if t in "MD=X")
                    path.insert(i1 + 1, ("D", d))
                    if rng.random() < 0.7:
                        k = B.EnumKeySpec(end, d, "", candidate=True)
                        extra.setdefault(k.order(), k)
            elif u < 0.75:  # a private indel in the middle of the first long match: not a window entry
                for i, (t, ln) in enumerate(path):
                    if t == "M" and ln > 20:
                        a = int(rng.integers(5, ln - 5))
                        if rng.random() < 0.5:
                            path[i:i + 1] = [("M", a), ("D", int(rng.integers(1, 4))), ("M", ln - a)]
                        else:
                            n = int(rng.integers(1, 4))
                            path[i:i + 1] = [("M", a), ("I", n), ("D", int(rng.integers(1, 4))), ("M", ln - a - n)] if rng.random() < 0.5 else [("M", a), ("I", n), ("M", ln - a - n)]
                        break
            if rng.random() < 0.3:  # '=' and IUPAC letters among the read bases
                s = list(seq)
                for _i in range(3):
                    s[int(rng.integers(0, len(s)))] = str(rng.choice(list("=NRYM")))
                seq = "".join(s)
            out_reads.append(B.EnumReadSpec(seq, pos, path, r.use_keys))
        keys = {k.order(): k for k in win}
        # the read-specific `use_keys` were window indices of the old window: recompute them by key
        old_order = [k.order() for k in win]
        keys.update({o: k for o, k in extra.items() if o not in keys})
        new_win = [keys[o] for o in sorted(keys)]
        index_of = {k.order(): i for i, k in enumerate(new_win)}
        for r in out_reads:
            r.use_keys = sorted({index_of[old_order[w]] for w in r.use_keys} | {i for i, k in enumerate(new_win) if not k.candidate and rng.random() < 0.5})
        regions.append((ref, ref_begin, realign, new_win, out_reads))
    return B.EnumBatch(regions, strict=False)


# K9 choose_realignment: the batches whose reference results are frozen in tests/golden/realign_ref.npz
REALIGN_GOLDEN_CASES = [("enum", c) for c in range(10)] + [("edge", c) for c in (1, 3, 5, 7)]
REALIGN_MODES = {"ln10": (True, 2.302585092994046), "off": (False, 2.3), "wide": (True, 25.0), "all": (True, 400.0)}


def realign_case_batch(name: str, case: int):
    return enum_edge_case(case) if name == "edge" else enum_case(case)


def realign_quals(eb, case: int) -> np.ndarray:
    """one quality per read base of the batch (the K1 read pools of the realignment tests use the same values)."""
    rng = np.random.default_rng(4242 + case)
    return rng.choice(np.array([11, 25, 37], np.uint8), int(eb.read_off[eb.n_reads]) + 1)


def raw_alignments_for(eb, case: int):
    """Mapper-style alignments for the reads of an EnumBatch: its normalized input alignments made raw again -- soft clips cut out of the
    first / last match, edge insertions and deletions kept, sometimes an over-long deletion (not realignable) -- so that every gate of
    realignAndScoreRead has something to decide."""
    rng = np.random.default_rng(31000 + case)
    raw = []
    for r in range(eb.n_reads):
        path = [(B.AP_CHAR[int(s["kind"])], int(s["len"])) for s in eb.in_segs[int(eb.in_seg_off[r]) : int(eb.in_seg_off[r + 1])]]
        pos = int(eb.in_pos[r])
        body = [i for i, (t, _l) in enumerate(path) if t != "H"]
        u = rng.random()
        if u < 0.35 and path[body[0]][0] == "M" and path[body[0]][1] > 6:  # leading soft clip
            n = int(rng.integers(1, 5))
            i0 = body[0]
            path[i0] = ("M", path[i0][1] - n)
            path.insert(i0, ("S", n))
            pos += n
        if rng.random() < 0.35:
            body = [i for i, (t, _l) in enumerate(path) if t != "H"]
            i1 = body[-1]
            if path[i1][0] == "M" and path[i1][1] > 6:  # trailing soft clip
                n = int(rng.integers(1, 5))
                path[i1] = ("M", path[i1][1] - n)
                path.insert(i1 + 1, ("S", n))
        if rng.random() < 0.05:  # an interior deletion longer than maxIndelSize
            for i, (t, ln) in enumerate(path):
                if t == "M" and ln > 20 and 0 < i < len(path) - 1 or (t == "M" and ln > 20 and len(path) == 1):
                    a = ln // 2
                    path[i:i + 1] = [("M", a), ("D", 60), ("M", ln - a)]
                    break
        raw.append((pos, path))
    return raw


GATES_GOLDEN_CASES = 12


# ------------------------------------------------------------------------------------------------------------------------------
# K2b / K5 edge batches, run at every parameter point of tests/site_params.py
# ------------------------------------------------------------------------------------------------------------------------------
SOMATIC_EDGE_KINDS = ("plain", "normal_empty", "tumor_empty", "both_empty", "q_extreme", "t1_tier_filtered", "t1_all_filtered", "n_ref", "alt_tie", "deep",
                      "t1_weak")
# the kinds that are computed only when forced: both samples empty, or no tier1 call left in either (an all-reference tier1 view ends the
# site before the model, position_somatic_snv_strand_grid.cpp:253).  An 'N' reference is never computed.  A tier1 result of qphred 0
# ("t1_weak") makes the tier2 result a copy of it (:272-277), which is reported only when forced (:311-312).
SOMATIC_FORCED_ONLY_KINDS = ("both_empty", "t1_all_filtered")
_ORD_Q = np.array([11, 17, 25, 30, 37, 40, 41, 60], np.uint8)
_ORD_Q_P = np.array([0.04, 0.04, 0.1, 0.1, 0.5, 0.1, 0.08, 0.04])


def _edge_calls(rng, n, ref_id, mix, q=None, filt=0.0, tfilt=0.0):
    """n calls: base ids drawn from mix {base_id: weight} (the rest of the weight goes to ref_id), ordinary qualities unless `q` is
    given, both strands, a few neighbour mismatches, a fraction `filt` filtered of which a fraction `tfilt` tier-specifically."""
    ids = [ref_id] + list(mix)
    w = np.array([max(0.0, 1.0 - sum(mix.values()))] + list(mix.values()))
    base = rng.choice(np.array(ids), size=n, p=w / w.sum()) if n else np.zeros(0, np.int64)
    if q is None:
        q = rng.choice(_ORD_Q, size=n, p=_ORD_Q_P)
    f = rng.random(n) < filt
    tf = f & (rng.random(n) < tfilt)
    return list(B.pack_call(q, base, rng.random(n) < 0.5, rng.random(n) < 0.1, f, tf))


def somatic_edge_sites(rng: np.random.Generator, reps: int = 120):
    """-> (normal PileupBatch, tumor PileupBatch, forced[n], kind[n]): `reps` sites of each SOMATIC_EDGE_KINDS kind in random order,
    about 40% of them forced, tier2 calls on both samples (somatic_tier2_view drops them).  Kinds: ordinary sites; an empty normal,
    tumor or both; qualities 0, 1 and 63 among ordinary ones; tier1 calls mostly filtered, tier-specifically, so that they survive into
    the tier2 view; every tier1 call filtered; an 'N' reference; two or three alt bases of equal count; several hundred calls per
    sample; a tier1 view too weak for a call with a strong tier2 one."""
    kinds = rng.permutation(np.repeat(np.arange(len(SOMATIC_EDGE_KINDS)), reps))
    sn, st, sn2, st2, refs = [], [], [], [], []
    for k in kinds.tolist():
        kind = SOMATIC_EDGE_KINDS[k]
        ref_id = int(rng.integers(0, 4))
        alt = (ref_id + int(rng.integers(1, 4))) % 4
        noise = {alt: float(rng.choice([0.0, 0.0, 0.01, 0.02]))}
        taf = {alt: float(rng.choice([0.05, 0.15, 0.3, 0.5]))}
        n_n, n_t = int(rng.poisson(30)), int(rng.poisson(50))
        m_n, m_t = int(rng.poisson(4)), int(rng.poisson(8))
        nmix, tmix, t2mix = noise, taf, taf
        nkw, tkw = {}, {}
        ref = BASES[ref_id]
        if kind == "normal_empty":
            n_n = m_n = 0
        elif kind == "tumor_empty":
            n_t = m_t = 0
            nmix = {alt: float(rng.choice([0.0, 0.3, 0.5]))}
        elif kind == "both_empty":
            n_n = m_n = n_t = m_t = 0
        elif kind == "q_extreme":
            for kw, nn in ((nkw, n_n), (tkw, n_t)):
                q = rng.choice(_ORD_Q, size=nn, p=_ORD_Q_P)
                x = rng.random(nn) < float(rng.choice([0.1, 0.3, 0.6]))
                q[x] = rng.choice(np.array([0, 1, 63], np.uint8), size=int(x.sum()))
                kw["q"] = q
        elif kind == "t1_tier_filtered":
            nkw = dict(filt=0.3, tfilt=0.8)
            tkw = dict(filt=float(rng.choice([0.5, 0.7, 0.9])), tfilt=0.85)
        elif kind == "t1_all_filtered":
            nkw = tkw = dict(filt=1.0, tfilt=0.5)
        elif kind == "n_ref":
            ref = "N"
        elif kind == "alt_tie":
            others = [b for b in range(4) if b != ref_id]
            rng.shuffle(others)
            c = int(rng.integers(1, 12))
            ties = others[: int(rng.choice([2, 2, 3]))]
            nr = int(rng.poisson(30))
            sample = [ref_id] * nr + [b for b in ties for _ in range(c)]
            sample = [sample[i] for i in rng.permutation(len(sample))]
            n_t, tmix = len(sample), None
            tkw = dict(base=np.array(sample))
            if rng.random() < 0.5:  # a tie in the normal as well
                nsample = [ref_id] * int(rng.poisson(30)) + ties[:2] * int(rng.integers(1, 3))
                n_n, nmix, nkw = len(nsample), None, dict(base=np.array(nsample))
        elif kind == "deep":
            n_n, n_t = int(rng.integers(300, 800)), int(rng.integers(300, 800))
            tmix = {alt: float(rng.choice([0.02, 0.05, 0.1, 0.3]))}
        elif kind == "t1_weak":
            n_t, tmix = int(rng.integers(40, 80)), {alt: 1.0 / 80}
            m_t, t2mix = int(rng.integers(15, 40)), {alt: 0.5}

        def calls(n, mix, kw):
            if "base" in kw:  # the exact base sequence given
                b = kw["base"]
                return list(B.pack_call(rng.choice(_ORD_Q, size=len(b), p=_ORD_Q_P), b, rng.random(len(b)) < 0.5, 0, 0, 0))
            return _edge_calls(rng, n, ref_id, mix, **kw)

        sn.append(calls(n_n, nmix, nkw))
        st.append(calls(n_t, tmix, tkw))
        # tier2 calls: a third of them filtered (a filtered tier2 call never survives)
        sn2.append(_edge_calls(rng, m_n, ref_id, nmix or noise, filt=0.3))
        st2.append(_edge_calls(rng, m_t, ref_id, t2mix or taf, filt=0.3))
        refs.append(ref)
    refs = "".join(refs)
    forced = (rng.random(len(kinds)) < 0.4).astype(np.uint8)
    return B.PileupBatch.from_sites(sn, refs, None, sn2), B.PileupBatch.from_sites(st, refs, None, st2), forced, kinds.astype(np.uint8)


SOMATIC_TIER2_MODES = ("both", "neither", "normal_only", "tumor_only")


def somatic_tier2_view(npb, tpb, mode: str):
    """the pair with tier2 calls on both samples, on neither, or on one only (the ABI then evaluates tier1 only, like the reference's
    is_tier2 = both samples have them)"""
    keep_n, keep_t = {"both": (True, True), "neither": (False, False), "normal_only": (True, False), "tumor_only": (False, True)}[mode]

    def view(pb, keep):
        return pb if keep else B.PileupBatch(pb.site_off, pb.calls, pb.ref_base, pb.ploidy)

    return view(npb, keep_n), view(tpb, keep_t)


def pileup_take(pb, idx) -> "B.PileupBatch":
    """the sites idx[0], idx[1], ... of pb as a new batch (calls, tier2 calls, reference bases)"""
    idx = np.asarray(idx, np.int64)

    def gather(off, calls):
        off = off.astype(np.int64)
        depth = off[idx + 1] - off[idx]
        new_off = np.concatenate([[0], np.cumsum(depth)])
        src = np.repeat(off[idx] - new_off[:-1], depth) + np.arange(int(new_off[-1]))
        return new_off.astype(np.uint32), calls[src]

    off, calls = gather(pb.site_off, pb.calls)
    t2_off = t2_calls = None
    if pb.t2_off is not None:
        t2_off, t2_calls = gather(pb.t2_off, pb.t2_calls)
    return B.PileupBatch(off, calls, pb.ref_base[idx], None if pb.ploidy is None else pb.ploidy[idx], t2_off, t2_calls)


INDEL_EDGE_READ_COUNTS = (0, 1, 31, 32, 33, 63, 64, 65)  # K5 evaluates 32 reads per step


def indel_edge_loci(rng: np.random.Generator, reps: int = 2):
    """K5 loci: every read count of INDEL_EDGE_READ_COUNTS with A = 1..4 alleles at ploidy 1 and 2 (ploidy 2 with four alleles has
    SX_INDEL_MAX_GT = 15 genotypes), `reps` times.  Allele lengths from 0 to past the read length; read lengths and non-ambiguous base
    counts from 0 up, many below twice the largest flank; per read one strongly supported allele, an exact tie of two or more
    alleles, all alleles equal, or scores close together (posteriors near the support thresholds)."""
    lens = np.array([0, 0, 1, 2, 5, 20, 39, 40, 41, 79, 80, 81, 200], np.int64)
    loci = []
    for _ in range(reps):
        for n in INDEL_EDGE_READ_COUNTS:
            for A_ in range(1, 5):
                for ploidy in (1, 2):
                    alleles = []
                    for _a in range(A_):
                        d, i = int(rng.choice(lens)), int(rng.choice(lens))
                        u = rng.random()
                        alleles.append((max(d, 1), 0) if u < 0.4 else (0, max(i, 1)) if u < 0.8 else (d, i))
                    reads = []
                    for _r in range(n):
                        rl = int(rng.choice([1, 8, 20, 50, 78, 79, 80, 81, 100, 150, 151, 300]))
                        na = int(rng.choice([rl, rl, max(0, rl - 3), int(rng.integers(0, rl + 1))]))
                        u = rng.random()
                        v = rng.normal(-60.0, 15.0, A_ + 1)
                        if u < 0.4:
                            v[int(rng.integers(0, A_ + 1))] = rng.normal(-8.0, 4.0)
                        elif u < 0.65:
                            tie = rng.choice(A_ + 1, size=int(rng.integers(2, A_ + 2)), replace=False)
                            v[tie] = rng.normal(-8.0, 4.0)
                        elif u < 0.75:
                            v[:] = v[0]
                        else:
                            v = rng.normal(-10.0, 1.0, A_ + 1)
                        v = np.minimum(v, -0.01)
                        if rng.random() < 0.05:
                            v[int(rng.integers(0, A_ + 1))] = -1000.0
                        reads.append(([float(np.float32(x)) for x in v], rl, na, int(rng.random() < 0.5)))
                    loci.append({"ploidy": ploidy, "alleles": alleles, "reads": reads})
    return loci
