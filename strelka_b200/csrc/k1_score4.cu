// k1_score4.cu -- K1 fast path: scoreCandidateAlignment for batches in the 4-bit quality wire format (qual_bits == 4).
//
// Same contract as k1_score.cu (reference: starling_common/starling_read_align_score.cpp:260-499, one running double per (read,
// alignment) path, terms added in read order with __dadd_rn, addends from the host-built table), re-organised around what a
// profile of that kernel showed: it was bound by issue slots and shared-memory wavefronts, not by HBM, and less than half of its
// instructions were the per-cell work.  Here
//   * a read base is ONE byte: quality code << 4 | page << 2 | base (A C G T = 0..3).  The byte is, up to two masks, the address of
//     its term in a 1 KB table built per CTA from the quality dictionary: tab[page][quality code][mismatch], page 0 = ordinary base
//     (match, mismatch), 1 = '=' read base (match, match), 2 = 'N' read base (0, 0), 3 = any other read base (mismatch, mismatch).
//     Reference bases are 0..3 or 4 ("matches nothing"), so "mismatch" is ((entry & 3) ^ reference) != 0.  Rows are 16 bytes, so the
//     (match, mismatch) terms of different qualities lie in different banks.
//   * reads are expanded by one linear pass over the region's packed bytes (4 packed bytes -> 8 entries per lane and iteration,
//     through a 256-entry (nibble, quality code) table), not read by read;
//   * each alignment's segments are turned into 8-byte run records by a converged pre-pass, so the divergent part of the scoring loop
//     is a 10-instruction record fetch;
//   * the scoring loop handles 8 cells per iteration with SIMD-in-a-register byte arithmetic: 3+3 aligned 32-bit shared loads and
//     PRMT funnels fetch the 8 entries and 8 reference codes, six logic ops per 4 cells produce the table addresses (including the
//     substitution of the zero page for the cells past a run's end), and a cell is PRMT + LDS.64 + DADD.
// Regions that do not fit the 16-bit shared-window addresses used here (KQ_MAX_SMEM) are scored by the general kernel.
#include "k1_stage.cuh"

#include <cstring>

namespace
{
using namespace k1;

constexpr uint32_t PAGE_BASE = 0, PAGE_EQ = 1, PAGE_ZERO = 2, PAGE_NOMATCH = 3;
constexpr uint32_t REF_OTHER = 4;
constexpr uint32_t ENTRY_BAD = (PAGE_ZERO << 2) | 3u; // low nibble of an entry whose quality is out of range (scores as zero; flagged)
enum { REC_RUN = 0, REC_SOFT = 1, REC_OOW = 2, REC_END = 3 };

// shared-window loads by 32-bit address
__device__ __forceinline__ uint32_t lds_u8(uint32_t a)
{
    uint32_t v;
    asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t a)
{
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint2 lds_u64(uint32_t a)
{
    uint2 v;
    asm("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
    return v;
}
// run records are written and read back by the same thread: keep both in program order
__device__ __forceinline__ void sts_rec(uint32_t a, uint32_t x, uint32_t y) { asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory"); }
__device__ __forceinline__ uint2 lds_rec(uint32_t a)
{
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t s)
{
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(s));
    return d;
}

__device__ __forceinline__ uint32_t ref_code_of_char(uint32_t c) { return c == 'A' ? 0u : c == 'C' ? 1u : c == 'G' ? 2u : c == 'T' ? 3u : REF_OTHER; }

__device__ __forceinline__ uint32_t dict_at(const uint4& qd, uint32_t c)
{
    const uint32_t w = c < 4 ? qd.x : c < 8 ? qd.y : c < 12 ? qd.z : qd.w;
    return (w >> ((c & 3u) * 8u)) & 0xffu;
}

__global__ void __launch_bounds__(THREADS) k1q_score_kernel(const sx_region* __restrict__ regions, const uint16_t* __restrict__ read_len,
                                                            const uint8_t* __restrict__ seq4, const uint8_t* __restrict__ qual4,
                                                            const char* __restrict__ ref, const sx_aln* __restrict__ alns,
                                                            const sx_aln_seg* __restrict__ segs, const char* __restrict__ ins,
                                                            const sx_tables* __restrict__ tables, uint32_t region_begin, double* __restrict__ lnp_out,
                                                            int* __restrict__ status, uint32_t smem_bytes, uint4 qual_dict, uint32_t fmt, uint32_t qual_bits,
                                                            const uint32_t* __restrict__ exc_off, const uint32_t* __restrict__ exc)
{
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t ri = region_begin + blockIdx.x;
    const sx_region r0 = regions[ri];
    const sx_region r1 = regions[ri + 1];
    const qlayout L = make_qlayout(slices_of(r0, r1, fmt));
    if (L.n_alns == 0) return;
    const uint32_t sbase = smem_u32(smem);
    const uint32_t tab_saddr = (sbase + L.tab + 1023u) & ~1023u; // 1 KB-aligned in the shared window: a cell's address is two PRMT'd bytes
    if (L.total > smem_bytes || sbase + L.total > 0xffffu || tab_saddr + 1024u > 0x7f00u || L.n_segs > 0xffffu)
    {
        if (threadIdx.x == 0) atomicOr(status, SX_ST_TILE);
        return;
    }
    const uint32_t tid = threadIdx.x;
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
    uint2* lut = reinterpret_cast<uint2*>(smem + L.lut);
    uint8_t* e8 = smem + L.e8;
    double* tab = reinterpret_cast<double*>(smem + (tab_saddr - sbase)); // [4 pages][16 quality codes][match, mismatch]
    const bool aln8 = fmt & SX_FMT_ALN8, seg2 = fmt & SX_FMT_SEG2, baseq = fmt & SX_FMT_BASEQ, ref4 = fmt & SX_FMT_REF4;
    const aln_reader rd(smem, L, r0, aln8, seg2);
    uint8_t* ref_s = smem + L.ref;
    uint8_t* ins_s = smem + L.ins;
    uint16_t* rlen_s = reinterpret_cast<uint16_t*>(smem + L.rlen);
    uint32_t* soff_s = reinterpret_cast<uint32_t*>(smem + L.soff);

    // ---- per-CTA tables (independent of the TMA data)
    if (tid < 64)
    {
        const uint32_t page = tid >> 4, q = min(dict_at(qual_dict, tid & 15u), (uint32_t)SX_MAX_QSCORE);
        const double x = tables->k1_tab[2 * q + 0], m = tables->k1_tab[2 * q + 1]; // (mismatch, match) terms of quality q
        tab[2 * tid + 0] = page == PAGE_ZERO ? 0.0 : page == PAGE_NOMATCH ? x : m;
        tab[2 * tid + 1] = page == PAGE_ZERO ? 0.0 : page == PAGE_EQ ? m : x;
    }
    for (uint32_t idx = tid; idx < 256; idx += THREADS)
    {
        // (read nibble << 4 | quality code) -> entry.  bam_seq::get_code nibbles: 0 '=', 1 A, 2 C, 4 G, 8 T, 15 N, others IUPAC.
        const uint32_t nib = idx >> 4, qc = idx & 15u;
        uint32_t e;
        if (nib == 15u) e = PAGE_ZERO << 2;                                          // skipped: adds +0.0, quality ignored
        else if (dict_at(qual_dict, qc) > SX_MAX_QSCORE) e = ENTRY_BAD;              // qphred_cache::qscore_check would throw
        else if (nib == 0u) e = PAGE_EQ << 2;                                        // always "is_ref"
        else if (nib == 1u || nib == 2u || nib == 4u || nib == 8u) e = (PAGE_BASE << 2) | (nib == 1u ? 0u : nib == 2u ? 1u : nib == 4u ? 2u : 3u);
        else e = PAGE_NOMATCH << 2;                                                  // IUPAC codes match nothing
        e8[idx] = static_cast<uint8_t>((qc << 4) | e);
    }
    if (tid < 9)
    {
        // page-field masks of the first n cells of a chunk (0x03 in the bytes of cells 0..n-1)
        const uint32_t nlo = min(tid, 4u), nhi = tid > 4u ? tid - 4u : 0u;
        const uint32_t lo = nlo ? (0x03030303u >> (32u - 8u * nlo)) : 0u, hi = nhi ? (0x03030303u >> (32u - 8u * nhi)) : 0u;
        lut[tid] = make_uint2(lo, hi);
    }

    if (tid == 0) issue_copies(smem, L, r0, aln8, seg2, ref4, alns, segs, ref, ins, seq4, qual4);
    for (uint32_t r = tid; r < L.n_reads; r += THREADS) rlen_s[r] = read_len[r0.read_begin + r];
    __syncthreads(); // rlen, tables visible; mbarrier initialised
    // packed-byte offset of every read (reads lie back to back, each padded to a whole byte): warp 0, shuffle scan
    if (tid < 32)
    {
        uint32_t carry = 0;
        for (uint32_t base = 0; base < L.n_reads; base += 32)
        {
            const uint32_t r = base + tid;
            const uint32_t nb = r < L.n_reads ? (rlen_s[r] + 1u) >> 1 : 0u;
            uint32_t x = nb;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1)
            {
                const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
                if (tid >= (uint32_t)d) x += y;
            }
            if (r < L.n_reads) soff_s[r] = carry + x - nb;
            carry += __shfl_sync(0xffffffffu, x, 31);
        }
        if (tid == 0) soff_s[L.n_reads] = carry;
    }
    mbar_wait(bar, 0);
    __syncthreads();
    if (soff_s[L.n_reads] > L.seq_bytes || (!baseq && (qual_bits == 2 ? (soff_s[L.n_reads] + 1) / 2 : soff_s[L.n_reads]) > L.qual_bytes))
    {
        if (tid == 0) atomicOr(status, SX_ST_TILE);
        return;
    }
    // ---- expansion: entry byte 2p / 2p+1 <- packed byte p (high nibble first), for the whole region at once
    {
        const uint32_t* seq32 = reinterpret_cast<const uint32_t*>(smem + L.seq);
        const uint32_t* qual32 = reinterpret_cast<const uint32_t*>(smem + L.qual);
        uint2* ent64 = reinterpret_cast<uint2*>(smem + L.ent);
        const uint32_t e8_s = sbase + L.e8;
        const uint32_t nw = (soff_s[L.n_reads] + 3u) >> 2;
        uint32_t acc = 0;
        if (baseq)
        {
            // one nibble per base, (base << 2) | quality code: the entry (code << 4 | page 0 << 2 | base) is a bit shuffle, no lookup;
            // the host guarantees every dictionary quality <= 70 in this format
            for (uint32_t w = tid; w < nw; w += THREADS)
            {
                const uint32_t s = seq32[w];
                const uint32_t h = (s >> 4) & 0x0f0f0f0fu, l = s & 0x0f0f0f0fu;  // first / second bases of the four packed bytes
                const uint32_t eh = ((h & 0x03030303u) << 4) | ((h >> 2) & 0x03030303u);
                const uint32_t el = ((l & 0x03030303u) << 4) | ((l >> 2) & 0x03030303u);
                ent64[w] = make_uint2(prmt(eh, el, 0x5140u), prmt(eh, el, 0x7362u)); // interleave back into read order
            }
            // the bases that are not A/C/G/T: 'N' -> zero page, '=' -> always-match page, IUPAC -> never-match page (quality code kept)
            const uint32_t x0 = exc_off[ri], x1 = exc_off[ri + 1];
            if (x1 > x0)
            {
                __syncthreads();
                uint8_t* ent8 = smem + L.ent;
                for (uint32_t i = x0 + tid; i < x1; i += THREADS)
                {
                    const uint32_t v = exc[i], pos = v & 0xffffffu, code = v >> 24;
                    if (pos >= 2u * soff_s[L.n_reads])
                    {
                        atomicOr(status, SX_ST_TILE);
                        continue;
                    }
                    const uint32_t page = code == 15u ? PAGE_ZERO : code == 0u ? PAGE_EQ : PAGE_NOMATCH;
                    ent8[pos] = static_cast<uint8_t>((ent8[pos] & 0xf0u) | (page << 2));
                }
            }
        }
        else
        for (uint32_t w = tid; w < nw; w += THREADS)
        {
            const uint32_t s = seq32[w];
            uint32_t q;
            if (qual_bits == 2)
            {
                // 16 bits = the 2-bit codes of this word's 8 nibbles, first nibble in the two high bits of the first byte; spread them
                // to the nibble layout of the 4-bit format (byte k: code of base 2k in the high nibble, of base 2k+1 in the low one)
                const uint32_t h = reinterpret_cast<const uint16_t*>(qual32)[w];
                const uint32_t b0 = h & 0xffu, b1 = h >> 8;
                q = (((b0 >> 2) & 0x30u) | ((b0 >> 4) & 0x03u)) | ((((b0 << 2) & 0x30u) | (b0 & 0x03u)) << 8) |
                    ((((b1 >> 2) & 0x30u) | ((b1 >> 4) & 0x03u)) << 16) | ((((b1 << 2) & 0x30u) | (b1 & 0x03u)) << 24);
            }
            else q = qual32[w];
            const uint32_t hi = (s & 0xf0f0f0f0u) | ((q >> 4) & 0x0f0f0f0fu); // table indices of the four first bases of the packed bytes
            const uint32_t lo = ((s << 4) & 0xf0f0f0f0u) | (q & 0x0f0f0f0fu); // ... and of the four second bases
            const uint32_t a0 = lds_u8(e8_s + (hi & 0xffu)), a1 = lds_u8(e8_s + (lo & 0xffu));
            const uint32_t a2 = lds_u8(e8_s + ((hi >> 8) & 0xffu)), a3 = lds_u8(e8_s + ((lo >> 8) & 0xffu));
            const uint32_t a4 = lds_u8(e8_s + ((hi >> 16) & 0xffu)), a5 = lds_u8(e8_s + ((lo >> 16) & 0xffu));
            const uint32_t a6 = lds_u8(e8_s + (hi >> 24)), a7 = lds_u8(e8_s + (lo >> 24));
            const uint32_t w0 = a0 | (a1 << 8) | (a2 << 16) | (a3 << 24);
            const uint32_t w1 = a4 | (a5 << 8) | (a6 << 16) | (a7 << 24);
            // ENTRY_BAD: low nibble 1011
            acc |= (w0 & (w0 >> 1) & ~(w0 >> 2) & (w0 >> 3)) | (w1 & (w1 >> 1) & ~(w1 >> 2) & (w1 >> 3));
            ent64[w] = make_uint2(w0, w1);
        }
        if (acc & 0x01010101u) atomicOr(status, SX_ST_QUAL);
        uint32_t* ref32 = reinterpret_cast<uint32_t*>(ref_s);
        if (ref4)
        {
            // packed BAM codes -> one reference code per byte (two per packed byte, high nibble first)
            const uint8_t* rp = smem + L.refp;
            uint16_t* ref16 = reinterpret_cast<uint16_t*>(ref_s);
            for (uint32_t i = tid; i < L.ref_bytes / 2; i += THREADS)
            {
                const uint32_t b = i < L.refp_bytes ? rp[i] : 0xffu;
                const uint32_t hi = b >> 4, lo = b & 15u;
                const uint32_t ch = hi == 1u ? 0u : hi == 2u ? 1u : hi == 4u ? 2u : hi == 8u ? 3u : REF_OTHER;
                const uint32_t cl = lo == 1u ? 0u : lo == 2u ? 1u : lo == 4u ? 2u : lo == 8u ? 3u : REF_OTHER;
                ref16[i] = static_cast<uint16_t>(ch | (cl << 8));
            }
        }
        else
        for (uint32_t i = tid; i < L.ref_bytes / 4; i += THREADS)
        {
            const uint32_t v = ref32[i];
            ref32[i] = ref_code_of_char(v & 0xffu) | (ref_code_of_char((v >> 8) & 0xffu) << 8) | (ref_code_of_char((v >> 16) & 0xffu) << 16) |
                       (ref_code_of_char(v >> 24) << 24);
        }
        for (uint32_t i = tid; i < L.ins_bytes; i += THREADS) ins_s[i] = static_cast<uint8_t>(ref_code_of_char(ins_s[i]));
    }
    __syncthreads();

    const double softclip = tables->k1_softclip;
    const double noncand = tables->k1_noncand;
    const int ref_len = static_cast<int>(r0.ref_len);
    const uint32_t ent_s0 = sbase + L.ent, ref_s0 = sbase + L.ref, ins_s0 = sbase + L.ins, recs_s0 = sbase + L.recs, lut_s0 = sbase + L.lut;
    // high address byte of a masked cell, in every byte lane: table page 2 (all zeros).  Bits 0-1 of tab_saddr >> 8 are clear, bit 7 too.
    const uint32_t k2 = ((tab_saddr >> 8) | PAGE_ZERO) * 0x01010101u;

    for (uint32_t a = tid; a < L.n_alns; a += THREADS)
    {
        const uint4 h = rd.aln_at(a);
        const uint32_t rl = h.x;
        const uint32_t seg0 = h.z, seg1 = rd.seg_end(a);
        if (rl >= L.n_reads || seg1 > L.n_segs || seg0 > seg1)
        {
            atomicOr(status, SX_ST_TILE);
            continue;
        }
        const uint32_t rec0 = recs_s0 + (seg0 + a) * 8u; // this alignment's records: one per segment at most, + END
        // ---- pass 1 (lanes run it together): segments -> run records.  A record is {x, y}: y = n | type << 16 | pre << 24, where `pre`
        // non-candidate-indel penalties are added before the record is executed (the reference adds the penalty of a non-candidate indel
        // segment after that segment's bases, score.cpp:404-470).
        {
            uint32_t ent = ent_s0 + 2u * soff_s[rl];
            int read_left = rlen_s[rl];
            int refp = static_cast<int>(h.y);
            uint32_t insp = ins_s0 + h.w;
            uint32_t rp = rec0, pre = 0;
            for (uint32_t s = seg0; s < seg1; ++s)
            {
                const uint32_t seg = rd.seg_at(s);
                const int len = static_cast<int>(seg & 0xffffu);
                const uint32_t kind = (seg >> 16) & 0xffu;
                if (kind == SX_SEG_MATCH || kind == SX_SEG_INSERT || kind == SX_SEG_SOFTCLIP)
                {
                    if (len > read_left)
                    {
                        atomicOr(status, SX_ST_READ_OVERRUN);
                        break;
                    }
                    read_left -= len;
                }
                if (kind == SX_SEG_MATCH)
                {
                    if (refp >= 0 && refp + len <= ref_len) sts_rec(rp, ent | ((ref_s0 + refp) << 16), len | (REC_RUN << 16) | (pre << 24));
                    else sts_rec(rp, ent | (s << 16), len | (REC_OOW << 16) | (pre << 24)); // leaves the held reference window
                    rp += 8;
                    pre = 0;
                    ent += len;
                    refp += len;
                }
                else if (kind == SX_SEG_INSERT)
                {
                    sts_rec(rp, ent | (insp << 16), len | (REC_RUN << 16) | (pre << 24));
                    rp += 8;
                    pre = 0;
                    ent += len;
                    insp += len;
                }
                else if (kind == SX_SEG_REFSKIP) refp += len;
                else if (kind == SX_SEG_SOFTCLIP)
                {
                    sts_rec(rp, len, (REC_SOFT << 16) | (pre << 24));
                    rp += 8;
                    pre = 0;
                    ent += len;
                }
                else if (kind != SX_SEG_HARDCLIP) atomicOr(status, SX_ST_SEG_KIND);
                if ((seg >> 24) & SX_SEGF_NONCANDIDATE)
                {
                    if (pre == 255u) atomicOr(status, SX_ST_SEG_KIND);
                    else ++pre;
                }
            }
            sts_rec(rp, 0, (REC_END << 16) | (pre << 24));
        }
        // ---- pass 2: execute the records
        double lnp = 0.0;
        uint32_t rem = 0, ent = 0, cp = 0, sel_e = 0, sel_c = 0, rp = rec0;
        for (;;)
        {
            bool done = false;
            while (rem == 0)
            {
                const uint2 rec = lds_rec(rp);
                rp += 8;
#pragma unroll 1
                for (uint32_t p = rec.y >> 24; p; --p) lnp = __dadd_rn(lnp, noncand);
                const uint32_t type = (rec.y >> 16) & 0xffu;
                if (type == REC_RUN)
                {
                    ent = rec.x & 0xffffu;
                    cp = rec.x >> 16;
                    rem = rec.y & 0xffffu;
                    sel_e = 0x3210u + 0x1111u * (ent & 3u); // PRMT selectors: bytes (addr & 3) .. +3 of an aligned word pair
                    sel_c = 0x3210u + 0x1111u * (cp & 3u);
                }
                else if (type == REC_SOFT)
                {
                    lnp = __dadd_rn(lnp, __dmul_rn(static_cast<double>(rec.x), softclip));
                }
                else if (type == REC_OOW)
                {
                    // part of the segment lies outside the held reference window: those positions read as 'N'.  Rare: plain loop.
                    int p0 = static_cast<int>(h.y);
                    for (uint32_t ss = seg0; ss < (rec.x >> 16); ++ss)
                    {
                        const uint32_t sg = rd.seg_at(ss), k = (sg >> 16) & 0xffu;
                        if (k == SX_SEG_MATCH || k == SX_SEG_REFSKIP) p0 += static_cast<int>(sg & 0xffffu);
                    }
                    const uint32_t ea = rec.x & 0xffffu, len = rec.y & 0xffffu;
                    for (uint32_t i = 0; i < len; ++i)
                    {
                        const uint32_t e = lds_u8(ea + i);
                        const int p = p0 + static_cast<int>(i);
                        const uint32_t c = (p >= 0 && p < ref_len) ? ref_s[p] : REF_OTHER;
                        lnp = __dadd_rn(lnp, lds_f64(tab_saddr + ((e >> 2) & 3u) * 256u + (e & 0xf0u) + (((e & 3u) ^ c) ? 8u : 0u)));
                    }
                }
                else
                {
                    done = true;
                    break;
                }
            }
            if (done) break;
            // One chunk of 8 cells.  Cells past the end of the run are sent to the all-zero table page through the byte masks of lut[n]
            // (x + 0.0 == x exactly for every x this sum can hold); surplus loads stay inside the CTA's shared memory, and whatever they
            // return only picks a row inside that page.
            {
                const uint32_t n = min(rem, 8u);
                const uint2 mk = lds_u64(lut_s0 + n * 8u);
                const uint32_t ea = ent & ~3u, ca = cp & ~3u;
                const uint32_t w0 = lds_u32(ea), w1 = lds_u32(ea + 4), w2 = lds_u32(ea + 8);
                const uint32_t v0 = lds_u32(ca), v1 = lds_u32(ca + 4), v2 = lds_u32(ca + 8);
                const uint32_t e0 = prmt(w0, w1, sel_e), e1 = prmt(w1, w2, sel_e);
                const uint32_t c0 = prmt(v0, v1, sel_c), c1 = prmt(v1, v2, sel_c);
                // per byte: low address byte = quality code * 16 + mismatch * 8, high address byte = table base | page
                // ((e & 3) ^ c is 0..7 in a live cell, so + 7 sets bit 3 iff it is non-zero; a surplus byte may carry, but only upwards,
                // into other surplus bytes)
                const uint32_t a0 = (e0 & 0xf0f0f0f0u) | ((((e0 & 0x03030303u) ^ c0) + 0x07070707u) & 0x08080808u);
                const uint32_t a1 = (e1 & 0xf0f0f0f0u) | ((((e1 & 0x03030303u) ^ c1) + 0x07070707u) & 0x08080808u);
                const uint32_t x0 = ((e0 >> 2) & mk.x) | (k2 & ~mk.x);
                const uint32_t x1 = ((e1 >> 2) & mk.y) | (k2 & ~mk.y);
                // selector: byte 0 = a[k], byte 1 = x[k], bytes 2-3 = sign of x[k] replicated (= 0)
                lnp = __dadd_rn(lnp, lds_f64(prmt(a0, x0, 0xcc40u)));
                lnp = __dadd_rn(lnp, lds_f64(prmt(a0, x0, 0xdd51u)));
                lnp = __dadd_rn(lnp, lds_f64(prmt(a0, x0, 0xee62u)));
                lnp = __dadd_rn(lnp, lds_f64(prmt(a0, x0, 0xff73u)));
                lnp = __dadd_rn(lnp, lds_f64(prmt(a1, x1, 0xcc40u)));
                lnp = __dadd_rn(lnp, lds_f64(prmt(a1, x1, 0xdd51u)));
                lnp = __dadd_rn(lnp, lds_f64(prmt(a1, x1, 0xee62u)));
                lnp = __dadd_rn(lnp, lds_f64(prmt(a1, x1, 0xff73u)));
                ent += n;
                cp += n;
                rem -= n;
            }
        }
        lnp_out[r0.aln_begin + a] = lnp;
    }
}
} // namespace

int sx_k1q_launch(sx_ctx* ctx, const sx_align_batch* d, uint32_t region_begin, uint32_t region_end, double* lnp_dev, size_t smem_bytes, cudaStream_t st)
{
    if (region_end <= region_begin) return SX_OK;
    if (smem_bytes > 48 * 1024)
        SX_CUDA(ctx, cudaFuncSetAttribute(k1q_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(k1::KQ_MAX_SMEM)));
    uint4 qd;
    memcpy(&qd, d->qual_dict, 16);
    k1q_score_kernel<<<region_end - region_begin, k1::THREADS, smem_bytes, st>>>(d->regions, d->read_len, d->seq4, d->qual, d->ref, d->alns, d->segs, d->ins,
                                                                                 ctx->d_tables, region_begin, lnp_dev, ctx->d_status, static_cast<uint32_t>(smem_bytes), qd, d->format, d->qual_bits, d->exc_off, d->exc);
    SX_CUDA(ctx, cudaGetLastError());
    return SX_OK;
}
