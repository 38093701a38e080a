// k1_score.cu -- K1 score_alignments: ln P(read | one candidate alignment path) for every (read, alignment) pair.
//
// Replaces scoreCandidateAlignment  (/root/reference/src/c++/lib/starling_common/starling_read_align_score.cpp:260-499,
// scoreMatchSegment :142-170, scoreInsertSegment :108-137) over the loop at starling_read_align.cpp:1568-1571.
//
// Bit-exactness contract: the reference accumulates one running double per path, term by term in read order
// (score.cpp:104-106 explains why: equal scores must stay exactly equal so ambiguous alignments tie).  A reduction tree
// would reorder the additions, so each (read, alignment) pair is summed by ONE thread in read order with __dadd_rn; the
// parallelism is across pairs.  The addends come from a 143-row table built on the host with the host libm
// (sx_context.cu), so there is no transcendental on the device.
//
// Data movement: one CTA per region.  Every pool slice of the region (packed bases, qualities, reference window,
// alignment headers, segments, inserted bases, the term table) is pulled into shared memory by TMA bulk copies
// (cp.async.bulk ... mbarrier::complete_tx) issued by one thread; each read is then expanded ONCE into a 16-bit
// (table-row | one-hot base) entry that all of its H alignments share, so HBM sees every read byte exactly once.
#include "sx_internal.h"
#include "k1q_layout.cuh"

#include <algorithm>
#include <cstring>

namespace
{
constexpr int K1_THREADS = 128;
constexpr int K1_TAB_BYTES = SX_K1_ROWS * 16;
constexpr int K1_CHUNK = 8;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase)
{
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(phase)
        : "memory");
}
// TMA 1-D bulk copy global -> shared, completion counted in bytes on an mbarrier.  16-byte aligned src/dst/size.
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)), "l"(src_gmem),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// 8-byte shared-memory load from a shared-window address
__device__ __forceinline__ double lds_f64(uint32_t saddr)
{
    double v;
    asm("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(saddr));
    return v;
}

__host__ __device__ __forceinline__ uint32_t pad16(uint32_t x) { return (x + 15u) & ~15u; }

struct k1_layout
{
    uint32_t tab, alns, segs, ref, refp, ins, seq, qual, rlen, boff, soff, eoff, desc, ent, total;
    uint32_t n_reads, n_alns, seg_bytes, ref_bytes, refp_bytes, ins_bytes, seq_bytes, qual_bytes;
};

__host__ __device__ __forceinline__ k1_layout k1_make_layout(const sx_region& r0, const sx_region& r1, uint32_t fmt)
{
    k1_layout L;
    L.n_reads = r1.read_begin - r0.read_begin;
    L.n_alns = r1.aln_begin - r0.aln_begin;
    L.seg_bytes = pad16((r1.seg_begin - r0.seg_begin) * ((fmt & SX_FMT_SEG2) ? 2u : 4u));
    L.ref_bytes = pad16(r0.ref_len);
    L.ins_bytes = pad16(r1.ins_begin - r0.ins_begin);
    L.seq_bytes = pad16(static_cast<uint32_t>(r1.seq_off - r0.seq_off));
    L.qual_bytes = (fmt & SX_FMT_BASEQ) ? 0u : pad16(static_cast<uint32_t>(r1.qual_off - r0.qual_off));
    L.refp_bytes = (fmt & SX_FMT_REF4) ? pad16((r0.ref_len + 1u) / 2u) : 0u;
    uint32_t o = 16; // mbarrier
    L.tab = o;
    o += K1_TAB_BYTES;
    L.alns = o;
    o += k1q::aln_slice_bytes(r0.aln_begin, L.n_alns, fmt);
    L.segs = o;
    o += L.seg_bytes;
    L.ref = o;
    o += L.ref_bytes;
    L.refp = o;
    o += L.refp_bytes;
    L.ins = o;
    o += L.ins_bytes;
    L.seq = o;
    o += L.seq_bytes;
    L.qual = o;
    o += L.qual_bytes;
    L.rlen = o;
    o += pad16(L.n_reads * 2u);
    L.boff = o;
    o += pad16((L.n_reads + 1) * 4u);
    L.soff = o;
    o += pad16((L.n_reads + 1) * 4u);
    L.eoff = 0;
    L.desc = o;
    o += 64 + 16; // 16 nibble descriptors + the 16-entry quality dictionary
    L.ent = o;
    // entries: 2 bytes per base, every read padded to an even count; + slack: the uniform chunk loop may load (and discard) up to
    // K1_CHUNK-1 entries past a read
    o += L.seq_bytes * 4u + 32u;
    L.total = o;
    return L;
}

// reference base (ASCII) -> one-hot nibble; everything that is not ACGT (N, '=', IUPAC) -> 0, which ANDs to "mismatch" with every
// read nibble.  (get_bam_seq_code maps such characters to ANY=15; a read nibble of 15 never reaches the compare, and 15 equals no
// other read nibble, so "never matches" is the same relation.)
__device__ __forceinline__ uint8_t onehot_of_char(uint8_t c)
{
    return c == 'A' ? 1 : c == 'C' ? 2 : c == 'G' ? 4 : c == 'T' ? 8 : 0;
}

__global__ void __launch_bounds__(K1_THREADS) k1_score_kernel(const sx_region* __restrict__ regions, const uint16_t* __restrict__ read_len,
                                                              const uint8_t* __restrict__ seq4, const uint8_t* __restrict__ qual,
                                                              const char* __restrict__ ref, const sx_aln* __restrict__ alns,
                                                              const sx_aln_seg* __restrict__ segs, const char* __restrict__ ins,
                                                              const sx_tables* __restrict__ tables, uint32_t region_begin, double* __restrict__ lnp_out,
                                                              int* __restrict__ status, uint32_t smem_bytes, uint32_t qual_bits, uint4 qual_dict, uint32_t fmt,
                                                              const uint32_t* __restrict__ exc_off, const uint32_t* __restrict__ exc)
{
    extern __shared__ __align__(128) unsigned char smem[];
    const uint32_t ri = region_begin + blockIdx.x;
    const sx_region r0 = regions[ri];
    const sx_region r1 = regions[ri + 1];
    const k1_layout L = k1_make_layout(r0, r1, fmt);
    if (L.n_alns == 0) return;
    if (L.total > smem_bytes)
    {
        if (threadIdx.x == 0) atomicOr(status, SX_ST_TILE);
        return;
    }
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
    const double* tab = reinterpret_cast<const double*>(smem + L.tab);
    // alignment headers and segments, read through accessors that hide the wire format (sx_aln / sx_aln8, sx_aln_seg / sx_aln_seg2)
    const bool aln8 = fmt & SX_FMT_ALN8, seg2 = fmt & SX_FMT_SEG2, baseq = fmt & SX_FMT_BASEQ, ref4 = fmt & SX_FMT_REF4;
    const uint32_t aln_skew = aln8 ? (r0.aln_begin & 1u) : 0u; // the sx_aln8 slice is staged from a 16-byte boundary
    const uint32_t n_segs_region = r1.seg_begin - r0.seg_begin;
    const unsigned char* alns_raw = smem + L.alns;
    const unsigned char* segs_raw = smem + L.segs;
    auto aln_at = [&](uint32_t a) -> uint4 { // region-relative: x read, y first reference position, z first segment, w first inserted base
        if (aln8)
        {
            const uint2 v = reinterpret_cast<const uint2*>(alns_raw)[a + aln_skew];
            return make_uint4(v.x & 0xffffu, static_cast<uint32_t>(static_cast<int32_t>(v.x) >> 16), v.y & 0xffffu, v.y >> 16);
        }
        const uint4 h = reinterpret_cast<const uint4*>(alns_raw)[a];
        return make_uint4(h.x - r0.read_begin, h.y - static_cast<uint32_t>(r0.ref_begin), h.z - r0.seg_begin, h.w - r0.ins_begin);
    };
    auto seg_end_of = [&](uint32_t a) -> uint32_t {
        if (aln8) return a + 1 < L.n_alns ? aln_at(a + 1).z : n_segs_region;
        return reinterpret_cast<const uint4*>(alns_raw)[a + 1].z - r0.seg_begin;
    };
    auto seg_at = [&](uint32_t s) -> uint32_t { // len | kind << 16 | flags << 24
        if (seg2)
        {
            const uint32_t v = reinterpret_cast<const uint16_t*>(segs_raw)[s];
            return (v & 0xfffu) | (((v >> 12) & 7u) << 16) | ((v >> 15) << 24);
        }
        return reinterpret_cast<const uint32_t*>(segs_raw)[s];
    };
    uint8_t* ref_s = smem + L.ref;
    uint8_t* ins_s = smem + L.ins;
    const uint8_t* seq_s = smem + L.seq;
    const uint8_t* qual_s = smem + L.qual;
    uint16_t* rlen_s = reinterpret_cast<uint16_t*>(smem + L.rlen);
    uint32_t* boff_s = reinterpret_cast<uint32_t*>(smem + L.boff);
    uint32_t* soff_s = reinterpret_cast<uint32_t*>(smem + L.soff);
    uint32_t* desc_s = reinterpret_cast<uint32_t*>(smem + L.desc);
    uint16_t* ent_s = reinterpret_cast<uint16_t*>(smem + L.ent);
    const uint32_t tab_saddr = smem_u32(tab); // shared-window address of the term table
    if (tab_saddr + K1_TAB_BYTES > 0xfff0u || (tab_saddr & 15u))
    {
        if (threadIdx.x == 0) atomicOr(status, SX_ST_TILE);
        return;
    }
    // quality dictionary of the 4-bit wire format lives in the descriptor block's tail (16 bytes after the 16 descriptors)
    uint8_t* qd_s = reinterpret_cast<uint8_t*>(desc_s + 16);
    if (threadIdx.x < 16)
    {
        const uint32_t w = threadIdx.x >> 2, sh = (threadIdx.x & 3u) * 8u;
        const uint32_t word = w == 0 ? qual_dict.x : w == 1 ? qual_dict.y : w == 2 ? qual_dict.z : qual_dict.w;
        qd_s[threadIdx.x] = static_cast<uint8_t>(word >> sh);
    }
    if (threadIdx.x < 16)
    {
        const uint32_t code = threadIdx.x;
        uint32_t d;
        if (code == 15u) d = (SX_K1_ROW_ZERO << 4);                                   // BAM_BASE::ANY: skipped (adds +0.0), q ignored
        else if (code == 0u) d = (SX_K1_ROW_EQ << 4) | 0xffff0000u;                   // BAM_BASE::REF: always "is_ref"
        else d = ((code == 1u || code == 2u || code == 4u || code == 8u) ? code : 0u) | 0xffff0000u; // other nibbles match nothing
        // entries carry the ABSOLUTE shared-memory address of their table row (16-byte aligned, < 64 KB), so the scoring loop
        // forms the load address with one LOP3 and no add
        desc_s[code] = d + tab_saddr;
    }

    if (threadIdx.x == 0)
    {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        const uint32_t aln_bytes = k1q::aln_slice_bytes(r0.aln_begin, L.n_alns, fmt);
        const uint32_t ref_tx = ref4 ? L.refp_bytes : L.ref_bytes;
        const uint32_t tx = K1_TAB_BYTES + aln_bytes + L.seg_bytes + ref_tx + L.ins_bytes + L.seq_bytes + L.qual_bytes;
        mbar_expect_tx(bar, tx);
        tma_bulk_g2s(smem + L.tab, tables->k1_tab, K1_TAB_BYTES, bar);
        tma_bulk_g2s(smem + L.alns, reinterpret_cast<const unsigned char*>(alns) + (aln8 ? (size_t)(r0.aln_begin & ~1u) * 8u : (size_t)r0.aln_begin * 16u), aln_bytes, bar);
        if (L.seg_bytes) tma_bulk_g2s(smem + L.segs, reinterpret_cast<const unsigned char*>(segs) + (size_t)r0.seg_begin * (seg2 ? 2u : 4u), L.seg_bytes, bar);
        if (ref_tx) tma_bulk_g2s(smem + (ref4 ? L.refp : L.ref), ref + r0.ref_off, ref_tx, bar);
        if (L.ins_bytes) tma_bulk_g2s(smem + L.ins, ins + r0.ins_begin, L.ins_bytes, bar);
        if (L.seq_bytes) tma_bulk_g2s(smem + L.seq, seq4 + r0.seq_off, L.seq_bytes, bar);
        if (L.qual_bytes) tma_bulk_g2s(smem + L.qual, qual + r0.qual_off, L.qual_bytes, bar);
    }
    // read lengths: tiny, plain coalesced loads (their offset has no 16-byte alignment guarantee)
    for (uint32_t r = threadIdx.x; r < L.n_reads; r += K1_THREADS) rlen_s[r] = read_len[r0.read_begin + r];
    __syncthreads(); // rlen visible, mbarrier initialised
    // per-read base / packed-byte offsets: warp 0, shuffle scan
    if (threadIdx.x < 32)
    {
        uint32_t carry_b = 0, carry_s = 0;
        for (uint32_t base = 0; base < L.n_reads; base += 32)
        {
            const uint32_t r = base + threadIdx.x;
            const uint32_t len = r < L.n_reads ? rlen_s[r] : 0;
            uint32_t xb = len, xs = (len + 1) >> 1;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1)
            {
                const uint32_t yb = __shfl_up_sync(0xffffffffu, xb, d);
                const uint32_t ys = __shfl_up_sync(0xffffffffu, xs, d);
                if (threadIdx.x >= d)
                {
                    xb += yb;
                    xs += ys;
                }
            }
            if (r < L.n_reads)
            {
                boff_s[r] = carry_b + xb - len;
                soff_s[r] = carry_s + xs - ((len + 1) >> 1);
            }
            carry_b += __shfl_sync(0xffffffffu, xb, 31);
            carry_s += __shfl_sync(0xffffffffu, xs, 31);
        }
        if (threadIdx.x == 0)
        {
            boff_s[L.n_reads] = carry_b;
            soff_s[L.n_reads] = carry_s;
        }
    }
    mbar_wait(bar, 0);
    __syncthreads();
    if ((!baseq && (qual_bits == 2 ? (soff_s[L.n_reads] + 1) / 2 : qual_bits == 4 ? soff_s[L.n_reads] : boff_s[L.n_reads]) > L.qual_bytes) || soff_s[L.n_reads] > L.seq_bytes)
    {
        if (threadIdx.x == 0) atomicOr(status, SX_ST_TILE);
        return;
    }
    // expand each read once: entry = (table row << 4) | one-hot base.  One packed byte (two bases) per lane and iteration; the
    // per-nibble part of the entry comes from a 16-entry descriptor table: low half = (row base << 4) | one-hot nibble, high half =
    // mask applied to (q << 4)  (0 for 'N': the zero row ignores q).
    {
        const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
        uint32_t qmax = 0; // largest quality seen on a non-N base: the reference only looks at those (score.cpp:125-126,158-159)
        for (uint32_t r = warp; r < L.n_reads; r += K1_THREADS / 32)
        {
            const uint32_t len = rlen_s[r];
            const uint8_t* sq = seq_s + soff_s[r];
            const uint8_t* ql = qual_s + (qual_bits == 4 ? soff_s[r] : boff_s[r]);
            uint32_t* en2 = reinterpret_cast<uint32_t*>(ent_s) + soff_s[r]; // every read is padded to an even entry count: entry offset = 2*soff
            const uint32_t npair = (len + 1) >> 1;
            for (uint32_t p = lane; p < npair; p += 32)
            {
                const uint32_t byte = sq[p];
                // bam_seq::get_code nibbles, high nibble first; SX_FMT_BASEQ nibbles are (base << 2) | quality code
                const uint32_t d0 = desc_s[baseq ? (1u << (byte >> 6)) : (byte >> 4)], d1 = desc_s[baseq ? (1u << ((byte >> 2) & 3u)) : (byte & 15u)];
                uint32_t q0, q1;
                if (baseq)
                {
                    q0 = qd_s[(byte >> 4) & 3u];
                    q1 = (2 * p + 1 < len) ? qd_s[byte & 3u] : 0u;
                }
                else if (qual_bits == 4)
                {
                    const uint32_t qb = ql[p]; // both qualities of the pair in one byte, high nibble first
                    q0 = qd_s[qb >> 4];
                    q1 = (2 * p + 1 < len) ? qd_s[qb & 15u] : 0u;
                }
                else if (qual_bits == 2)
                {
                    // one 2-bit code per nibble position of the region's seq4 slice: packed byte b = soff + p holds positions 2b, 2b+1
                    const uint32_t b = soff_s[r] + p, qb = qual_s[b >> 1] >> ((~b & 1u) << 2);
                    q0 = qd_s[(qb >> 2) & 3u];
                    q1 = (2 * p + 1 < len) ? qd_s[qb & 3u] : 0u;
                }
                else
                {
                    q0 = ql[2 * p];
                    q1 = (2 * p + 1 < len) ? ql[2 * p + 1] : 0u;
                }
                qmax = max(qmax, (d0 >> 16) ? q0 : 0u);
                qmax = max(qmax, (d1 >> 16) ? q1 : 0u);
                const uint32_t lo = (d0 & 0xffffu) + ((min(q0, (uint32_t)SX_MAX_QSCORE) << 4) & (d0 >> 16));
                const uint32_t hi = (d1 & 0xffffu) + ((min(q1, (uint32_t)SX_MAX_QSCORE) << 4) & (d1 >> 16));
                en2[p] = lo | (hi << 16);
            }
        }
        if (qmax > SX_MAX_QSCORE) atomicOr(status, SX_ST_QUAL);
        if (baseq && exc_off[ri + 1] > exc_off[ri])
        {
            // the bases that are not A/C/G/T: rebuild their entries from the real code (the nibble kept the quality code)
            __syncthreads();
            for (uint32_t i = exc_off[ri] + threadIdx.x; i < exc_off[ri + 1]; i += K1_THREADS)
            {
                const uint32_t v = exc[i], pos = v & 0xffffffu, d = desc_s[(v >> 24) & 15u];
                if (pos >= 2u * soff_s[L.n_reads])
                {
                    atomicOr(status, SX_ST_TILE);
                    continue;
                }
                const uint32_t q = qd_s[(seq_s[pos >> 1] >> ((~pos & 1u) << 2)) & 3u];
                ent_s[pos] = static_cast<uint16_t>((d & 0xffffu) + ((min(q, (uint32_t)SX_MAX_QSCORE) << 4) & (d >> 16)));
            }
        }
        if (ref4)
        {
            const uint8_t* rp = smem + L.refp; // packed BAM codes -> one-hot codes, two per packed byte
            for (uint32_t i = threadIdx.x; i < L.ref_bytes; i += K1_THREADS)
            {
                const uint32_t b = (i >> 1) < L.refp_bytes ? rp[i >> 1] : 0xffu, c = (i & 1u) ? (b & 15u) : (b >> 4);
                ref_s[i] = static_cast<uint8_t>((c == 1u || c == 2u || c == 4u || c == 8u) ? c : 0u);
            }
        }
        else
        for (uint32_t i = threadIdx.x; i < L.ref_bytes; i += K1_THREADS) ref_s[i] = onehot_of_char(ref_s[i]);
        for (uint32_t i = threadIdx.x; i < L.ins_bytes; i += K1_THREADS) ins_s[i] = onehot_of_char(ins_s[i]);
    }
    __syncthreads();

    const double softclip = tables->k1_softclip;
    const double noncand = tables->k1_noncand;
    const uint32_t zero_entry = (SX_K1_ROW_ZERO << 4) + tab_saddr; // the all-zero table row: adds +0.0
    const int ref_len = static_cast<int>(r0.ref_len);

    for (uint32_t a = threadIdx.x; a < L.n_alns; a += K1_THREADS)
    {
        const uint4 h = aln_at(a);
        const uint32_t rl = h.x;
        if (rl >= L.n_reads)
        {
            atomicOr(status, SX_ST_TILE);
            continue;
        }
        const uint16_t* ent = ent_s + 2u * soff_s[rl];
        int read_left = static_cast<int>(boff_s[rl + 1] - boff_s[rl]);
        int refp = static_cast<int>(h.y);
        const uint8_t* insp = ins_s + h.w;
        uint32_t s = h.z;
        const uint32_t s_end = seg_end_of(a);
        double lnp = 0.0;
        int rem = 0;
        bool pend = false;
        const uint8_t* cp = ref_s;
        for (;;)
        {
            bool done = false;
            while (rem == 0)
            {
                if (pend)
                {
                    lnp = __dadd_rn(lnp, noncand);
                    pend = false;
                }
                if (s == s_end)
                {
                    done = true;
                    break;
                }
                const uint32_t seg = seg_at(s++);
                const int len = static_cast<int>(seg & 0xffffu);
                const uint32_t kind = (seg >> 16) & 0xffu;
                pend = (seg >> 24) & SX_SEGF_NONCANDIDATE;
                if (kind == SX_SEG_MATCH || kind == SX_SEG_INSERT || kind == SX_SEG_SOFTCLIP)
                {
                    if (len > read_left)
                    {
                        atomicOr(status, SX_ST_READ_OVERRUN);
                        done = true;
                        break;
                    }
                    read_left -= len;
                }
                if (kind == SX_SEG_MATCH)
                {
                    if (refp >= 0 && refp + len <= ref_len)
                    {
                        cp = ref_s + refp;
                        rem = len;
                    }
                    else
                    {
                        // part of the segment lies outside the held reference window: those positions read as 'N'
                        for (int i = 0; i < len; ++i)
                        {
                            const uint32_t e = ent[i];
                            const int p = refp + i;
                            const uint32_t c = (p >= 0 && p < ref_len) ? ref_s[p] : 0u;
                            lnp = __dadd_rn(lnp, lds_f64((e & 0xfff0u) | ((e & c) ? 8u : 0u)));
                        }
                        ent += len;
                    }
                    refp += len;
                }
                else if (kind == SX_SEG_INSERT)
                {
                    cp = insp;
                    insp += len;
                    rem = len;
                }
                else if (kind == SX_SEG_REFSKIP)
                {
                    refp += len;
                }
                else if (kind == SX_SEG_SOFTCLIP)
                {
                    lnp = __dadd_rn(lnp, __dmul_rn(static_cast<double>(static_cast<unsigned>(len)), softclip));
                    ent += len;
                }
                else if (kind != SX_SEG_HARDCLIP)
                {
                    atomicOr(status, SX_ST_SEG_KIND);
                }
            }
            if (done) break;
            // One uniform chunk of K1_CHUNK read bases.  Lanes whose segment ends inside the chunk substitute the all-zero table row
            // for the surplus steps (x + 0.0 == x exactly for every x this sum can hold), so all lanes run the same straight-line
            // code and a warp diverges only in the short segment fetch above.  Surplus loads stay inside the CTA's shared memory
            // (the entry array carries slack; ref/ins/seq areas follow each other).
            {
                const int n = rem < K1_CHUNK ? rem : K1_CHUNK;
#pragma unroll
                for (int k = 0; k < K1_CHUNK; ++k)
                {
                    const uint32_t e = (k < n) ? static_cast<uint32_t>(ent[k]) : zero_entry;
                    const uint32_t c = cp[k];
                    lnp = __dadd_rn(lnp, lds_f64((e & 0xfff0u) | ((e & c) ? 8u : 0u)));
                }
                ent += n;
                cp += n;
                rem -= n;
            }
        }
        lnp_out[r0.aln_begin + a] = lnp;
    }
}

// max shared-memory footprint over regions [begin, end) (device-resident batches: the region table is not on the host)
// out[0]: general kernel, out[1]: fast path (k1_score4.cu)
__global__ void k1_smem_need_kernel(const sx_region* __restrict__ regions, uint32_t begin, uint32_t end, uint32_t* __restrict__ out, uint32_t fmt)
{
    uint32_t m = 0, mq = 0;
    for (uint32_t i = begin + blockIdx.x * blockDim.x + threadIdx.x; i < end; i += gridDim.x * blockDim.x)
    {
        const sx_region a = regions[i], b = regions[i + 1];
        m = max(m, k1_make_layout(a, b, fmt).total);
        mq = max(mq, k1q::make_layout(a, b, fmt).total);
    }
    for (int d = 16; d; d >>= 1)
    {
        m = max(m, __shfl_xor_sync(0xffffffffu, m, d));
        mq = max(mq, __shfl_xor_sync(0xffffffffu, mq, d));
    }
    if ((threadIdx.x & 31) == 0 && m)
    {
        atomicMax(out, m);
        atomicMax(out + 1, mq);
    }
}

// per-read max over its alignments (first max in batch order), one thread per read; alignments are sorted by read
// the same for sx_aln8 headers (read indices relative to the region): find the read's region, then its alignments inside the region
__global__ void k1_read_max8_kernel(const sx_region* __restrict__ regions, uint32_t n_regions, const sx_aln8* __restrict__ alns, uint32_t n_reads,
                                    const double* __restrict__ lnp, double* __restrict__ max_lnp, uint32_t* __restrict__ max_aln)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    uint32_t lo = 0, hi = n_regions; // last region with read_begin <= r (regions without reads share a read_begin: take the last)
    while (lo + 1 < hi)
    {
        const uint32_t mid = (lo + hi) >> 1;
        if (regions[mid].read_begin <= r) lo = mid;
        else hi = mid;
    }
    const uint32_t a0 = regions[lo].aln_begin, a1 = regions[lo + 1].aln_begin, rel = r - regions[lo].read_begin;
    uint32_t l2 = a0, h2 = a1;
    while (l2 < h2)
    {
        const uint32_t mid = (l2 + h2) >> 1;
        if (alns[mid].read < rel) l2 = mid + 1;
        else h2 = mid;
    }
    double best = 0;
    uint32_t besta = 0xffffffffu;
    for (uint32_t a = l2; a < a1 && alns[a].read == rel; ++a)
    {
        const double v = lnp[a];
        if (besta == 0xffffffffu || v > best)
        {
            best = v;
            besta = a;
        }
    }
    max_lnp[r] = best;
    max_aln[r] = besta;
}

__global__ void k1_read_max_kernel(const sx_aln* __restrict__ alns, uint32_t n_alns, uint32_t n_reads, const double* __restrict__ lnp,
                                   double* __restrict__ max_lnp, uint32_t* __restrict__ max_aln)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n_reads) return;
    // lower bound of r in alns[].read
    uint32_t lo = 0, hi = n_alns;
    while (lo < hi)
    {
        const uint32_t mid = (lo + hi) >> 1;
        if (alns[mid].read < r) lo = mid + 1;
        else hi = mid;
    }
    double best = 0;
    uint32_t besta = 0xffffffffu;
    for (uint32_t a = lo; a < n_alns && alns[a].read == r; ++a)
    {
        const double v = lnp[a];
        if (besta == 0xffffffffu || v > best)
        {
            best = v;
            besta = a;
        }
    }
    max_lnp[r] = best;
    max_aln[r] = besta;
}

int k1_smem_need_dev(sx_ctx* ctx, const sx_region* regions_dev, uint32_t begin, uint32_t end, uint32_t need[2], uint32_t fmt)
{
    uint32_t* d = nullptr;
    int rc = sx_take(ctx, SX_SLOT_K1_SMEM_NEED, 2, d, 0);
    if (rc) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(d, 0, 2 * sizeof(uint32_t), ctx->s_compute));
    const uint32_t n = end - begin;
    const int blocks = static_cast<int>(std::min<uint32_t>((n + 255) / 256, 1184));
    k1_smem_need_kernel<<<blocks, 256, 0, ctx->s_compute>>>(regions_dev, begin, end, d, fmt);
    SX_CUDA(ctx, cudaMemcpyAsync(need, d, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->s_compute));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    return SX_OK;
}
} // namespace

size_t sx_k1_region_smem(const sx_region* r0, const sx_region* r1, const sx_aln*)
{
    return k1_make_layout(*r0, *r1, 0).total;
}

// smem_bytes: largest region footprint of the general kernel; smem_fast: of the 4-bit fast path (0: not computed)
int sx_k1_launch(sx_ctx* ctx, const sx_align_batch* d, uint32_t region_begin, uint32_t region_end, double* lnp_dev, size_t smem_bytes, size_t smem_fast, cudaStream_t st)
{
    if (region_end <= region_begin) return SX_OK;
    if ((d->qual_bits == 4 || d->qual_bits == 2) && smem_fast && smem_fast <= k1q::KQ_MAX_SMEM) return sx_k1q_launch(ctx, d, region_begin, region_end, lnp_dev, smem_fast, st);
    if (smem_bytes > ctx->smem_optin)
        return sx_fail(ctx, SX_ERR_ARG, "sx_score_alignments: a region needs %zu bytes of shared memory (limit %zu); split it into smaller regions", smem_bytes,
                       ctx->smem_optin);
    // the opt-in is a property of (function, device), so it is set per launch like the other kernels' (cheap: a driver-side attribute write)
    if (smem_bytes > 48 * 1024)
        SX_CUDA(ctx, cudaFuncSetAttribute(k1_score_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ctx->smem_optin)));
    uint4 qd;
    memcpy(&qd, d->qual_dict, 16);
    k1_score_kernel<<<region_end - region_begin, K1_THREADS, smem_bytes, st>>>(d->regions, d->read_len, d->seq4, d->qual, d->ref, d->alns, d->segs, d->ins,
                                                                              ctx->d_tables, region_begin, lnp_dev, ctx->d_status, static_cast<uint32_t>(smem_bytes), d->qual_bits == 4 ? 4u : d->qual_bits == 2 ? 2u : 8u, qd, d->format, d->exc_off, d->exc);
    SX_CUDA(ctx, cudaGetLastError());
    return SX_OK;
}

// ------------------------------------------------------------------------------------------------------------------
// entry points
// ------------------------------------------------------------------------------------------------------------------
extern "C" uint64_t sx_align_batch_cells(const sx_align_batch* b)
{
    uint64_t n = 0;
    for (uint32_t i = 0; i < b->n_segs; ++i)
    {
        uint32_t kind, len;
        if (b->format & SX_FMT_SEG2)
        {
            const uint32_t v = reinterpret_cast<const sx_aln_seg2*>(b->segs)[i];
            kind = (v >> 12) & 7u;
            len = v & 0xfffu;
        }
        else
        {
            kind = b->segs[i].kind;
            len = b->segs[i].len;
        }
        if (kind == SX_SEG_MATCH || kind == SX_SEG_INSERT) n += len;
    }
    return n;
}

static int validate_host_batch(sx_ctx* ctx, const sx_align_batch* b, size_t* max_smem, size_t* max_smem_fast)
{
    if (!b || !b->regions || !b->alns || (b->n_reads && !b->read_len)) return sx_fail(ctx, SX_ERR_ARG, "sx_score_alignments: NULL batch array");
    if (b->format & SX_FMT_BASEQ)
    {
        if (b->qual_bits != 2 || !b->exc_off || (b->exc_off[b->n_regions] && !b->exc))
            return sx_fail(ctx, SX_ERR_ARG, "sx_score_alignments: SX_FMT_BASEQ needs qual_bits == 2 and the exception arrays");
        for (int i = 0; i < 4; ++i)
            if (b->qual_dict[i] > SX_MAX_QSCORE)
                return sx_fail(ctx, SX_ERR_RANGE, "sx_score_alignments: SX_FMT_BASEQ dictionary quality %d above %d (send such batches with a quality pool)", b->qual_dict[i], SX_MAX_QSCORE);
    }
    size_t m = 0, mq = 0;
    for (uint32_t i = 0; i < b->n_regions; ++i)
    {
        const sx_region& r = b->regions[i];
        const sx_region& n = b->regions[i + 1];
        if ((r.seq_off | ((b->format & SX_FMT_BASEQ) ? 0u : r.qual_off) | r.ref_off | r.ins_begin) & 15u || (r.seg_begin & ((b->format & SX_FMT_SEG2) ? 7u : 3u)))
            return sx_fail(ctx, SX_ERR_ALIGNMENT, "sx_score_alignments: region %u violates the 16-byte staging rule (seq_off %llu qual_off %llu ref_off %llu ins_begin %u seg_begin %u)", i,
                           (unsigned long long)r.seq_off, (unsigned long long)r.qual_off, (unsigned long long)r.ref_off, r.ins_begin, r.seg_begin);
        if (n.read_begin < r.read_begin || n.aln_begin < r.aln_begin || n.seg_begin < r.seg_begin || n.ins_begin < r.ins_begin || n.seq_off < r.seq_off ||
            n.qual_off < r.qual_off)
            return sx_fail(ctx, SX_ERR_ARG, "sx_score_alignments: region table is not monotone at region %u", i);
        m = std::max<size_t>(m, k1_make_layout(r, n, b->format).total);
        mq = std::max<size_t>(mq, k1q::make_layout(r, n, b->format).total);
    }
    if (b->n_regions)
    {
        const sx_region& e = b->regions[b->n_regions];
        if (e.read_begin != b->n_reads || e.aln_begin != b->n_alns) return sx_fail(ctx, SX_ERR_ARG, "sx_score_alignments: sentinel region does not close the batch");
    }
    *max_smem = m;
    *max_smem_fast = mq;
    return SX_OK;
}

extern "C" int sx_score_alignments_dev(sx_ctx* ctx, const sx_align_batch* d, double* lnp_out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!d || !lnp_out_dev) return sx_fail(ctx, SX_ERR_ARG, "sx_score_alignments_dev: NULL argument");
    if (d->n_regions == 0) return SX_OK;
    const int rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k1_run(ctx, d, lnp_out_dev, launches); });
    if (rc) return rc;
    return sx_check_status(ctx, "sx_score_alignments");
}

extern "C" int sx_read_max_dev(sx_ctx* ctx, const sx_align_batch* d, const double* lnp_dev, double* max_lnp_dev, uint32_t* max_aln_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!d || !lnp_dev || !max_lnp_dev || !max_aln_dev) return sx_fail(ctx, SX_ERR_ARG, "sx_read_max_dev: NULL argument");
    if (d->n_reads == 0) return SX_OK;
    return sx_run_timed(ctx, [&](unsigned* launches) { return sx_k1_read_max_run(ctx, d, lnp_dev, max_lnp_dev, max_aln_dev, launches); });
}

// Host-buffer entry: the batch is cut into chunks of whole regions; chunk k+1's H2D copies overlap chunk k's kernel and chunk
// k-1's D2H (three streams, events).  Device pools keep the HOST offsets (a chunk is copied to the same byte offsets it has on
// the host), so nothing is re-based.
extern "C" int sx_score_alignments(sx_ctx* ctx, const sx_align_batch* b, double* lnp_out)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!b || !lnp_out) return sx_fail(ctx, SX_ERR_ARG, "sx_score_alignments: NULL argument");
    if (b->n_regions == 0 || b->n_alns == 0) return SX_OK;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    size_t smem = 0, smem_fast = 0;
    int rc = validate_host_batch(ctx, b, &smem, &smem_fast);
    if (rc) return rc;

    sx_align_batch d = *b;
    const size_t reg_bytes = (size_t)(b->n_regions + 1) * sizeof(sx_region);
    const size_t aln_sz = (b->format & SX_FMT_ALN8) ? sizeof(sx_aln8) : sizeof(sx_aln), seg_sz = (b->format & SX_FMT_SEG2) ? sizeof(sx_aln_seg2) : sizeof(sx_aln_seg);
    const size_t aln_bytes = (size_t)(b->n_alns + 1) * aln_sz + 16; // + slack: an sx_aln8 slice is staged from a 16-byte boundary
    const size_t seg_bytes = (size_t)b->n_segs * seg_sz + SX_POOL_SLACK;
    void *alns = nullptr, *segs = nullptr;
    if ((rc = sx_take(ctx, sx_host_slot(0), (size_t)b->n_regions + 1, d.regions, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(1), b->n_reads, d.read_len, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(2), b->seq4_bytes, d.seq4, SX_POOL_SLACK))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(3), b->qual_bytes, d.qual, SX_POOL_SLACK))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(4), b->ref_bytes, d.ref, SX_POOL_SLACK))) return rc;
    if ((rc = sx_ensure(ctx, sx_host_slot(5), aln_bytes, &alns))) return rc; // (sx_aln or sx_aln8 entries)
    if ((rc = sx_ensure(ctx, sx_host_slot(6), seg_bytes, &segs))) return rc;
    d.alns = static_cast<const sx_aln*>(alns);
    d.segs = static_cast<const sx_aln_seg*>(segs);
    if ((rc = sx_take(ctx, sx_host_slot(7), b->ins_bytes, d.ins, SX_POOL_SLACK))) return rc;
    if (b->format & SX_FMT_BASEQ)
    {
        if ((rc = sx_take(ctx, sx_host_slot(24), (size_t)b->n_regions + 1, d.exc_off, 0))) return rc;
        if ((rc = sx_take(ctx, sx_host_slot(25), b->exc_off[b->n_regions], d.exc, 16))) return rc;
    }
    double* d_out = nullptr;
    if ((rc = sx_take(ctx, sx_host_slot(8), b->n_alns, d_out, 0))) return rc;

    int chunks = ctx->params.pipeline_chunks;
    if (chunks <= 0)
    {
        // ~128 MB of input per chunk: small enough that the first kernel starts early, large enough to keep copies at link rate
        const uint64_t in_bytes = b->seq4_bytes + b->qual_bytes + aln_bytes + seg_bytes + b->ins_bytes;
        chunks = static_cast<int>(std::min<uint64_t>(64, std::max<uint64_t>(1, in_bytes >> 27)));
    }
    chunks = std::max(1, std::min<int>(chunks, (int)b->n_regions));
    while (ctx->ev_pool.size() < (size_t)chunks * 2)
    {
        cudaEvent_t ev;
        SX_CUDA(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        ctx->ev_pool.push_back(ev);
    }
    cudaEvent_t t0, t1;
    t0 = ctx->ev_a;
    t1 = ctx->ev_b;
    SX_CUDA(ctx, cudaEventRecord(t0, ctx->s_h2d));
    // the small tables go first, whole
    SX_CUDA(ctx, cudaMemcpyAsync(const_cast<sx_region*>(d.regions), b->regions, reg_bytes, cudaMemcpyHostToDevice, ctx->s_h2d));
    SX_CUDA(ctx, cudaMemcpyAsync(const_cast<uint16_t*>(d.read_len), b->read_len, (size_t)b->n_reads * 2, cudaMemcpyHostToDevice, ctx->s_h2d));
    SX_CUDA(ctx, cudaMemcpyAsync(const_cast<char*>(d.ref), b->ref, b->ref_bytes, cudaMemcpyHostToDevice, ctx->s_h2d));
    if (b->format & SX_FMT_BASEQ)
    {
        SX_CUDA(ctx, cudaMemcpyAsync(const_cast<uint32_t*>(d.exc_off), b->exc_off, (size_t)(b->n_regions + 1) * 4, cudaMemcpyHostToDevice, ctx->s_h2d));
        if (b->exc_off[b->n_regions])
            SX_CUDA(ctx, cudaMemcpyAsync(const_cast<uint32_t*>(d.exc), b->exc, (size_t)b->exc_off[b->n_regions] * 4, cudaMemcpyHostToDevice, ctx->s_h2d));
    }
    for (int c = 0; c < chunks; ++c)
    {
        const uint32_t ra = (uint32_t)((uint64_t)b->n_regions * c / chunks);
        const uint32_t rb = (uint32_t)((uint64_t)b->n_regions * (c + 1) / chunks);
        const sx_region& A = b->regions[ra];
        const sx_region& B = b->regions[rb];
        auto cp = [&](const void* hbase, const void* dbase, size_t lo, size_t hi) -> cudaError_t {
            if (hi <= lo) return cudaSuccess;
            return cudaMemcpyAsync((char*)const_cast<void*>(dbase) + lo, (const char*)hbase + lo, hi - lo, cudaMemcpyHostToDevice, ctx->s_h2d);
        };
        SX_CUDA(ctx, cp(b->seq4, d.seq4, A.seq_off, B.seq_off));
        if (!(b->format & SX_FMT_BASEQ)) SX_CUDA(ctx, cp(b->qual, d.qual, A.qual_off, B.qual_off));
        SX_CUDA(ctx, cp(b->alns, d.alns, (size_t)A.aln_begin * aln_sz, (size_t)(B.aln_begin + 1) * aln_sz));
        SX_CUDA(ctx, cp(b->segs, d.segs, (size_t)A.seg_begin * seg_sz, (size_t)B.seg_begin * seg_sz));
        SX_CUDA(ctx, cp(b->ins, d.ins, A.ins_begin, B.ins_begin));
        SX_CUDA(ctx, cudaEventRecord(ctx->ev_pool[2 * c], ctx->s_h2d));
        SX_CUDA(ctx, cudaStreamWaitEvent(ctx->s_compute, ctx->ev_pool[2 * c], 0));
        if ((rc = sx_k1_launch(ctx, &d, ra, rb, d_out, smem, smem_fast, ctx->s_compute))) return rc;
        SX_CUDA(ctx, cudaEventRecord(ctx->ev_pool[2 * c + 1], ctx->s_compute));
        SX_CUDA(ctx, cudaStreamWaitEvent(ctx->s_d2h, ctx->ev_pool[2 * c + 1], 0));
        if (B.aln_begin > A.aln_begin)
            SX_CUDA(ctx, cudaMemcpyAsync(lnp_out + A.aln_begin, d_out + A.aln_begin, (size_t)(B.aln_begin - A.aln_begin) * sizeof(double), cudaMemcpyDeviceToHost,
                                         ctx->s_d2h));
    }
    SX_CUDA(ctx, cudaEventRecord(t1, ctx->s_d2h));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_d2h));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    float ms = 0;
    cudaEventElapsedTime(&ms, t0, t1);
    ctx->timing.kernel_ms = ms; // whole pipelined call (copies + kernels), see sx_timing
    ctx->timing.launches = chunks;
    ctx->total_launches += chunks;
    return sx_check_status(ctx, "sx_score_alignments");
}

// K1's launcher: one 8-byte round trip picks the shared-memory tile, the kernel is only enqueued
int sx_k1_run(sx_ctx* ctx, const sx_align_batch* d, double* lnp_dev, unsigned* launches)
{
    if (d->n_regions == 0) return SX_OK;
    uint32_t need[2] = {0, 0};
    int rc = k1_smem_need_dev(ctx, d->regions, 0, d->n_regions, need, d->format);
    if (rc) return rc;
    rc = sx_k1_launch(ctx, d, 0, d->n_regions, lnp_dev, need[0], need[1], ctx->s_compute);
    *launches += 2;
    return rc;
}

// the per-read maximum of K1's scores (one launch)
int sx_k1_read_max_run(sx_ctx* ctx, const sx_align_batch* d, const double* lnp_dev, double* max_lnp_dev, uint32_t* max_aln_dev, unsigned* launches)
{
    if (d->format & SX_FMT_ALN8)
        k1_read_max8_kernel<<<(d->n_reads + 255) / 256, 256, 0, ctx->s_compute>>>(d->regions, d->n_regions, reinterpret_cast<const sx_aln8*>(d->alns), d->n_reads, lnp_dev,
                                                                                  max_lnp_dev, max_aln_dev);
    else
        k1_read_max_kernel<<<(d->n_reads + 255) / 256, 256, 0, ctx->s_compute>>>(d->alns, d->n_alns, d->n_reads, lnp_dev, max_lnp_dev, max_aln_dev);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}
