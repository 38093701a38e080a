// k1_stage.cuh -- staging one region into shared memory, the first half of both K1 kernels: the general kernel (k1_score.cu) and the
// fast path (k1_score4.cu).  One CTA of THREADS per region; thread 0 pulls every slice of the region (alignment headers, segments,
// reference window, inserted bases, packed bases, qualities) into shared memory with TMA bulk copies (cp.async.bulk ...
// mbarrier::complete_tx) counted on one mbarrier at offset 0.  The slice sizes, both kernels' layouts and the host-side sizing all
// start from slices_of, so a wire-format change (an SX_FMT_* bit, a header width, the 16-byte staging rule) is made here once.
#pragma once

#include "sx_internal.h"

namespace k1
{
constexpr uint32_t THREADS = 128;
// fast path: records and entries carry 16-bit shared-window addresses, and the term table must sit below 0x7f00 (see the kernel):
// regions that need more than this go to the general kernel
constexpr uint32_t KQ_MAX_SMEM = 60u * 1024u;
constexpr uint32_t TAB_BYTES = SX_K1_ROWS * 16;   // general kernel: the host-built term table
constexpr uint32_t KQ_LUT_BYTES = 80;             // fast path: 9 x 8
constexpr uint32_t KQ_TAB_RESERVE = 2048;         // fast path: 4 pages x 16 rows x 2 doubles, placed on a 1 KB boundary of the shared window inside this reserve

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

// bytes of the alignment-header slice as the kernels stage it: wide headers are 16 bytes each (+ the next one, which closes the last
// segment list); sx_aln8 headers are copied from the 16-byte boundary at or below the region's first header
__host__ __device__ __forceinline__ uint32_t aln_slice_bytes(uint32_t aln_begin, uint32_t n_alns, uint32_t fmt)
{
    return (fmt & SX_FMT_ALN8) ? pad16((n_alns + (aln_begin & 1u)) * 8u) : (n_alns + 1) * 16u;
}

// one region's staged slices: counts, byte sizes (multiples of 16), and the shared-memory offset of each, which the kernel's layout sets
struct slices
{
    uint32_t n_reads, n_alns, n_segs;
    uint32_t aln_bytes, seg_bytes, ref_bytes, refp_bytes, ins_bytes, seq_bytes, qual_bytes;
    uint32_t alns, segs, ref, refp, ins, seq, qual;
};

__host__ __device__ __forceinline__ slices slices_of(const sx_region& r0, const sx_region& r1, uint32_t fmt)
{
    slices S{};
    S.n_reads = r1.read_begin - r0.read_begin;
    S.n_alns = r1.aln_begin - r0.aln_begin;
    S.n_segs = r1.seg_begin - r0.seg_begin;
    S.seg_bytes = pad16(S.n_segs * ((fmt & SX_FMT_SEG2) ? 2u : 4u));
    S.ref_bytes = pad16(r0.ref_len);
    S.ins_bytes = pad16(r1.ins_begin - r0.ins_begin);
    S.seq_bytes = pad16(static_cast<uint32_t>(r1.seq_off - r0.seq_off));
    S.qual_bytes = (fmt & SX_FMT_BASEQ) ? 0u : pad16(static_cast<uint32_t>(r1.qual_off - r0.qual_off)); // BASEQ: qualities ride in the base nibbles
    S.refp_bytes = (fmt & SX_FMT_REF4) ? pad16((r0.ref_len + 1u) / 2u) : 0u;                         // REF4: packed window, unpacked into `ref`
    S.aln_bytes = aln_slice_bytes(r0.aln_begin, S.n_alns, fmt);
    return S;
}

// general kernel: the term table, the slices, read lengths, per-read base and packed-byte offsets, nibble descriptors, 16-bit entries
struct layout : slices
{
    uint32_t tab, rlen, boff, soff, desc, ent, total;
};

__host__ __device__ __forceinline__ layout make_layout(const slices& s)
{
    layout L{s};
    uint32_t o = 16; // mbarrier
    L.tab = o;
    o += TAB_BYTES;
    L.alns = o;
    o += L.aln_bytes;
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
    L.desc = o;
    o += 64 + 16; // 16 nibble descriptors + the 16-entry quality dictionary
    L.ent = o;
    // entries: 2 bytes per base, every read padded to an even count; + slack: the uniform chunk loop may load (and discard) up to
    // K1_CHUNK-1 entries past a read (k1_score.cu)
    o += L.seq_bytes * 4u + 32u;
    L.total = o;
    return L;
}

// fast path: the chunk-mask LUT, the entry table, the term-table reserve, the slices with one run record per segment and alignment,
// read lengths, per-read packed-byte offsets, byte entries
struct qlayout : slices
{
    uint32_t lut, e8, tab, recs, rlen, soff, ent, total;
};

__host__ __device__ __forceinline__ qlayout make_qlayout(const slices& s)
{
    qlayout L{s};
    uint32_t o = 16; // mbarrier
    L.lut = o;
    o += KQ_LUT_BYTES;
    L.e8 = o;
    o += 256;
    L.tab = o;
    o += KQ_TAB_RESERVE;
    L.alns = o;
    o += L.aln_bytes;
    L.segs = o;
    o += L.seg_bytes;
    L.recs = o; // one 8-byte record per segment + one END per alignment
    o += pad16((L.n_segs + L.n_alns) * 8u);
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
    L.soff = o;
    o += pad16((L.n_reads + 1) * 4u);
    L.ent = o;
    // one byte per base (two per packed byte) + slack: the chunk loop loads (and masks off) up to 11 bytes past a run
    o += L.seq_bytes * 2u + 32u;
    L.total = o;
    return L;
}

// shared-memory bytes one region needs in each kernel
struct footprint
{
    uint32_t general, fast;
};

__host__ __device__ __forceinline__ footprint footprint_of(const sx_region& r0, const sx_region& r1, uint32_t fmt)
{
    const slices s = slices_of(r0, r1, fmt);
    return {make_layout(s).total, make_qlayout(s).total};
}

// the staged alignment headers and segments, read through the wire format (sx_aln / sx_aln8, sx_aln_seg / sx_aln_seg2).  aln8, seg2 (and
// ref4 below) are the batch's SX_FMT_ALN8, SX_FMT_SEG2 and SX_FMT_REF4 bits, which each kernel decodes once.
struct aln_reader
{
    const unsigned char* alns;
    const unsigned char* segs;
    const sx_region& r0;
    uint32_t n_alns, n_segs;
    bool aln8, seg2;
    uint32_t skew; // the sx_aln8 slice is staged from a 16-byte boundary

    __device__ __forceinline__ aln_reader(const unsigned char* smem, const slices& s, const sx_region& r0_, bool aln8_, bool seg2_)
        : alns(smem + s.alns), segs(smem + s.segs), r0(r0_), n_alns(s.n_alns), n_segs(s.n_segs), aln8(aln8_), seg2(seg2_),
          skew(aln8 ? (r0_.aln_begin & 1u) : 0u)
    {
    }
    // region-relative header of alignment a: x read, y first reference position, z first segment, w first inserted base
    __device__ __forceinline__ uint4 aln_at(uint32_t a) const
    {
        if (aln8)
        {
            const uint2 v = reinterpret_cast<const uint2*>(alns)[a + skew];
            return make_uint4(v.x & 0xffffu, static_cast<uint32_t>(static_cast<int32_t>(v.x) >> 16), v.y & 0xffffu, v.y >> 16);
        }
        const uint4 h = reinterpret_cast<const uint4*>(alns)[a];
        return make_uint4(h.x - r0.read_begin, h.y - static_cast<uint32_t>(r0.ref_begin), h.z - r0.seg_begin, h.w - r0.ins_begin);
    }
    // end of alignment a's segment list
    __device__ __forceinline__ uint32_t seg_end(uint32_t a) const
    {
        if (aln8) return a + 1 < n_alns ? aln_at(a + 1).z : n_segs;
        return reinterpret_cast<const uint4*>(alns)[a + 1].z - r0.seg_begin;
    }
    // segment s as len | kind << 16 | flags << 24
    __device__ __forceinline__ uint32_t seg_at(uint32_t s) const
    {
        if (seg2)
        {
            const uint32_t v = reinterpret_cast<const uint16_t*>(segs)[s];
            return (v & 0xfffu) | (((v >> 12) & 7u) << 16) | ((v >> 15) << 24);
        }
        return reinterpret_cast<const uint32_t*>(segs)[s];
    }
};

// thread 0: initialise the mbarrier at smem[0], expect every byte and issue the bulk copies of the region's slices.  `first` (the
// general kernel's term table) is copied before them.  The caller's __syncthreads publishes the barrier; then mbar_wait(bar, 0).
__device__ __forceinline__ void issue_copies(unsigned char* smem, const slices& s, const sx_region& r0, bool aln8, bool seg2, bool ref4, const sx_aln* alns,
                                             const sx_aln_seg* segs, const char* ref, const char* ins, const uint8_t* seq4, const uint8_t* qual,
                                             uint32_t first_off = 0, const void* first_src = nullptr, uint32_t first_bytes = 0)
{
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem);
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    const uint32_t ref_tx = ref4 ? s.refp_bytes : s.ref_bytes;
    mbar_expect_tx(bar, first_bytes + s.aln_bytes + s.seg_bytes + ref_tx + s.ins_bytes + s.seq_bytes + s.qual_bytes);
    if (first_bytes) tma_bulk_g2s(smem + first_off, first_src, first_bytes, bar);
    tma_bulk_g2s(smem + s.alns, reinterpret_cast<const unsigned char*>(alns) + (aln8 ? (size_t)(r0.aln_begin & ~1u) * 8u : (size_t)r0.aln_begin * 16u), s.aln_bytes, bar);
    if (s.seg_bytes) tma_bulk_g2s(smem + s.segs, reinterpret_cast<const unsigned char*>(segs) + (size_t)r0.seg_begin * (seg2 ? 2u : 4u), s.seg_bytes, bar);
    if (ref_tx) tma_bulk_g2s(smem + (ref4 ? s.refp : s.ref), ref + r0.ref_off, ref_tx, bar);
    if (s.ins_bytes) tma_bulk_g2s(smem + s.ins, ins + r0.ins_begin, s.ins_bytes, bar);
    if (s.seq_bytes) tma_bulk_g2s(smem + s.seq, seq4 + r0.seq_off, s.seq_bytes, bar);
    if (s.qual_bytes) tma_bulk_g2s(smem + s.qual, qual + r0.qual_off, s.qual_bytes, bar);
}
} // namespace k1
