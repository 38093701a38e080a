// sx_read_index.cuh -- the per-read body of the window's read index (sx_read_index.cu): the 'N' count of a read's packed bases from 32-bit
// words, its buffer position, and the region of a read where there is no index.  __host__ __device__: tests/cpp/read_index_host.cpp runs exactly this code on the CPU.
#pragma once

#include "strelka_b200.h"

#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define SXI_HD __host__ __device__ __forceinline__
#else
#define SXI_HD inline
#endif

SXI_HD unsigned sxi_popc(const uint32_t x)
{
#if defined(__CUDA_ARCH__)
    return (unsigned)__popc(x);
#else
    return (unsigned)__builtin_popcount(x);
#endif
}

// nibbles equal to 15 ('N') among the first len of the packed bases at p (two per byte, the high nibble first: bam_seq::get_code).  The
// 32-bit words holding them are read whole -- the pool's slack covers the bytes past the end -- and the bytes outside the read, and the low
// nibble past an odd length, are masked off.
SXI_HD uint32_t sxi_count_n(const uint8_t* p, const uint32_t len)
{
    if (len == 0) return 0;
    const uint32_t packed((len + 1u) / 2u);
    const uintptr_t begin((uintptr_t)p), end(begin + packed);
    uint32_t n(0);
    for (uintptr_t w = begin & ~(uintptr_t)3; w < end; w += 4)
    {
#if defined(__CUDA_ARCH__)
        uint32_t x(*(const uint32_t*)w); // little-endian: byte k of the word is bits 8k .. 8k+7
#else
        const uint8_t* q((const uint8_t*)w);
        uint32_t x((uint32_t)q[0] | ((uint32_t)q[1] << 8) | ((uint32_t)q[2] << 16) | ((uint32_t)q[3] << 24));
#endif
        uint32_t keep(0xFFFFFFFFu);
        if (w < begin) keep &= 0xFFFFFFFFu << (8u * (uint32_t)(begin - w));
        if (w + 4 > end) keep &= 0xFFFFFFFFu >> (8u * (uint32_t)(w + 4 - end));
        if ((len & 1u) && w + 4 >= end) keep &= ~(0xFu << (8u * (uint32_t)(end - 1 - w))); // the low nibble of the last byte is past the read
        x &= keep;
        n += sxi_popc(x & (x >> 1) & (x >> 2) & (x >> 3) & 0x11111111u);
    }
    return n;
}

// the region of read r without an index: reads of a region are consecutive, so a binary search of region_read_off (the stages' own entry
// points, where no window pass built the index and a launch of its own would cost more than the search)
SXI_HD uint32_t sxi_region_of(const uint32_t* region_read_off, const uint32_t n_regions, const uint32_t r)
{
    uint32_t lo(0), hi(n_regions);
    while (lo + 1 < hi)
    {
        const uint32_t mid((lo + hi) / 2);
        if (region_read_off[mid] <= r) lo = mid;
        else hi = mid;
    }
    return lo;
}

// get_alignment_buffer_pos (starling_read_util.cpp:30-35): pos - unalignedPrefixSize
SXI_HD int32_t sxi_buffer_pos(const int32_t pos, const sx_aln_seg* segs, const uint32_t n_segs)
{
    uint32_t lead(0);
    for (uint32_t s = 0; s < n_segs; ++s)
    {
        const unsigned t(segs[s].kind);
        if (!(t == SX_AP_INSERT || t == SX_AP_HARD_CLIP || t == SX_AP_SOFT_CLIP)) break;
        if (t != SX_AP_HARD_CLIP) lead += segs[s].len;
    }
    return pos - (int32_t)lead;
}
