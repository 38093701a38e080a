// k4_read.cuh -- the per-read preamble of pileup_read_segment and the base-code look-ups, shared by K4 (k4_pileup.cu) and its metrics
// pass (k4m_metrics.cu).  The functions are __host__ __device__, so g++ compiles them too (tests/cpp/k4m_core_host.cpp).
#pragma once

#include "strelka_b200.h"

#include <cstdint>

#ifdef __CUDACC__
#define K4_HD __host__ __device__ __forceinline__
#else
#define K4_HD inline
#endif

// the bam_seq code of base i of a read packed two bases a byte, high nibble first
K4_HD uint32_t code_at(const uint8_t* seq, uint32_t i) { return (seq[i >> 1] >> ((~i & 1u) << 2)) & 15u; }

// bam_seq code -> base_call id (0..3 ACGT, 4 for '=' / 'N', 5 = bam_seq_code_to_id would throw) and -> bam_seq::get_char, as nibble /
// byte look-ups in 64-bit literals: a branch per base value makes the compiler duplicate the whole loop body per branch
K4_HD uint32_t id_of_code(uint32_t c) { return static_cast<uint32_t>(0x4555555355525104ull >> (4u * c)) & 15u; }
K4_HD char char_of_code(uint32_t c)
{
    // codes 0..7: '=', 'A', 'C', 'N', 'G', 'N', 'N', 'N'; codes 8..15: 'T', 'N' x 7
    const unsigned long long lut = c < 8u ? 0x4e4e4e474e43413dull : 0x4e4e4e4e4e4e4e54ull;
    return static_cast<char>((lut >> (8u * (c & 7u))) & 0xffu);
}

K4_HD uint32_t lower_bound_key(const uint32_t* keys, uint32_t n, uint32_t key)
{
    uint32_t lo = 0, hi = n;
    while (lo < hi)
    {
        const uint32_t mid = (lo + hi) >> 1;
        if (keys[mid] < key) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// the per-read preamble of pileup_read_segment (:1175-1233): the report-range test, getReadAmbiguousEndLength and minDistanceFromReadEdge.
// false = the read contributes nothing; else [read_begin, read_end) are the read offsets it piles up.
struct read_window
{
    uint32_t read_begin, read_end, ref_span;
};
template <typename CodeFn>
K4_HD bool k4_trim_read(const sx_pileup_opts& opt, int32_t report_begin, int32_t report_end, const sx_pileup_read& rd, uint32_t ref_span, CodeFn code,
                        read_window& w)
{
    if (rd.pos >= report_end) return false;
    if (static_cast<int64_t>(rd.pos) + ref_span <= report_begin) return false;
    const uint32_t read_size = rd.len;
    uint32_t ambig = 0; // getReadAmbiguousEndLength: the run of 'N' (code 15) at the 3' end of the read as sequenced
    if (rd.flags & SX_PRF_FWD)
    {
        uint32_t e = read_size;
        while (e > 0 && code(e - 1) == 15u) --e;
        ambig = read_size - e;
    }
    else
    {
        while (ambig < read_size && code(ambig) == 15u) ++ambig;
    }
    w.read_begin = 0;
    w.read_end = read_size;
    if (ambig > 0)
    {
        if (rd.flags & SX_PRF_FWD) w.read_end -= ambig;
        else w.read_begin += ambig;
    }
    if (opt.minDistanceFromReadEdge > 0)
    {
        w.read_begin += opt.minDistanceFromReadEdge;
        if (opt.minDistanceFromReadEdge <= w.read_end) w.read_end -= opt.minDistanceFromReadEdge;
        else w.read_end = 0;
        if (w.read_end <= w.read_begin) return false;
    }
    w.ref_span = ref_span;
    return true;
}
