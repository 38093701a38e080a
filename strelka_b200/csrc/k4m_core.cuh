// k4m_core.cuh -- the body of K4m (pile-up scoring metrics, k4m_metrics.cu) that g++ also compiles (tests/cpp/k4m_core_host.cpp): the
// observation word of one visited base, and the per-site statistics built from a site's words.
//
// The statistics are order-free, so the words of a site may come in any order:
//   MapqTracker            count, zeroCount and sumSquare are integer sums (sumSquare < 2^53: exact in the reference's double)
//   fastRanksum::get_z_stat  the rank weight of a value is (#smaller) + (#equal + 1) / 2, a half-integer, so 2 R1 and 2 R2 are integer sums;
//                          mean, var and the z-score are then the reference's own expressions on the same exact operands
//   getExpectedCategory2Value, MeanTracker::mean   an exact integer sum divided once
//   median (math_util.hh:54-62)   the element at index size/2 of the sorted values: an order statistic
// so every output has the reference's bits without replaying its insertion order.
#pragma once

#include "k4_read.cuh"

#include <cmath>
#include <cstdint>

// One visited base (a matched base inside [read_begin, read_end) and the report range, of a read without SX_PRF_SKIP), 64 bits:
//   bits  0.. 7  mapq (raw: MapqTracker and mq_ranksum)       bits 24..35  align_strand_read_pos (cycle: germline readPositionRankSum)
//   bits  8..15  qscore (after the MAPQ adjustment K4 applies)  bits 36..47  read_pos (un-flipped: somatic readPositionRankSum, alt list)
//   bit  16      is_ref (ref_char == id_to_base(call_id))      bits 48..59  read_size (alt list)
//   bit  17      sub-mapped read
//   bit  18      somatic-eligible: tier-1 read, current_call_filter false (SX_PM_SOMATIC only)
//   bits 19..23  min(20, distance from the edge of the full read) (SX_PM_GERMLINE only)
// Read lengths are at most K4M_MAX_READ (< 4096), so the 12-bit fields hold every position.
#define K4M_MAX_READ 1024u

struct k4m_obs
{
    uint32_t mapq, qscore, is_ref, submapped, somatic, edge, cycle, read_pos, read_size;
};

K4_HD uint64_t k4m_pack(const k4m_obs& o)
{
    return static_cast<uint64_t>(o.mapq & 0xffu) | (static_cast<uint64_t>(o.qscore & 0xffu) << 8) | (static_cast<uint64_t>(o.is_ref & 1u) << 16) |
           (static_cast<uint64_t>(o.submapped & 1u) << 17) | (static_cast<uint64_t>(o.somatic & 1u) << 18) | (static_cast<uint64_t>(o.edge & 31u) << 19) |
           (static_cast<uint64_t>(o.cycle & 0xfffu) << 24) | (static_cast<uint64_t>(o.read_pos & 0xfffu) << 36) |
           (static_cast<uint64_t>(o.read_size & 0xfffu) << 48);
}
K4_HD uint32_t k4m_mapq(uint64_t w) { return static_cast<uint32_t>(w) & 0xffu; }
K4_HD uint32_t k4m_qscore(uint64_t w) { return static_cast<uint32_t>(w >> 8) & 0xffu; }
K4_HD bool k4m_is_ref(uint64_t w) { return (w >> 16) & 1u; }
K4_HD bool k4m_submapped(uint64_t w) { return (w >> 17) & 1u; }
K4_HD bool k4m_somatic(uint64_t w) { return (w >> 18) & 1u; }
K4_HD uint32_t k4m_edge(uint64_t w) { return static_cast<uint32_t>(w >> 19) & 31u; }
K4_HD uint32_t k4m_cycle(uint64_t w) { return static_cast<uint32_t>(w >> 24) & 0xfffu; }
K4_HD uint32_t k4m_read_pos(uint64_t w) { return static_cast<uint32_t>(w >> 36) & 0xfffu; }
K4_HD uint32_t k4m_read_size(uint64_t w) { return static_cast<uint32_t>(w >> 48) & 0xfffu; }

// id_to_base (blt_util/seq_util.hh): 0..3 -> ACGT, 4 -> 'N'
K4_HD char k4m_base_of_id(uint32_t id) { return static_cast<char>((0x4e54474341ull >> (8u * id)) & 0xffu); }

// the zero-indexed distance of read base p from the edge of the full read (:1351-1353), capped at 20 (pos_basecall_buffer.cpp:65-66); the
// reference's unsigned arithmetic, wrap included
K4_HD uint32_t k4m_edge_distance(uint32_t p, uint32_t full_off, uint32_t full_size)
{
    const uint32_t fp = p + full_off, d0 = full_size - (fp + 1u), d = fp < d0 ? fp : d0;
    return d < 20u ? d : 20u;
}

// fastRanksum of one site in closed form: 2 R1, 2 R2 (R = the category's rank sum), N1, N2 and the sum of the category-2 values
struct k4m_rank
{
    uint64_t r1x2, r2x2, n1, n2, sum2;
};

// fastRanksum::get_z_stat + getMannWhitneyZScore (fastRanksum.cpp).  n1 * (n1 + n2 + 1) is an int product there: where it would overflow
// the reference's value is undefined, so *overflow is set and 0 returned.
K4_HD double k4m_z_stat(const k4m_rank& k, bool* overflow)
{
    const double R1 = static_cast<double>(k.r1x2) * 0.5, R2 = static_cast<double>(k.r2x2) * 0.5; // (half-integers below 2^52: exact)
    const bool swap = R1 > R2;
    const int64_t n1 = static_cast<int64_t>(swap ? k.n2 : k.n1), n2 = static_cast<int64_t>(swap ? k.n1 : k.n2);
    const double w1 = swap ? R2 : R1;
    const int64_t prod = n1 * (n1 + n2 + 1);
    if (prod > 2147483647ll || n1 + n2 > 2147483647ll)
    {
        *overflow = true;
        return 0.0;
    }
    const double mean = static_cast<double>(static_cast<int32_t>(prod)) / 2.0;
    const double var = std::sqrt(static_cast<double>(static_cast<int32_t>(n2)) * mean / 6.0);
    if (std::fabs(var) < 0.0001) return 0.0;
    return (w1 - mean) / var;
}

// fastRanksum::getExpectedCategory2Value
K4_HD double k4m_expected2(const k4m_rank& k) { return k.n2 == 0 ? 0.0 : static_cast<double>(k.sum2) / static_cast<double>(static_cast<uint32_t>(k.n2)); }

// MeanTracker::mean
K4_HD double k4m_mean(uint64_t total, uint32_t count) { return count == 0 ? 0.0 : static_cast<double>(total) / static_cast<double>(count); }

// MapqTracker's sumSquare as the reference holds it
K4_HD double k4m_sum_sq(uint64_t s) { return static_cast<double>(s); }

// ---------------------------------------------------------------------------------------------------------------------------------------
// the per-site statistics on one thread (the CPU build; the kernel computes the same sums across a warp)
// ---------------------------------------------------------------------------------------------------------------------------------------
#ifndef __CUDACC__
#include <algorithm>
#include <vector>

// the ranks of val(w) over the words with sel(w), category 1 = is_ref
template <class Sel, class Val> inline k4m_rank k4m_rank_scalar(const uint64_t* w, uint32_t n, Sel sel, Val val)
{
    std::vector<uint64_t> h1(4096, 0), h2(4096, 0);
    for (uint32_t i = 0; i < n; ++i)
        if (sel(w[i])) (k4m_is_ref(w[i]) ? h1 : h2)[val(w[i])]++;
    k4m_rank k = {0, 0, 0, 0, 0};
    uint64_t before = 0;
    for (uint32_t v = 0; v < 4096; ++v)
    {
        const uint64_t t = h1[v] + h2[v], wx2 = 2 * before + t + 1;
        k.r1x2 += h1[v] * wx2;
        k.r2x2 += h2[v] * wx2;
        k.n1 += h1[v];
        k.n2 += h2[v];
        k.sum2 += static_cast<uint64_t>(v) * h2[v];
        before += t;
    }
    return k;
}

inline void k4m_site_scalar(const uint64_t* w, uint32_t n, uint32_t mode, sx_pileup_metrics_rec* o)
{
    *o = sx_pileup_metrics_rec{};
    uint64_t sq = 0;
    uint32_t zero = 0;
    for (uint32_t i = 0; i < n; ++i)
    {
        const uint32_t m = k4m_mapq(w[i]);
        sq += m * m;
        zero += m == 0;
    }
    o->mapq_count = n;
    o->mapq_zero = zero;
    o->mapq_sum_sq = k4m_sum_sq(sq);
    bool ov = false;
    if (mode == SX_PM_GERMLINE)
    {
        const auto all = [](uint64_t) { return true; };
        const auto mapped = [](uint64_t x) { return !k4m_submapped(x); };
        ov = false;
        o->mq_ranksum = k4m_z_stat(k4m_rank_scalar(w, n, all, k4m_mapq), &ov);
        if (ov) o->status |= SX_PM_ST_MQ_OVERFLOW;
        const k4m_rank bq = k4m_rank_scalar(w, n, mapped, k4m_qscore);
        ov = false;
        o->baseq_ranksum = k4m_z_stat(bq, &ov);
        if (ov) o->status |= SX_PM_ST_BASEQ_OVERFLOW;
        o->raw_baseq = k4m_expected2(bq);
        const k4m_rank rp = k4m_rank_scalar(w, n, mapped, k4m_cycle);
        ov = false;
        o->read_pos_ranksum = k4m_z_stat(rp, &ov);
        if (ov) o->status |= SX_PM_ST_READ_POS_OVERFLOW;
        o->raw_pos = k4m_expected2(rp);
        uint64_t et = 0;
        uint32_t ec = 0;
        for (uint32_t i = 0; i < n; ++i)
            if (!k4m_submapped(w[i]) && !k4m_is_ref(w[i]))
            {
                et += k4m_edge(w[i]);
                ++ec;
            }
        o->mean_edge_distance = k4m_mean(et, ec);
    }
    else if (mode == SX_PM_SOMATIC)
    {
        const auto eligible = [](uint64_t x) { return k4m_somatic(x); };
        o->read_pos_ranksum = k4m_z_stat(k4m_rank_scalar(w, n, eligible, k4m_read_pos), &ov);
        if (ov) o->status |= SX_PM_ST_READ_POS_OVERFLOW;
        std::vector<uint32_t> p, c;
        for (uint32_t i = 0; i < n; ++i)
            if (k4m_somatic(w[i]) && !k4m_is_ref(w[i]))
            {
                p.push_back(k4m_read_pos(w[i]));
                c.push_back(k4m_read_size(w[i]) - k4m_read_pos(w[i]));
            }
        o->n_alt_read_pos = static_cast<uint32_t>(p.size());
        if (!p.empty())
        {
            std::sort(p.begin(), p.end());
            std::sort(c.begin(), c.end());
            const uint32_t pm = p[p.size() / 2], lm = c[c.size() / 2];
            o->median_read_pos = static_cast<uint16_t>(std::min(pm, lm));
            if (p.size() >= 3)
            {
                for (uint32_t& x : p) x = x > pm ? x - pm : pm - x;
                std::sort(p.begin(), p.end());
                o->median_read_pos_var = static_cast<uint16_t>(p[p.size() / 2]);
            }
        }
    }
}
#endif
