// k4m_metrics.cu -- K4m pileup_metrics: the per-position MAPQ tallies and scoring-metric accumulators of pileup_read_segment
// (starling_pos_processor_base.cpp:1345-1362) read out as the callers read them (include/strelka_b200.h, K4m).
//
// A separate pass over K4's bases (K4's fill is left as it is):
//   1. k4m_count_kernel (thread per read): the visited bases of every matched segment as +1 over a site range of a difference array.
//   2. sx_scan: differences -> per-site counts -> offsets.  One 4-byte round trip sizes the word buffer.
//   3. k4m_walk_kernel (warp per read): the read's trimming (k4_read.cuh, K4's own preamble), MAPQ adjustment and -- SX_PM_SOMATIC, tier1
//      reads -- mismatch-density map, then one 64-bit observation word per visited base (k4m_core.cuh), placed in its site's slots by an
//      atomic cursor.  The order within a site is arbitrary; every statistic below is order-free.
//   4. k4m_reduce_kernel (warp per site): the site's words, staged in shared memory when they fit the tile and read in place otherwise,
//      reduced by 256-bin histograms in shared memory: the tallies by warp sums, each rank sum in closed form from the histogram's prefix
//      sums, the medians as order statistics by a histogram search.
#include "k4m_core.cuh"
#include "sx_internal.h"

#include <algorithm>

namespace
{
constexpr unsigned FULL = 0xffffffffu;
constexpr uint32_t K4M_MAX_SEGS = 64;
constexpr uint32_t K4M_WALK_WARPS = 4;
constexpr uint32_t K4M_RED_WARPS = 4;
constexpr uint32_t K4M_TILE = 512; // words a warp stages in shared memory; deeper sites are reduced from global memory
constexpr uint32_t K4M_BINS = 256;

struct k4m_args
{
    const sx_pileup_read* reads;
    const uint8_t* seq4;
    const uint8_t* qual;
    const sx_aln_seg* segs;
    const char* ref;
    const uint32_t* cand_snv;
    const uint16_t* full_len;
    const uint16_t* full_off;
    uint32_t n_reads, n_cand_snv, ref_len, n_sites, mode, qual_bits;
    int32_t ref_begin, report_begin, report_end;
    uint8_t qual_dict[16];
    sx_pileup_opts opt;
};

__device__ __forceinline__ bool seg_ref(uint32_t k) { return k == SX_SEG_MATCH || k == SX_SEG_DELETE || k == SX_SEG_SKIP; }
__device__ __forceinline__ bool seg_read(uint32_t k) { return k == SX_SEG_MATCH || k == SX_SEG_INSERT || k == SX_SEG_SOFTCLIP; }

// the read's path facts (reference span, first / last matched segment) and its trimmed window; false: the read contributes nothing
__device__ __forceinline__ bool read_setup(const k4m_args& A, uint32_t r, sx_pileup_read& rd, uint32_t& as, uint32_t& first, uint32_t& last, read_window& w,
                                           int* status, bool report)
{
    rd = A.reads[r];
    if (rd.flags & SX_PRF_SKIP) return false;
    as = A.reads[r + 1].seg_off - rd.seg_off;
    if (rd.len > K4M_MAX_READ || as > K4M_MAX_SEGS)
    {
        if (report) atomicOr(status, SX_ST_READ_LIMIT);
        return false;
    }
    const sx_aln_seg* path = A.segs + rd.seg_off;
    uint32_t ref_span = 0;
    first = last = as;
    for (uint32_t i = 0; i < as; ++i)
    {
        const uint32_t k = path[i].kind;
        if (report && k > SX_SEG_SKIP) atomicOr(status, SX_ST_SEG_KIND);
        if (seg_ref(k)) ref_span += path[i].len;
        if (k == SX_SEG_MATCH)
        {
            if (first == as) first = i;
            last = i;
        }
    }
    const uint8_t* seq = A.seq4 + rd.seq_off;
    return k4_trim_read(A.opt, A.report_begin, A.report_end, rd, ref_span, [&](uint32_t i) { return code_at(seq, i); }, w);
}

// +1 over sites [a, b) of a difference array with n + 1 entries
__device__ __forceinline__ void diff_add(uint32_t* d, int64_t a, int64_t b)
{
    if (a >= b) return;
    atomicAdd(&d[a], 1u);
    atomicAdd(&d[b], 0xffffffffu);
}

// ---------------------------------------------------------------------------------------------------------------------------------------
// pass 1: the visited bases of each site, as differences
// ---------------------------------------------------------------------------------------------------------------------------------------
__global__ void k4m_count_kernel(k4m_args A, uint32_t* __restrict__ diff, int* __restrict__ status)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < A.n_reads; r += gridDim.x * blockDim.x)
    {
        sx_pileup_read rd;
        uint32_t as, first, last;
        read_window w;
        if (!read_setup(A, r, rd, as, first, last, w, status, true)) continue;
        const sx_aln_seg* path = A.segs + rd.seg_off;
        int64_t ref_head = rd.pos;
        uint32_t read_head = 0;
        for (uint32_t i = 0; i < as; ++i)
        {
            const uint32_t k = path[i].kind, len = path[i].len;
            if (k == SX_SEG_MATCH)
            {
                const uint32_t rb = max(read_head, w.read_begin), re = min(read_head + len, w.read_end);
                if (rb < re)
                {
                    const int64_t p0 = ref_head + (rb - read_head), p1 = p0 + (re - rb);
                    const int64_t a = (p0 > A.report_begin ? p0 : A.report_begin) - A.report_begin;
                    const int64_t b = (p1 < A.report_end ? p1 : A.report_end) - A.report_begin;
                    diff_add(diff, a, b);
                }
            }
            if (seg_read(k)) read_head += len;
            if (seg_ref(k)) ref_head += len;
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------------
// pass 3: one warp per read, one word per visited base
// ---------------------------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(K4M_WALK_WARPS * 32) k4m_walk_kernel(k4m_args A, const uint32_t* __restrict__ site_off, uint32_t* __restrict__ cursor,
                                                                        uint64_t* __restrict__ words, const sx_tables* __restrict__ tables, int* __restrict__ status)
{
    // per warp: the mismatch-density deltas [K4M_MAX_READ + 4] (SX_PM_SOMATIC only)
    __shared__ int delta_all[K4M_WALK_WARPS][K4M_MAX_READ + 4];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int* delta = delta_all[warp];
    const uint32_t fs = A.opt.mismatchDensityFilterFlankSize, fs2 = fs * 2;
    const bool isDensity = fs > 0;
    for (uint32_t r = blockIdx.x * K4M_WALK_WARPS + warp; r < A.n_reads; r += gridDim.x * K4M_WALK_WARPS)
    {
        sx_pileup_read rd;
        uint32_t as, first, last;
        read_window w;
        if (!read_setup(A, r, rd, as, first, last, w, status, false)) continue; // (uniform across the warp)
        const sx_aln_seg* path = A.segs + rd.seg_off;
        const uint8_t* seq = A.seq4 + rd.seq_off;
        const uint8_t* ql = A.qual + rd.qual_off;
        const uint32_t read_size = rd.len;
        const bool submapped = !(rd.flags & SX_PRF_TIER1OR2), tier1 = rd.flags & SX_PRF_TIER1, fwd = rd.flags & SX_PRF_FWD;
        const uint32_t adjustedMapq = max(5u, (uint32_t)rd.mapq);
        const bool is_mapq_adjust = A.opt.isBasecallQualAdjustedForMapq && adjustedMapq <= 80u;
        const uint8_t* mqrow = tables->mappedq[min(adjustedMapq, 90u)];
        const uint32_t full_off = A.full_off ? A.full_off[r] : 0u, full_size = A.full_len ? A.full_len[r] : read_size;
        const auto ref_char = [&](int64_t pos) -> char {
            const int64_t i = pos - A.ref_begin;
            return i >= 0 && i < static_cast<int64_t>(A.ref_len) ? A.ref[i] : 'N';
        };
        // create_mismatch_filter_map (starling_read_util.cpp:120-217) where the somatic filter needs it: a tier1, non-sub-mapped read
        const bool density = A.mode == SX_PM_SOMATIC && tier1 && !submapped && isDensity;
        const uint32_t delta_size = max(1u + fs2, read_size) - fs2;
        if (density)
        {
            for (uint32_t i = lane; i < delta_size; i += 32) delta[i] = 0;
            __syncwarp();
            auto inc = [&](uint32_t start_pos, uint32_t length) {
                atomicAdd(&delta[max(fs2, start_pos) - fs2], 1);
                if (start_pos + length < delta_size) atomicAdd(&delta[start_pos + length], -1);
            };
            int64_t ref_head = rd.pos;
            uint32_t read_head = 0;
            for (uint32_t i = 0; i < as; ++i)
            {
                const uint32_t k = path[i].kind, len = path[i].len;
                const bool edge = (i < first) || (i > last);
                if (k == SX_SEG_INSERT && !edge && lane == 0) inc(read_head, len);
                else if (k == SX_SEG_DELETE && !edge && lane == 0) inc(read_head, 0);
                else if (k == SX_SEG_SKIP && lane == 0) atomicOr(status, SX_ST_SEG_KIND); // "Can't handle cigar code"
                else if (k == SX_SEG_MATCH)
                {
                    const uint32_t p_lo = max(read_head, w.read_begin), p_hi = min(read_head + len, w.read_end);
                    for (uint32_t p = p_lo + lane; p < p_hi; p += 32)
                    {
                        const int64_t pos = ref_head + (p - read_head);
                        const uint32_t code = code_at(seq, p);
                        if (char_of_code(code) == ref_char(pos)) continue;
                        // CandidateSnvBuffer::isCandidateSnvAnySample
                        bool cand = false;
                        const uint32_t id = id_of_code(code);
                        const int64_t rel = pos - A.report_begin;
                        if (id < 4 && rel >= 0 && rel < (1 << 30))
                        {
                            const uint32_t key = (static_cast<uint32_t>(rel) << 2) | id;
                            const uint32_t l = lower_bound_key(A.cand_snv, A.n_cand_snv, key);
                            cand = l < A.n_cand_snv && A.cand_snv[l] == key;
                        }
                        if (!cand) inc(p, 1);
                    }
                }
                if (seg_read(k)) read_head += len;
                if (seg_ref(k)) ref_head += len;
            }
            __syncwarp();
            int carry = 0; // ddata::total
            for (uint32_t b = 0; b < delta_size; b += 32)
            {
                const uint32_t i = b + lane;
                int v = i < delta_size ? delta[i] : 0;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1)
                {
                    const int y = __shfl_up_sync(FULL, v, d);
                    if (lane >= (uint32_t)d) v += y;
                }
                v += carry;
                if (i < delta_size) delta[i] = v;
                carry = __shfl_sync(FULL, v, 31);
            }
            __syncwarp();
        }
        unsigned long long qd_lo, qd_hi;
        memcpy(&qd_lo, A.qual_dict, 8);
        memcpy(&qd_hi, A.qual_dict + 8, 8);
        const int max_pass = static_cast<int>(A.opt.mismatchDensityFilterMaxMismatchCount);
        int64_t ref_head = rd.pos;
        uint32_t read_head = 0;
        for (uint32_t i = 0; i < as; ++i)
        {
            const uint32_t k = path[i].kind, len = path[i].len;
            if (k == SX_SEG_MATCH)
            {
                const uint32_t p_lo = max(read_head, w.read_begin), p_hi = min(read_head + len, w.read_end);
                for (uint32_t p = p_lo + lane; p < p_hi; p += 32)
                {
                    const int64_t pos = ref_head + (p - read_head);
                    if (pos < A.report_begin || pos >= A.report_end) continue; // is_pos_reportable
                    const uint32_t s = static_cast<uint32_t>(pos - A.report_begin);
                    const uint32_t call_code = code_at(seq, p), call_id = id_of_code(call_code);
                    if (call_id > 4u)
                    {
                        atomicOr(status, SX_ST_BASE);
                        continue;
                    }
                    uint32_t qscore;
                    if (A.qual_bits == 4)
                    {
                        const uint32_t c = (ql[p >> 1] >> ((~p & 1u) << 2)) & 15u;
                        qscore = static_cast<uint32_t>((c < 8u ? qd_lo : qd_hi) >> (8u * (c & 7u))) & 0xffu;
                    }
                    else qscore = ql[p];
                    if (is_mapq_adjust)
                    {
                        if (qscore > SX_MAX_QSCORE)
                        {
                            atomicOr(status, SX_ST_QUAL);
                            continue;
                        }
                        qscore = mqrow[qscore];
                    }
                    k4m_obs o;
                    o.mapq = rd.mapq;
                    o.qscore = qscore;
                    o.is_ref = ref_char(pos) == k4m_base_of_id(call_id);
                    o.submapped = submapped;
                    o.somatic = 0;
                    if (A.mode == SX_PM_SOMATIC && tier1 && !submapped)
                    {
                        bool is_call_filter = (call_code == 15u) || (static_cast<int>(qscore) < A.opt.minBasecallErrorPhredProb);
                        if (!is_call_filter && density) is_call_filter = max_pass < delta[min(delta_size - 1, max(fs, p) - fs)];
                        o.somatic = !is_call_filter;
                    }
                    o.edge = A.mode == SX_PM_GERMLINE ? k4m_edge_distance(p, full_off, full_size) : 0u;
                    o.cycle = fwd ? p : read_size - (p + 1);
                    o.read_pos = p;
                    o.read_size = read_size;
                    words[site_off[s] + atomicAdd(&cursor[s], 1u)] = k4m_pack(o);
                }
            }
            if (seg_read(k)) read_head += len;
            if (seg_ref(k)) ref_head += len;
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------------------------------------------
// pass 4: one warp per site
// ---------------------------------------------------------------------------------------------------------------------------------------
template <typename T> __device__ __forceinline__ T warp_sum(T v)
{
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL, v, d);
    return v;
}
__device__ __forceinline__ uint32_t warp_max(uint32_t v)
{
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v = max(v, __shfl_xor_sync(FULL, v, d));
    return v;
}
__device__ __forceinline__ uint32_t warp_excl(uint32_t v, uint32_t& total)
{
    const uint32_t lane = threadIdx.x & 31;
    uint32_t x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1)
    {
        const uint32_t y = __shfl_up_sync(FULL, x, d);
        if (lane >= (uint32_t)d) x += y;
    }
    total = __shfl_sync(FULL, x, 31);
    return x - v;
}

// the histograms of val(w) over the words with sel(w), values [base, base + 256): h1 (is_ref) and h2 (or h1 alone with one category)
template <class Sel, class Val>
__device__ __forceinline__ void hist_chunk(const uint64_t* w, uint32_t n, uint32_t base, Sel sel, Val val, bool by_ref, uint32_t* h1, uint32_t* h2)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t i = lane; i < K4M_BINS; i += 32) h1[i] = h2[i] = 0;
    __syncwarp();
    for (uint32_t i = lane; i < n; i += 32)
    {
        const uint64_t x = w[i];
        if (!sel(x)) continue;
        const uint32_t v = val(x);
        if (v < base || v >= base + K4M_BINS) continue;
        atomicAdd(&((by_ref && !k4m_is_ref(x)) ? h2 : h1)[v - base], 1u);
    }
    __syncwarp();
}

// fastRanksum over val(w) (< 4096) of the words with sel(w), category 1 = is_ref, in closed form (k4m_core.cuh)
template <class Sel, class Val> __device__ k4m_rank warp_rank(const uint64_t* w, uint32_t n, Sel sel, Val val, uint32_t* h1, uint32_t* h2)
{
    const uint32_t lane = threadIdx.x & 31;
    uint32_t vmax = 0;
    for (uint32_t i = lane; i < n; i += 32)
        if (sel(w[i])) vmax = max(vmax, val(w[i]) + 1u);
    vmax = warp_max(vmax);
    unsigned long long r1 = 0, r2 = 0, n1 = 0, n2 = 0, s2 = 0;
    uint32_t carry = 0;
    for (uint32_t base = 0; base < vmax; base += K4M_BINS)
    {
        hist_chunk(w, n, base, sel, val, true, h1, h2);
        // lane holds bins [8 lane, 8 lane + 8)
        uint32_t t = 0;
        for (uint32_t j = 0; j < 8; ++j) t += h1[8 * lane + j] + h2[8 * lane + j];
        uint32_t chunk;
        unsigned long long before = carry + warp_excl(t, chunk);
        for (uint32_t j = 0; j < 8; ++j)
        {
            const unsigned long long c1 = h1[8 * lane + j], c2 = h2[8 * lane + j], wx2 = 2 * before + c1 + c2 + 1;
            r1 += c1 * wx2;
            r2 += c2 * wx2;
            n1 += c1;
            n2 += c2;
            s2 += (base + 8 * lane + j) * c2;
            before += c1 + c2;
        }
        carry += chunk;
        __syncwarp();
    }
    k4m_rank k;
    k.r1x2 = warp_sum(r1);
    k.r2x2 = warp_sum(r2);
    k.n1 = warp_sum(n1);
    k.n2 = warp_sum(n2);
    k.sum2 = warp_sum(s2);
    return k;
}

// the k-th smallest (0-based) of val(w) (< 4096) over the words with sel(w): a histogram search chunk by chunk
template <class Sel, class Val> __device__ uint32_t warp_kth(const uint64_t* w, uint32_t n, uint32_t k, Sel sel, Val val, uint32_t* h)
{
    const uint32_t lane = threadIdx.x & 31;
    for (uint32_t base = 0; base < 4096; base += K4M_BINS)
    {
        hist_chunk(w, n, base, sel, val, false, h, h + K4M_BINS);
        uint32_t t = 0;
        for (uint32_t j = 0; j < 8; ++j) t += h[8 * lane + j];
        uint32_t chunk;
        uint32_t before = warp_excl(t, chunk);
        if (k < chunk)
        {
            uint32_t found = 0xffffffffu;
            if (k >= before && k < before + t)
                for (uint32_t j = 0; j < 8; ++j)
                {
                    before += h[8 * lane + j];
                    if (k < before)
                    {
                        found = base + 8 * lane + j;
                        break;
                    }
                }
            const uint32_t m = __ballot_sync(FULL, found != 0xffffffffu);
            const uint32_t v = __shfl_sync(FULL, found, __ffs(m) - 1);
            __syncwarp();
            return v;
        }
        k -= chunk;
        __syncwarp();
    }
    return 0; // (unreachable: k < the number of selected words)
}

__global__ void __launch_bounds__(K4M_RED_WARPS * 32) k4m_reduce_kernel(uint32_t n_sites, uint32_t mode, const uint32_t* __restrict__ site_off,
                                                                          const uint64_t* __restrict__ words, sx_pileup_metrics_rec* __restrict__ out)
{
    __shared__ uint64_t tile_all[K4M_RED_WARPS][K4M_TILE];
    __shared__ uint32_t hist_all[K4M_RED_WARPS][2 * K4M_BINS];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* h1 = hist_all[warp];
    uint32_t* h2 = h1 + K4M_BINS;
    for (uint32_t s = blockIdx.x * K4M_RED_WARPS + warp; s < n_sites; s += gridDim.x * K4M_RED_WARPS)
    {
        const uint32_t o0 = site_off[s], n = site_off[s + 1] - o0;
        const uint64_t* w = words + o0;
        if (n <= K4M_TILE)
        {
            for (uint32_t i = lane; i < n; i += 32) tile_all[warp][i] = w[i];
            __syncwarp();
            w = tile_all[warp];
        }
        sx_pileup_metrics_rec rec;
        memset(&rec, 0, sizeof(rec));
        unsigned long long sq = 0;
        uint32_t zero = 0;
        for (uint32_t i = lane; i < n; i += 32)
        {
            const uint32_t m = k4m_mapq(w[i]);
            sq += m * m;
            zero += m == 0;
        }
        rec.mapq_count = n;
        rec.mapq_zero = warp_sum(zero);
        rec.mapq_sum_sq = k4m_sum_sq(warp_sum(sq));
        bool ov = false;
        if (mode == SX_PM_GERMLINE)
        {
            const auto all = [](uint64_t) { return true; };
            const auto mapped = [](uint64_t x) { return !k4m_submapped(x); };
            rec.mq_ranksum = k4m_z_stat(warp_rank(w, n, all, [](uint64_t x) { return k4m_mapq(x); }, h1, h2), &ov);
            if (ov) rec.status |= SX_PM_ST_MQ_OVERFLOW;
            const k4m_rank bq = warp_rank(w, n, mapped, [](uint64_t x) { return k4m_qscore(x); }, h1, h2);
            ov = false;
            rec.baseq_ranksum = k4m_z_stat(bq, &ov);
            if (ov) rec.status |= SX_PM_ST_BASEQ_OVERFLOW;
            rec.raw_baseq = k4m_expected2(bq);
            const k4m_rank rp = warp_rank(w, n, mapped, [](uint64_t x) { return k4m_cycle(x); }, h1, h2);
            ov = false;
            rec.read_pos_ranksum = k4m_z_stat(rp, &ov);
            if (ov) rec.status |= SX_PM_ST_READ_POS_OVERFLOW;
            rec.raw_pos = k4m_expected2(rp);
            unsigned long long et = 0;
            uint32_t ec = 0;
            for (uint32_t i = lane; i < n; i += 32)
                if (!k4m_submapped(w[i]) && !k4m_is_ref(w[i]))
                {
                    et += k4m_edge(w[i]);
                    ++ec;
                }
            rec.mean_edge_distance = k4m_mean(warp_sum(et), warp_sum(ec));
        }
        else if (mode == SX_PM_SOMATIC)
        {
            const auto eligible = [](uint64_t x) { return k4m_somatic(x); };
            const auto alt = [](uint64_t x) { return k4m_somatic(x) && !k4m_is_ref(x); };
            rec.read_pos_ranksum = k4m_z_stat(warp_rank(w, n, eligible, [](uint64_t x) { return k4m_read_pos(x); }, h1, h2), &ov);
            if (ov) rec.status |= SX_PM_ST_READ_POS_OVERFLOW;
            uint32_t na = 0;
            for (uint32_t i = lane; i < n; i += 32) na += alt(w[i]);
            na = warp_sum(na);
            rec.n_alt_read_pos = na;
            if (na)
            {
                const uint32_t pm = warp_kth(w, n, na / 2, alt, [](uint64_t x) { return k4m_read_pos(x); }, h1);
                const uint32_t lm = warp_kth(w, n, na / 2, alt, [](uint64_t x) { return k4m_read_size(x) - k4m_read_pos(x); }, h1);
                rec.median_read_pos = static_cast<uint16_t>(min(pm, lm));
                if (na >= 3)
                    rec.median_read_pos_var = static_cast<uint16_t>(warp_kth(
                        w, n, na / 2, alt, [pm](uint64_t x) { const uint32_t p = k4m_read_pos(x); return p > pm ? p - pm : pm - p; }, h1));
            }
        }
        if (lane == 0) out[s] = rec;
        __syncwarp();
    }
}

bool pm_mode_ok(uint32_t m) { return m == SX_PM_MAPQ || m == SX_PM_GERMLINE || m == SX_PM_SOMATIC; }
} // namespace

// K4m's launcher: count, two scans, one 4-byte round trip (the word total), walk, reduce
int sx_k4m_run(sx_ctx* ctx, const sx_pileup_reads_batch* d, const sx_pileup_metrics_opts* o, sx_pileup_metrics_rec* out, unsigned* launches_out)
{
    if (!pm_mode_ok(o->mode)) return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_metrics: mode %u is not SX_PM_MAPQ, SX_PM_GERMLINE or SX_PM_SOMATIC", o->mode);
    if (d->qual_bits != 0 && d->qual_bits != 8 && d->qual_bits != 4) return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_metrics: qual_bits must be 0, 8 or 4");
    const uint32_t n_sites = static_cast<uint32_t>(d->report_end - d->report_begin);
    cudaStream_t st = ctx->s_compute;
    k4m_args A;
    memset(&A, 0, sizeof(A));
    A.reads = d->reads;
    A.seq4 = d->seq4;
    A.qual = d->qual;
    A.segs = d->segs;
    A.ref = d->ref;
    A.cand_snv = d->cand_snv;
    A.full_len = o->full_len;
    A.full_off = o->full_off;
    A.n_reads = d->n_reads;
    A.n_cand_snv = d->n_cand_snv;
    A.ref_len = d->ref_len;
    A.n_sites = n_sites;
    A.mode = o->mode;
    A.qual_bits = d->qual_bits;
    A.ref_begin = d->ref_begin;
    A.report_begin = d->report_begin;
    A.report_end = d->report_end;
    memcpy(A.qual_dict, d->qual_dict, 16);
    A.opt = d->opts;
    uint32_t *off = nullptr, *cursor = nullptr;
    int rc;
    if ((rc = sx_take(ctx, SX_SLOT_K4M_OFF, (size_t)n_sites + 1, off, 64))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K4M_CURSOR, (size_t)n_sites + 1, cursor, 64))) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(off, 0, ((size_t)n_sites + 1) * 4, st));
    SX_CUDA(ctx, cudaMemsetAsync(cursor, 0, ((size_t)n_sites + 1) * 4, st));
    unsigned launches = 0;
    const int cap_grid = ctx->sm_count * 16;
    if (d->n_reads)
    {
        k4m_count_kernel<<<std::max(1, std::min<int>((int)((d->n_reads + 127) / 128), cap_grid)), 128, 0, st>>>(A, off, ctx->d_status);
        SX_CUDA(ctx, cudaGetLastError());
        ++launches;
    }
    const sx_scan_set counts = {1, {{off, n_sites + 1, 0, nullptr}}};
    if ((rc = sx_scan(ctx, SX_SLOT_K4M_SUMS, counts, &launches))) return rc;
    const sx_scan_set offsets = {1, {{off, n_sites + 1, SX_SCAN_EXCLUSIVE, nullptr}}};
    if ((rc = sx_scan(ctx, SX_SLOT_K4M_SUMS, offsets, &launches))) return rc;
    uint32_t total = 0;
    SX_CUDA(ctx, cudaMemcpyAsync(&total, off + n_sites, 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    uint64_t* words = nullptr;
    if ((rc = sx_take(ctx, SX_SLOT_K4M_WORDS, (size_t)total + 1, words, 64))) return rc;
    if (total)
    {
        const int g = std::max(1, std::min<int>((int)((d->n_reads + K4M_WALK_WARPS - 1) / K4M_WALK_WARPS), cap_grid));
        k4m_walk_kernel<<<g, K4M_WALK_WARPS * 32, 0, st>>>(A, off, cursor, words, ctx->d_tables, ctx->d_status);
        SX_CUDA(ctx, cudaGetLastError());
        ++launches;
    }
    if (n_sites)
    {
        const int g = std::max(1, std::min<int>((int)((n_sites + K4M_RED_WARPS - 1) / K4M_RED_WARPS), cap_grid));
        k4m_reduce_kernel<<<g, K4M_RED_WARPS * 32, 0, st>>>(n_sites, o->mode, off, words, out);
        SX_CUDA(ctx, cudaGetLastError());
        ++launches;
    }
    *launches_out += launches;
    return SX_OK;
}

extern "C" int sx_pileup_metrics_dev(sx_ctx* ctx, const sx_pileup_reads_batch* d, const sx_pileup_metrics_opts* o, sx_pileup_metrics_rec* out)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!d || !o || !out) return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_metrics_dev: NULL argument");
    if (d->report_end < d->report_begin) return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_metrics_dev: empty report range");
    const int rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k4m_run(ctx, d, o, out, launches); });
    if (rc) return rc;
    return sx_check_status(ctx, "sx_pileup_metrics");
}

extern "C" int sx_pileup_metrics(sx_ctx* ctx, const sx_pileup_reads_batch* b, const sx_pileup_metrics_opts* o, sx_pileup_metrics_rec* out)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!b || !o || !out || !b->reads) return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_metrics: NULL argument");
    if (b->report_end < b->report_begin) return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_metrics: empty report range");
    if (!pm_mode_ok(o->mode)) return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_metrics: mode %u is not SX_PM_MAPQ, SX_PM_GERMLINE or SX_PM_SOMATIC", o->mode);
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint32_t n_sites = static_cast<uint32_t>(b->report_end - b->report_begin);
    sx_pileup_reads_batch d = *b;
    sx_pileup_metrics_opts od = *o;
    int rc;
    const sx_pileup_read& end = b->reads[b->n_reads];
    const size_t qual_bytes = end.qual_off;
    if ((rc = sx_upload(ctx, sx_host_slot(0), b->reads, (size_t)(b->n_reads + 1), d.reads, 64))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(1), b->seq4, end.seq_off, d.seq4, 64))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(2), b->qual, qual_bytes, d.qual, 64))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(3), b->segs, b->n_segs, d.segs, 64))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(4), b->ref, b->ref_len, d.ref, 64))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(5), b->cand_snv, b->n_cand_snv, d.cand_snv, 64))) return rc;
    if (o->full_len && (rc = sx_upload(ctx, sx_host_slot(6), o->full_len, b->n_reads, od.full_len, 64))) return rc;
    if (o->full_off && (rc = sx_upload(ctx, sx_host_slot(7), o->full_off, b->n_reads, od.full_off, 64))) return rc;
    sx_pileup_metrics_rec* dout = nullptr;
    if ((rc = sx_take(ctx, sx_host_slot(8), (size_t)n_sites + 1, dout, 64))) return rc;
    sx_call_timer timer(ctx);
    unsigned launches = 0;
    if ((rc = sx_k4m_run(ctx, &d, &od, dout, &launches))) return rc;
    if ((rc = sx_check_status(ctx, "sx_pileup_metrics"))) return rc;
    if ((rc = sx_download(ctx, out, dout, n_sites))) return rc;
    return timer.finish(launches);
}
