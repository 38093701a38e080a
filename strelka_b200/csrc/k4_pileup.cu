// k4_pileup.cu -- K4 pileup_reads (SURVEY 8f1): per-position base_call columns from reads with their best alignment.
//
// Replaces starling_pos_processor_base::pileup_read_segment (/root/reference/src/c++/lib/starling_common/
// starling_pos_processor_base.cpp:1127-1421) with create_mismatch_filter_map (starling_read_util.cpp:52-217),
// getReadAmbiguousEndLength (htsapi/bam_seq_read_util.cpp:29-54) and the mapq adjustment (blt_util/qscore_cache.cpp:44-47).
//
// What has to be preserved is ORDER: a position's column is a std::vector the reference push_backs into read after read, and K2's
// float sums run over that order.  The reference piles reads up in READ-BUFFER order: by rseg.buffer_pos -- the position of the
// MAPPER's alignment minus its unaligned prefix (starling_read_buffer.cpp:68-78, get_alignment_buffer_pos starling_read_util.cpp:30-35;
// the re-buffering after realignment is compiled out, starling_pos_processor_base.cpp:1034-1070) --, read index within a position,
// while each read contributes through its BEST alignment, whose start a realignment may have moved by up to D = max_pos_shift.  So
// reads arrive sorted by buffer position and the output range is cut into windows of W >= the longest alignment span + D: a read
// buffered in window c can only reach the sites of windows c-1 (its last D), c and c+1.  Three passes:
//   1. k4_count_kernel (thread per read): every covered interval is two atomics on difference arrays (tier1 / tier2 column sizes,
//      the part of each that spills forward into the next window and back into the previous one, spanning deletions, sub-mapped
//      bases).  Integer, order-free.
//   2. scans (k4_scan_*): difference arrays -> counts, counts -> CSR offsets.
//   3. k4_fill_kernel (one WARP per window): walks its reads in order; per read the 32 lanes compute the mismatch-density map
//      (shared-memory delta array + warp scan) and every base's base_call word, and place it at
//      site_off[s] + (calls already placed at s).  The running per-site counters live in shared memory for the 3W sites the window's
//      reads can touch.  A column holds, in this order, the calls of window c-1's reads (forward spill), of window c's own reads and of
//      window c+1's reads (back spill): all reads of an earlier window precede all reads of a later one.  So the cursors start at
//      site_off[s] + spill[s] for the window's own sites, at site_off[s] for the next window's sites and at site_off[s+1] - back[s]
//      for the previous window's.
// Everything is integer/byte work; the only table is qphred_cache::mappedq, built on the host (sx_context.cu).
#include "sx_internal.h"

#include <algorithm>
#include <cstring>

namespace
{
constexpr int K4_WARPS = 4;
constexpr uint32_t K4_MAX_W = 2048;    // window size limit (shared memory: 16 bytes per window site and warp)
constexpr uint32_t K4_MAX_READ = 1024; // read length limit (delta + mismatch arrays)
constexpr uint32_t K4_MAX_SEGS = 64;   // path segments per read
constexpr unsigned FULL = 0xffffffffu;
constexpr int ST_ORDER = 64, ST_BASE = 128, ST_LIMIT = 256, ST_QUAL = 1, ST_KIND = 4;

struct k4_args
{
    const sx_pileup_read* reads;
    const int32_t* bpos; // buffer positions (NULL: reads[].pos)
    uint32_t qual_bits;  // 4: dictionary-coded qualities, two per byte
    uint8_t qual_dict[16];
    const uint8_t* seq4;
    const uint8_t* qual;
    const sx_aln_seg* segs;
    const char* ref;
    const uint32_t* cand_snv;
    uint32_t n_reads, n_cand_snv, ref_len;
    int32_t ref_begin, report_begin, report_end;
    int32_t origin; // position of window 0's first site (= report_begin - W)
    uint32_t W, n_windows, n_sites;
    uint32_t Lcap; // read-length capacity of the per-warp arrays (the batch's longest read, rounded up)
    uint32_t span_max, shift_max; // the caller's max_ref_span and max_pos_shift (the gather plan's read range rests on them: checked per read)
    sx_pileup_opts opt;
};

__device__ __forceinline__ uint32_t code_at(const uint8_t* seq, uint32_t i) { return (seq[i >> 1] >> ((~i & 1u) << 2)) & 15u; }
__device__ __forceinline__ bool kind_ref(uint32_t k) { return k == SX_SEG_MATCH || k == SX_SEG_DELETE || k == SX_SEG_SKIP; }
__device__ __forceinline__ bool kind_read(uint32_t k) { return k == SX_SEG_MATCH || k == SX_SEG_INSERT || k == SX_SEG_SOFTCLIP; }

// bam_seq code -> base_call id (0..3 ACGT, 4 for '=' / 'N', 5 = bam_seq_code_to_id would throw) and -> bam_seq::get_char, as nibble /
// byte look-ups in 64-bit literals: a branch per base value makes the compiler duplicate the whole loop body per branch
__device__ __forceinline__ uint32_t id_of_code(uint32_t c) { return static_cast<uint32_t>(0x4555555355525104ull >> (4u * c)) & 15u; }
__device__ __forceinline__ char char_of_code(uint32_t c)
{
    // codes 0..7: '=', 'A', 'C', 'N', 'G', 'N', 'N', 'N'; codes 8..15: 'T', 'N' x 7
    const unsigned long long lut = c < 8u ? 0x4e4e4e474e43413dull : 0x4e4e4e4e4e4e4e54ull;
    return static_cast<char>((lut >> (8u * (c & 7u))) & 0xffu);
}

__device__ __forceinline__ int32_t bpos_of(const k4_args& A, uint32_t r) { return A.bpos ? A.bpos[r] : A.reads[r].pos; }

__device__ __forceinline__ int64_t i64max(int64_t a, int64_t b) { return a > b ? a : b; }
__device__ __forceinline__ int64_t i64min(int64_t a, int64_t b) { return a < b ? a : b; }

// +1 over sites [a, b) of a difference array with n entries
__device__ __forceinline__ void diff_add(int* d, int64_t a, int64_t b, uint32_t n)
{
    if (a >= b) return;
    atomicAdd(&d[a], 1);
    if (b < static_cast<int64_t>(n)) atomicAdd(&d[b], -1);
}

// the per-read preamble of pileup_read_segment (:1175-1233): false = the read contributes nothing
struct read_window
{
    uint32_t read_begin, read_end, ref_span;
};
template <typename CodeFn> __device__ __forceinline__ bool read_preamble(const k4_args& A, const sx_pileup_read& rd, uint32_t ref_span, CodeFn code, read_window& w)
{
    if (rd.pos >= A.report_end) return false;
    if (static_cast<int64_t>(rd.pos) + ref_span <= A.report_begin) return false;
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
    if (A.opt.minDistanceFromReadEdge > 0)
    {
        w.read_begin += A.opt.minDistanceFromReadEdge;
        if (A.opt.minDistanceFromReadEdge <= w.read_end) w.read_end -= A.opt.minDistanceFromReadEdge;
        else w.read_end = 0;
        if (w.read_end <= w.read_begin) return false;
    }
    w.ref_span = ref_span;
    return true;
}

// ---------------------------------------------------------------------------------------------------------------------
// pass 1: column sizes as difference arrays
// ---------------------------------------------------------------------------------------------------------------------
__global__ void k4_count_kernel(k4_args A, int* __restrict__ d1, int* __restrict__ d2, int* __restrict__ s1, int* __restrict__ s2, int* __restrict__ b1,
                                int* __restrict__ b2, int* __restrict__ dsd, int* __restrict__ dsm, int* __restrict__ status)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= A.n_reads) return;
    const sx_pileup_read rd = A.reads[r];
    const int32_t bp = bpos_of(A, r);
    if (r > 0 && bpos_of(A, r - 1) > bp) atomicOr(status, ST_ORDER);
    if (rd.flags & SX_PRF_SKIP) return;
    const sx_aln_seg* path = A.segs + rd.seg_off;
    const uint32_t as = A.reads[r + 1].seg_off - rd.seg_off;
    if (rd.len > A.Lcap || as > K4_MAX_SEGS)
    {
        atomicOr(status, ST_LIMIT);
        return;
    }
    uint32_t ref_span = 0, first = as, last = as;
    for (uint32_t i = 0; i < as; ++i)
    {
        const uint32_t k = path[i].kind;
        if (kind_ref(k)) ref_span += path[i].len;
        if (k == SX_SEG_MATCH)
        {
            if (first == as) first = i;
            last = i;
        }
        if (k > SX_SEG_SKIP) atomicOr(status, ST_KIND);
    }
    const uint8_t* seq = A.seq4 + rd.seq_off;
    read_window w;
    if (!read_preamble(A, rd, ref_span, [&](uint32_t i) { return code_at(seq, i); }, w)) return;
    if (ref_span > A.W || bp < A.origin)
    {
        atomicOr(status, ST_ORDER);
        return;
    }
    const bool submapped = !(rd.flags & SX_PRF_TIER1OR2), tier1 = rd.flags & SX_PRF_TIER1;
    const uint32_t c = static_cast<uint32_t>(bp - A.origin) / A.W;
    const int64_t this_win_pos = static_cast<int64_t>(A.origin) + static_cast<int64_t>(c) * A.W;
    const int64_t this_win_site = this_win_pos - A.report_begin;       // first site of window c (negative in window 0)
    const int64_t next_win_site = this_win_site + A.W;                 // first site of window c+1
    // the best alignment must stay within the three windows the fill pass holds cursors for (guaranteed by W >= span + max_pos_shift)
    if (static_cast<int64_t>(rd.pos) < this_win_pos - A.W || static_cast<int64_t>(rd.pos) + ref_span > this_win_pos + 2 * static_cast<int64_t>(A.W))
    {
        atomicOr(status, ST_ORDER);
        return;
    }
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
                const int64_t a = i64max(p0, A.report_begin) - A.report_begin, b = i64min(p1, A.report_end) - A.report_begin;
                if (submapped) diff_add(dsm, a, b, A.n_sites);
                else
                {
                    diff_add(tier1 ? d1 : d2, a, b, A.n_sites + 1);
                    diff_add(tier1 ? s1 : s2, i64max(a, next_win_site), b, A.n_sites);
                    diff_add(tier1 ? b1 : b2, a, i64min(b, this_win_site), A.n_sites);
                }
            }
        }
        else if (k == SX_SEG_DELETE)
        {
            const bool edge = (i < first) || (i > last);
            const bool pinned = ((i < first) && (rd.flags & SX_PRF_PIN_FIRST)) || ((i > last) && (rd.flags & SX_PRF_PIN_SECOND));
            if (!edge || pinned)
            {
                const int64_t a = i64max(ref_head, A.report_begin) - A.report_begin, b = i64min(ref_head + len, A.report_end) - A.report_begin;
                diff_add(submapped ? dsm : dsd, a, b, A.n_sites);
            }
        }
        if (kind_read(k)) read_head += len;
        if (kind_ref(k)) ref_head += len;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// pass 2: in-place scans of up to 8 int arrays at once (blockIdx.y picks the array).  Three kernels: tile sums, the scan of the tile
// sums (one CTA per array), tiles again with their offsets.  exclusive[k] selects the flavour.
// ---------------------------------------------------------------------------------------------------------------------
constexpr uint32_t SCAN_TILE = 4096, SCAN_THREADS = 256;
struct scan_job
{
    int* data[8];
    uint32_t n[8];
    int exclusive[8];
};

__device__ __forceinline__ int block_scan_incl(int v, int* warp_sums) // inclusive scan across SCAN_THREADS threads
{
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1)
    {
        const int y = __shfl_up_sync(FULL, v, d);
        if (lane >= (uint32_t)d) v += y;
    }
    if (lane == 31) warp_sums[wid] = v;
    __syncthreads();
    if (wid == 0)
    {
        int s = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1)
        {
            const int y = __shfl_up_sync(FULL, s, d);
            if (lane >= (uint32_t)d) s += y;
        }
        if (lane < SCAN_THREADS / 32) warp_sums[lane] = s;
    }
    __syncthreads();
    if (wid > 0) v += warp_sums[wid - 1];
    return v;
}

__global__ void __launch_bounds__(SCAN_THREADS) k4_scan_tile_sums(scan_job J, int* __restrict__ tile_sums, uint32_t tiles_per_array)
{
    const uint32_t k = blockIdx.y, tile = blockIdx.x;
    const uint32_t base = tile * SCAN_TILE;
    if (base >= J.n[k]) return;
    int s = 0;
    for (uint32_t i = base + threadIdx.x; i < min(base + SCAN_TILE, J.n[k]); i += SCAN_THREADS) s += J.data[k][i];
    __shared__ int ws[SCAN_THREADS / 32];
    const int incl = block_scan_incl(s, ws);
    if (threadIdx.x == SCAN_THREADS - 1) tile_sums[k * tiles_per_array + tile] = incl;
}

__global__ void __launch_bounds__(SCAN_THREADS) k4_scan_of_sums(scan_job J, int* __restrict__ tile_sums, uint32_t tiles_per_array)
{
    const uint32_t k = blockIdx.x;
    const uint32_t nt = (J.n[k] + SCAN_TILE - 1) / SCAN_TILE;
    __shared__ int ws[SCAN_THREADS / 32];
    __shared__ int carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (uint32_t b = 0; b < nt; b += SCAN_THREADS)
    {
        const uint32_t i = b + threadIdx.x;
        const int v = i < nt ? tile_sums[k * tiles_per_array + i] : 0;
        const int incl = block_scan_incl(v, ws);
        const int carry = carry_s;
        if (i < nt) tile_sums[k * tiles_per_array + i] = carry + incl - v; // exclusive prefix of the tile sums
        __syncthreads();
        if (threadIdx.x == SCAN_THREADS - 1) carry_s = carry + incl;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(SCAN_THREADS) k4_scan_tiles(scan_job J, const int* __restrict__ tile_sums, uint32_t tiles_per_array)
{
    const uint32_t k = blockIdx.y, tile = blockIdx.x;
    const uint32_t base = tile * SCAN_TILE, n = J.n[k];
    if (base >= n) return;
    __shared__ int ws[SCAN_THREADS / 32];
    int carry = tile_sums[k * tiles_per_array + tile];
    constexpr uint32_t PER = SCAN_TILE / SCAN_THREADS; // consecutive elements per thread
    int v[PER];
    int s = 0;
    const uint32_t i0 = base + threadIdx.x * PER;
#pragma unroll
    for (uint32_t e = 0; e < PER; ++e)
    {
        v[e] = (i0 + e) < n ? J.data[k][i0 + e] : 0;
        s += v[e];
    }
    const int incl = block_scan_incl(s, ws);
    int run = carry + incl - s;
#pragma unroll
    for (uint32_t e = 0; e < PER; ++e)
    {
        const int out = J.exclusive[k] ? run : run + v[e];
        run += v[e];
        if ((i0 + e) < n) J.data[k][i0 + e] = out;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// pass 3: one warp per window, reads in order
// ---------------------------------------------------------------------------------------------------------------------
__host__ __device__ inline uint32_t k4_warp_smem(uint32_t W, uint32_t Lcap)
{
    // run1[3W], run2[3W] (uint32), delta[Lcap + 4] (int), mism[Lcap] (uint8), segment table 3 x K4_MAX_SEGS uint32, and the staged
    // read: packed bases [Lcap/2 + 16], qualities [Lcap], reference bases under the alignment [W + 16], mappedq row [80]; Lcap % 16 == 0
    return 2u * 3u * W * 4u + (Lcap + 4u) * 4u + Lcap + 3u * K4_MAX_SEGS * 4u + (Lcap / 2u + 16u) + Lcap + (W + 16u) + 80u;
}

__device__ __forceinline__ uint32_t lower_bound_pos(const k4_args& A, int64_t pos)
{
    uint32_t lo = 0, hi = A.n_reads;
    while (lo < hi)
    {
        const uint32_t mid = (lo + hi) >> 1;
        if (bpos_of(A, mid) < pos) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(K4_WARPS * 32) k4_fill_kernel(k4_args A, const uint32_t* __restrict__ site_off, const uint32_t* __restrict__ t2_off,
                                                               const int* __restrict__ spill1, const int* __restrict__ spill2, const int* __restrict__ back1,
                                                               const int* __restrict__ back2, uint16_t* __restrict__ calls,
                                                               uint16_t* __restrict__ t2_calls, const sx_tables* __restrict__ tables, int* __restrict__ status)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t c = blockIdx.x * K4_WARPS + warp;
    if (c >= A.n_windows) return;
    unsigned char* wsm = smem + (size_t)warp * k4_warp_smem(A.W, A.Lcap);
    uint32_t* run1 = reinterpret_cast<uint32_t*>(wsm);
    uint32_t* run2 = run1 + 3 * A.W;
    int* delta = reinterpret_cast<int*>(run2 + 3 * A.W);
    uint8_t* mism = reinterpret_cast<uint8_t*>(delta + A.Lcap + 4);
    uint32_t* seg_kl = reinterpret_cast<uint32_t*>(mism + A.Lcap); // kind << 16 | len
    uint32_t* seg_rd = seg_kl + K4_MAX_SEGS;                            // read offset of the segment
    uint32_t* seg_rf = seg_rd + K4_MAX_SEGS;                            // reference offset (relative to the alignment position)
    uint8_t* seq = reinterpret_cast<uint8_t*>(seg_rf + K4_MAX_SEGS);    // the current read, staged once per read by coalesced loads
    uint8_t* ql = seq + (A.Lcap / 2u + 16u);
    char* refb = reinterpret_cast<char*>(ql + A.Lcap);                  // refb[i] = reference base at rd.pos + i ('N' outside the segment)
    uint8_t* mqrow = reinterpret_cast<uint8_t*>(refb + (A.W + 16u));    // mappedq[adjustedMapq][*]
    uint32_t mqrow_of = 0xffffffffu;

    const int64_t win_pos0 = static_cast<int64_t>(A.origin) + static_cast<int64_t>(c) * A.W;
    const int64_t site0 = win_pos0 - A.W - A.report_begin; // site index of local index 0: the first site of window c-1 (may be negative)
    uint32_t lo = 0, hi = 0;
    if (lane == 0)
    {
        lo = lower_bound_pos(A, win_pos0);
        hi = lower_bound_pos(A, win_pos0 + A.W);
    }
    lo = __shfl_sync(FULL, lo, 0);
    hi = __shfl_sync(FULL, hi, 0);
    if (lo == hi) return;
    // write cursor of every site this window's reads can reach: the start of its column + (own sites only) the calls of window c-1's
    // reads, which all precede this window's reads
    for (uint32_t li = lane; li < 3 * A.W; li += 32)
    {
        const int64_t s = site0 + li;
        const bool in = s >= 0 && s < static_cast<int64_t>(A.n_sites);
        uint32_t c1 = 0, c2 = 0;
        if (in)
        {
            if (li < A.W) // the previous window's sites: after its spill-in and its own reads' calls = before the back spill, which is ours
            {
                c1 = site_off[s + 1] - static_cast<uint32_t>(back1[s]);
                c2 = t2_off[s + 1] - static_cast<uint32_t>(back2[s]);
            }
            else if (li < 2 * A.W) // our own sites: after the calls spilling in from window c-1, whose reads all precede ours
            {
                c1 = site_off[s] + static_cast<uint32_t>(spill1[s]);
                c2 = t2_off[s] + static_cast<uint32_t>(spill2[s]);
            }
            else // the next window's sites: we are first
            {
                c1 = site_off[s];
                c2 = t2_off[s];
            }
        }
        run1[li] = c1;
        run2[li] = c2;
    }
    __syncwarp();
    const bool isDensity = A.opt.mismatchDensityFilterFlankSize > 0;
    const uint32_t fs = A.opt.mismatchDensityFilterFlankSize, fs2 = fs * 2;

    for (uint32_t r = lo; r < hi; ++r)
    {
        const sx_pileup_read rd = A.reads[r];
        if (!(rd.flags & SX_PRF_TIER1OR2) || (rd.flags & SX_PRF_SKIP)) continue; // sub-mapped reads only count (pass 1)
        const uint32_t as = A.reads[r + 1].seg_off - rd.seg_off;
        if (rd.len > A.Lcap || as > K4_MAX_SEGS) continue; // flagged by pass 1
        const sx_aln_seg* path = A.segs + rd.seg_off;
        const uint32_t read_size = rd.len;
        // segment table (lane 0; paths are a handful of segments)
        uint32_t ref_span = 0, first = as, last = as;
        if (lane == 0)
        {
            uint32_t rh = 0, fh = 0;
            for (uint32_t i = 0; i < as; ++i)
            {
                const uint32_t k = path[i].kind, len = path[i].len;
                seg_kl[i] = (k << 16) | len;
                seg_rd[i] = rh;
                seg_rf[i] = fh;
                if (k == SX_SEG_MATCH)
                {
                    if (first == as) first = i;
                    last = i;
                }
                if (kind_read(k)) rh += len;
                if (kind_ref(k)) fh += len;
            }
            ref_span = fh;
        }
        ref_span = __shfl_sync(FULL, ref_span, 0);
        first = __shfl_sync(FULL, first, 0);
        last = __shfl_sync(FULL, last, 0);
        __syncwarp();
        if (ref_span > A.W) continue; // flagged by pass 1
        if (rd.pos >= A.report_end || static_cast<int64_t>(rd.pos) + ref_span <= A.report_begin) continue; // (the preamble's range test, before staging)
        const uint32_t adjustedMapq = max(5u, (uint32_t)rd.mapq);
        {
            // stage the read: every later access is shared memory
            const uint8_t* gs = A.seq4 + rd.seq_off;
            const uint8_t* gq = A.qual + rd.qual_off;
            for (uint32_t i = lane; i < (read_size + 1) / 2; i += 32) seq[i] = gs[i];
            if (A.qual_bits == 4)
                for (uint32_t i = lane; i < read_size; i += 32) ql[i] = A.qual_dict[(gq[i >> 1] >> ((~i & 1u) << 2)) & 15u];
            else
                for (uint32_t i = lane; i < read_size; i += 32) ql[i] = gq[i];
            for (uint32_t i = lane; i < ref_span; i += 32)
            {
                const int64_t ri = static_cast<int64_t>(rd.pos) + i - A.ref_begin;
                refb[i] = (ri >= 0 && ri < static_cast<int64_t>(A.ref_len)) ? A.ref[ri] : 'N';
            }
            if (mqrow_of != adjustedMapq)
            {
                for (uint32_t i = lane; i <= SX_MAX_QSCORE; i += 32) mqrow[i] = tables->mappedq[min(adjustedMapq, 90u)][i];
                mqrow_of = adjustedMapq;
            }
        }
        __syncwarp();
        read_window w;
        if (!read_preamble(A, rd, ref_span, [&](uint32_t i) { return code_at(seq, i); }, w)) continue; // uniform across the warp
        const bool tier1 = rd.flags & SX_PRF_TIER1, fwd = rd.flags & SX_PRF_FWD;
        const bool is_mapq_adjust = A.opt.isBasecallQualAdjustedForMapq && adjustedMapq <= 80u;
        const uint32_t delta_size = max(1u + fs2, read_size) - fs2;

        // Both per-base passes walk the MATCH segments (a warp-uniform loop) and stride the lanes over each segment's trimmed bases:
        // no per-base segment search, and positions stay 32-bit offsets from the alignment start.
        const int32_t pos_rel = static_cast<int32_t>(static_cast<int64_t>(rd.pos) - A.report_begin); // site index of the alignment start
        const int32_t site0_32 = static_cast<int32_t>(site0);

        if (isDensity)
        {
            // create_mismatch_filter_map: ddata deltas, then their running sum
            for (uint32_t i = lane; i < delta_size; i += 32) delta[i] = 0;
            for (uint32_t i = lane; i < read_size; i += 32) mism[i] = 0;
            __syncwarp();
            auto inc = [&](uint32_t start_pos, uint32_t length) {
                atomicAdd(&delta[max(fs2, start_pos) - fs2], 1);
                if (start_pos + length < delta_size) atomicAdd(&delta[start_pos + length], -1);
            };
            for (uint32_t i = lane; i < as; i += 32)
            {
                const uint32_t k = seg_kl[i] >> 16, len = seg_kl[i] & 0xffffu;
                const bool edge = (i < first) || (i > last);
                if (k == SX_SEG_INSERT && !edge) inc(seg_rd[i], len);
                else if (k == SX_SEG_DELETE && !edge) inc(seg_rd[i], 0);
                else if (k == SX_SEG_SKIP) atomicOr(status, ST_KIND); // "Can't handle cigar code" in create_mismatch_filter_map
            }
            for (uint32_t si = 0; si < as; ++si)
            {
                const uint32_t kl = seg_kl[si];
                if ((kl >> 16) != SX_SEG_MATCH) continue;
                const uint32_t sb = seg_rd[si], sf = seg_rf[si];
                const uint32_t p_lo = max(sb, w.read_begin), p_hi = min(sb + (kl & 0xffffu), w.read_end);
            for (uint32_t p = p_lo + lane; p < p_hi; p += 32)
            {
                const uint32_t roff = sf + (p - sb); // reference offset from the alignment start
                const uint32_t code = code_at(seq, p);
                if (char_of_code(code) == refb[roff]) continue;
                // CandidateSnvBuffer::isCandidateSnvAnySample: a registered (position, base) is not counted as a mismatch
                bool cand = false;
                const int id = static_cast<int>(id_of_code(code));
                const int32_t rel = pos_rel + static_cast<int32_t>(roff);
                if (id < 4 && rel >= 0 && rel < (1 << 30))
                {
                    const uint32_t key = (static_cast<uint32_t>(rel) << 2) | static_cast<uint32_t>(id);
                    uint32_t l2 = 0, h2 = A.n_cand_snv;
                    while (l2 < h2)
                    {
                        const uint32_t mid = (l2 + h2) >> 1;
                        if (A.cand_snv[mid] < key) l2 = mid + 1;
                        else h2 = mid;
                    }
                    cand = l2 < A.n_cand_snv && A.cand_snv[l2] == key;
                }
                if (!cand)
                {
                    mism[p] = 1;
                    inc(p, 1);
                }
            }
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

        const int max_pass = static_cast<int>(A.opt.mismatchDensityFilterMaxMismatchCount), max_pass2 = A.opt.tier2MismatchDensityFilterMaxMismatchCount;
        for (uint32_t si = 0; si < as; ++si)
        {
            const uint32_t kl = seg_kl[si];
            if ((kl >> 16) != SX_SEG_MATCH) continue;
            const uint32_t sb = seg_rd[si], sf = seg_rf[si];
            const uint32_t p_lo = max(sb, w.read_begin), p_hi = min(sb + (kl & 0xffffu), w.read_end);
        for (uint32_t p = p_lo + lane; p < p_hi; p += 32)
        {
            const int32_t s = pos_rel + static_cast<int32_t>(sf + (p - sb)); // site index
            if (s < 0 || s >= static_cast<int32_t>(A.n_sites)) continue;       // is_pos_reportable
            const uint32_t call_code = code_at(seq, p);
            const uint32_t call_id = id_of_code(call_code);
            if (call_id > 4u)
            {
                atomicOr(status, ST_BASE);
                continue;
            }
            uint32_t qscore = ql[p];
            if (is_mapq_adjust)
            {
                if (qscore > SX_MAX_QSCORE)
                {
                    atomicOr(status, ST_QUAL);
                    continue;
                }
                qscore = mqrow[qscore];
            }
            bool is_call_filter = (call_code == 15u) || (static_cast<int>(qscore) < A.opt.minBasecallErrorPhredProb);
            bool is_tier2_call_filter = is_call_filter, is_neighbor_mismatch = false;
            if (isDensity)
            {
                const int del = delta[min(delta_size - 1, max(fs, p) - fs)]; // ddata::get
                if (!is_call_filter)
                {
                    is_call_filter = max_pass < del;
                    is_tier2_call_filter = A.opt.useTier2Evidence ? (max_pass2 < del) : is_call_filter;
                }
                is_neighbor_mismatch = (del - static_cast<int>(mism[p])) > 0;
            }
            const bool current_call_filter = tier1 ? is_call_filter : is_tier2_call_filter;
            const bool is_tier_specific_filter = tier1 && is_call_filter && !is_tier2_call_filter;
            const uint16_t bc = static_cast<uint16_t>(min(qscore, 63u) | (call_id << 6) | ((fwd ? 1u : 0u) << 10) | ((is_neighbor_mismatch ? 1u : 0u) << 11) |
                                                      ((current_call_filter ? 1u : 0u) << 12) | ((is_tier_specific_filter ? 1u : 0u) << 13));
            const uint32_t li = static_cast<uint32_t>(s - site0_32); // < 3W: the read is buffered in this window, its alignment within D of that, D + span <= W
            if (tier1) calls[run1[li]++] = bc;
            else t2_calls[run2[li]++] = bc;
        }
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// pass 3, second plan: the fill as two kernels without a serial chain.
//   k4_bases_kernel   THREAD per read, two flat loops over the read's bases (every lane of a warp runs the same loop; the read's own
//                     segment boundaries only move a small per-lane cursor): (1) the mismatch-density map as a prefix-count array in
//                     shared memory (one 16-bit entry per base: the events in a window are a difference of two entries; interior indels
//                     are a short event list), (2) the base_call word of every base of the MATCH segments, written to a per-read row of
//                     a scratch array, four calls per 64-bit store.  Packed bases and qualities arrive a 32-bit word at a time.
//   k4_gather_kernel  WARP per 32 neighbouring sites, a lane per site: the warp walks the reads whose alignment can reach the block, in
//                     read-buffer order -- one 32-byte record per read (its MATCH intervals as (first site, length, first read offset)),
//                     warp-uniform --, a lane the read covers fetches its call from the read's row (neighbouring lanes = neighbouring
//                     bases) and appends it to its column: the write cursor is a register.
// The columns are the same bytes in both plans: a column lists its reads in read-buffer order.
// ---------------------------------------------------------------------------------------------------------------------
constexpr uint32_t K4_REC_IV = 3; // MATCH intervals a record holds; a read with more keeps its path (the gather walks it)
struct __align__(16) k4_rrec // what the gather needs of a read (32 bytes)
{
    int32_t site_lo[K4_REC_IV]; // first site of interval j   | fallback: site of the alignment start, read_begin | read_end << 16, seg_off
    uint16_t len[K4_REC_IV];    // its length
    uint16_t p_lo[K4_REC_IV];   // read offset of its first base
    uint32_t n_iv;              // intervals (0: no call; K4_REC_IV + 1: fallback) | n_seg << 8 | tier1 << 31
};

constexpr int K4B_THREADS = 64;
constexpr uint32_t K4B_MAX_EV = 8; // interior indels kept per thread; a read with more walks its path per base

// a byte array read through its 4-byte-aligned words (device allocations: the base is 256-byte aligned), positions ascending
struct k4_wstream
{
    const uint32_t* w32;
    uint32_t off; // byte offset of the read's first byte from w32
    uint32_t cur; // word index held in w
    uint32_t w;
    __device__ __forceinline__ void init(const uint8_t* p)
    {
        const uintptr_t a = reinterpret_cast<uintptr_t>(p);
        w32 = reinterpret_cast<const uint32_t*>(a & ~static_cast<uintptr_t>(3));
        off = static_cast<uint32_t>(a & 3u);
        cur = 0xffffffffu;
        w = 0;
    }
    __device__ __forceinline__ uint32_t byte_at(uint32_t b)
    {
        const uint32_t ob = off + b, wi = ob >> 2;
        if (wi != cur)
        {
            cur = wi;
            w = __ldg(w32 + wi);
        }
        return (w >> (8u * (ob & 3u))) & 0xffu;
    }
    __device__ __forceinline__ uint32_t nibble_at(uint32_t i) { return (byte_at(i >> 1) >> ((~i & 1u) << 2)) & 15u; }
};

// per-lane cursor over a path while the read offset q runs 0, 1, 2, ...: the segment that holds base q
struct k4_segcur
{
    const sx_aln_seg* path;
    uint32_t as, i;   // segments, next segment to load
    uint32_t seg_end; // read offset one past the current read-consuming segment
    uint32_t kind;    // its kind (SX_SEG_*), 0xff before the first
    uint32_t rf;      // reference offset (from the alignment start) after the segments loaded so far
    int32_t rfd;      // MATCH: reference offset of base q = q + rfd
    __device__ __forceinline__ void init(const sx_aln_seg* p, uint32_t n)
    {
        path = p;
        as = n;
        i = 0;
        seg_end = 0;
        kind = 0xffu;
        rf = 0;
        rfd = 0;
    }
};

__global__ void __launch_bounds__(K4B_THREADS) k4_bases_kernel(k4_args A, k4_rrec* __restrict__ rec, uint16_t* __restrict__ bc, uint32_t Ls,
                                                               const sx_tables* __restrict__ tables, int* __restrict__ status)
{
    extern __shared__ __align__(16) uint16_t k4b_P[]; // per thread Lcap + 2 entries: P[i] = mismatches among bases [0, i)
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= A.n_reads) return;
    uint16_t* P = k4b_P + static_cast<size_t>(threadIdx.x) * (A.Lcap + 2u); // (Lcap % 16 == 0: an odd number of 32-bit words per thread, no bank conflicts)
    const sx_pileup_read rd = A.reads[r];
    const uint32_t as = A.reads[r + 1].seg_off - rd.seg_off;
    const sx_aln_seg* path = A.segs + rd.seg_off;
    k4_rrec out;
#pragma unroll
    for (uint32_t j = 0; j < K4_REC_IV; ++j)
    {
        out.site_lo[j] = 0;
        out.len[j] = 0;
        out.p_lo[j] = 0;
    }
    out.n_iv = 0;
    bool ok = (rd.flags & SX_PRF_TIER1OR2) && !(rd.flags & SX_PRF_SKIP) && rd.len <= A.Lcap && as <= K4_MAX_SEGS; // (sub-mapped reads only count, limits: pass 1)
    uint32_t ref_span = 0, first = as, last = as;
    if (ok)
    {
        for (uint32_t i = 0; i < as; ++i)
        {
            const uint32_t k = path[i].kind;
            if (kind_ref(k)) ref_span += path[i].len;
            if (k == SX_SEG_MATCH)
            {
                if (first == as) first = i;
                last = i;
            }
        }
        if (ref_span > A.W) ok = false; // flagged by pass 1
        // the gather looks for a site's reads among the buffer positions [P - span_max - shift_max, P + shift_max]
        const int64_t sh = static_cast<int64_t>(rd.pos) - bpos_of(A, r);
        if (ref_span > A.span_max || sh > static_cast<int64_t>(A.shift_max) || -sh > static_cast<int64_t>(A.shift_max))
        {
            atomicOr(status, ST_ORDER);
            ok = false;
        }
    }
    const uint8_t* gs = A.seq4 + rd.seq_off;
    read_window w;
    w.read_begin = w.read_end = 0;
    if (ok && !read_preamble(A, rd, ref_span, [&](uint32_t i) { return code_at(gs, i); }, w)) ok = false;
    if (!ok)
    {
        rec[r] = out;
        return;
    }
    const uint32_t read_size = rd.len;
    const uint32_t rb = w.read_begin, re = min(w.read_end, read_size);
    const uint32_t fs = A.opt.mismatchDensityFilterFlankSize, fs2 = fs * 2;
    const bool isDensity = fs > 0;
    const uint32_t delta_size = max(1u + fs2, read_size) - fs2;
    const int32_t site0 = static_cast<int32_t>(static_cast<int64_t>(rd.pos) - A.report_begin);
    const int64_t ref0 = static_cast<int64_t>(rd.pos) - A.ref_begin; // index of the alignment's first reference base in A.ref
    k4_wstream sq;
    k4_segcur sc;
    uint32_t ev[K4B_MAX_EV]; // interior indels: read offset << 16 | length (create_mismatch_filter_map's inc(start, length))
    uint32_t n_ev = 0;
    // the path once: the MATCH intervals for the gather, the interior indels for the density map
    {
        uint32_t p = 0, rf = 0, n_iv = 0;
        for (uint32_t i = 0; i < as; ++i)
        {
            const uint32_t k = path[i].kind, len = path[i].len;
            const bool edge = (i < first) || (i > last);
            if (k == SX_SEG_MATCH)
            {
                const uint32_t a = max(p, rb), e = min(p + len, re);
                if (a < e)
                {
                    // clipped to the reportable sites here: the gather asks for sites [0, n_sites) only
                    int64_t s_lo = static_cast<int64_t>(site0) + rf + (a - p), s_hi = s_lo + (e - a);
                    uint32_t a2 = a;
                    if (s_lo < 0)
                    {
                        a2 += static_cast<uint32_t>(-s_lo);
                        s_lo = 0;
                    }
                    if (s_hi > static_cast<int64_t>(A.n_sites)) s_hi = A.n_sites;
                    if (s_lo < s_hi)
                    {
                        if (n_iv < K4_REC_IV)
                        {
                            out.site_lo[n_iv] = static_cast<int32_t>(s_lo);
                            out.len[n_iv] = static_cast<uint16_t>(s_hi - s_lo);
                            out.p_lo[n_iv] = static_cast<uint16_t>(a2);
                        }
                        ++n_iv;
                    }
                }
            }
            if (isDensity)
            {
                if (!edge && (k == SX_SEG_INSERT || k == SX_SEG_DELETE))
                {
                    if (n_ev < K4B_MAX_EV) ev[n_ev] = (p << 16) | (k == SX_SEG_INSERT ? len : 0u);
                    ++n_ev;
                }
                else if (k == SX_SEG_SKIP) atomicOr(status, ST_KIND); // "Can't handle cigar code" in create_mismatch_filter_map
            }
            if (kind_read(k)) p += len;
            if (kind_ref(k)) rf += len;
        }
        if (n_iv > K4_REC_IV)
        {
            out.site_lo[0] = site0;
            out.site_lo[1] = static_cast<int32_t>(rb | (re << 16));
            out.site_lo[2] = static_cast<int32_t>(rd.seg_off);
            n_iv = K4_REC_IV + 1;
        }
        out.n_iv = n_iv | (as << 8) | ((rd.flags & SX_PRF_TIER1) ? 0x80000000u : 0u);
    }
// advance the cursor to the segment that holds base q (q ascends by one): warp-divergent only at a lane's own segment boundaries
#define K4_SEG_ADVANCE(sc, q)                                                         \
    while ((q) >= (sc).seg_end && (sc).i < (sc).as)                                   \
    {                                                                                 \
        const uint32_t k_ = (sc).path[(sc).i].kind, l_ = (sc).path[(sc).i].len;       \
        ++(sc).i;                                                                     \
        if (kind_read(k_))                                                            \
        {                                                                             \
            (sc).kind = k_;                                                           \
            (sc).rfd = static_cast<int32_t>((sc).rf) - static_cast<int32_t>((sc).seg_end); \
            (sc).seg_end += l_;                                                       \
        }                                                                             \
        if (kind_ref(k_)) (sc).rf += l_;                                              \
    }
    if (isDensity)
    {
        // create_mismatch_filter_map as counts: P[i] = mismatches (not registered candidate SNVs) among the bases before i, over the whole read
        sq.init(gs);
        sc.init(path, as);
        uint32_t c = 0;
        P[0] = 0;
        for (uint32_t q = 0; q < read_size; ++q)
        {
            K4_SEG_ADVANCE(sc, q)
            if (sc.kind == SX_SEG_MATCH && q < sc.seg_end && q >= rb && q < re)
            {
                const int32_t roff = static_cast<int32_t>(q) + sc.rfd;
                const int64_t ri = ref0 + roff;
                const char refc = (ri >= 0 && ri < static_cast<int64_t>(A.ref_len)) ? A.ref[ri] : 'N';
                const uint32_t code = sq.nibble_at(q);
                if (char_of_code(code) != refc)
                {
                    // CandidateSnvBuffer::isCandidateSnvAnySample: a registered (position, base) is not counted as a mismatch
                    bool cand = false;
                    const int id = static_cast<int>(id_of_code(code));
                    const int32_t rel = site0 + roff;
                    if (id < 4 && rel >= 0 && rel < (1 << 30))
                    {
                        const uint32_t key = (static_cast<uint32_t>(rel) << 2) | static_cast<uint32_t>(id);
                        uint32_t l2 = 0, h2 = A.n_cand_snv;
                        while (l2 < h2)
                        {
                            const uint32_t mid = (l2 + h2) >> 1;
                            if (A.cand_snv[mid] < key) l2 = mid + 1;
                            else h2 = mid;
                        }
                        cand = l2 < A.n_cand_snv && A.cand_snv[l2] == key;
                    }
                    if (!cand) ++c;
                }
            }
            P[q + 1] = static_cast<uint16_t>(c);
        }
    }
    // the calls
    const uint32_t adjustedMapq = max(5u, static_cast<uint32_t>(rd.mapq));
    const bool tier1 = rd.flags & SX_PRF_TIER1;
    const uint32_t fwd_bit = (rd.flags & SX_PRF_FWD) ? (1u << 10) : 0u;
    const bool is_mapq_adjust = A.opt.isBasecallQualAdjustedForMapq && adjustedMapq <= 80u;
    const uint8_t* mqrow = tables->mappedq[min(adjustedMapq, 90u)];
    // dictionary-coded qualities: the 16 possible results (dictionary value -> MAPQ-adjusted value, 255 = above the table) as two 64-bit literals
    unsigned long long qlut_lo = 0, qlut_hi = 0;
    if (A.qual_bits == 4)
    {
        for (uint32_t v = 0; v < 16; ++v)
        {
            uint32_t q = A.qual_dict[v];
            if (is_mapq_adjust) q = q > SX_MAX_QSCORE ? 255u : mqrow[q];
            if (v < 8) qlut_lo |= static_cast<unsigned long long>(q & 0xffu) << (8u * v);
            else qlut_hi |= static_cast<unsigned long long>(q & 0xffu) << (8u * (v - 8u));
        }
    }
    k4_wstream qq;
    sq.init(gs);
    qq.init(A.qual + rd.qual_off);
    sc.init(path, as);
    const int max_pass = static_cast<int>(A.opt.mismatchDensityFilterMaxMismatchCount), max_pass2 = A.opt.tier2MismatchDensityFilterMaxMismatchCount;
    const int min_q = A.opt.minBasecallErrorPhredProb;
    const bool use_t2 = A.opt.useTier2Evidence != 0;
    unsigned long long* row = reinterpret_cast<unsigned long long*>(bc + static_cast<size_t>(r) * Ls); // Ls % 16 == 0: 8-byte aligned groups of four calls
    unsigned long long acc = 0;
    for (uint32_t q = rb; q < re; ++q)
    {
        K4_SEG_ADVANCE(sc, q)
        uint32_t v16 = 0;
        const int32_t site = site0 + static_cast<int32_t>(q) + sc.rfd; // (meaningful for a MATCH base)
        if (sc.kind == SX_SEG_MATCH && q < sc.seg_end && site >= 0 && site < static_cast<int32_t>(A.n_sites)) // is_pos_reportable
        {
            const uint32_t call_code = sq.nibble_at(q);
            const uint32_t call_id = id_of_code(call_code);
            if (call_id > 4u) atomicOr(status, ST_BASE);
            uint32_t qscore;
            if (A.qual_bits == 4)
            {
                const uint32_t v = qq.nibble_at(q);
                qscore = static_cast<uint32_t>(((v < 8u ? qlut_lo : qlut_hi) >> (8u * (v & 7u))) & 0xffu);
                if (is_mapq_adjust && qscore == 255u)
                {
                    atomicOr(status, ST_QUAL);
                    qscore = 0;
                }
            }
            else
            {
                qscore = qq.byte_at(q);
                if (is_mapq_adjust)
                {
                    if (qscore > SX_MAX_QSCORE)
                    {
                        atomicOr(status, ST_QUAL);
                        qscore = 0;
                    }
                    else qscore = mqrow[qscore];
                }
            }
            bool is_call_filter = (call_code == 15u) || (static_cast<int>(qscore) < min_q);
            bool is_tier2_call_filter = is_call_filter, is_neighbor_mismatch = false;
            if (isDensity)
            {
                const uint32_t di = min(delta_size - 1u, max(fs, q) - fs); // ddata::get's index
                int del = static_cast<int>(P[min(di + fs2, read_size - 1u) + 1u]) - static_cast<int>(P[di]);
                if (n_ev)
                {
                    if (n_ev <= K4B_MAX_EV)
                    {
                        for (uint32_t e = 0; e < n_ev; ++e)
                        {
                            const uint32_t st = ev[e] >> 16, ln = ev[e] & 0xffffu;
                            del += (max(fs2, st) - fs2 <= di && di < st + ln) ? 1 : 0;
                        }
                    }
                    else
                    {
                        uint32_t p2 = 0;
                        for (uint32_t j = 0; j < as; ++j)
                        {
                            const uint32_t k2 = path[j].kind, l2 = path[j].len;
                            if (!((j < first) || (j > last)) && (k2 == SX_SEG_INSERT || k2 == SX_SEG_DELETE))
                            {
                                const uint32_t ln = k2 == SX_SEG_INSERT ? l2 : 0u;
                                del += (max(fs2, p2) - fs2 <= di && di < p2 + ln) ? 1 : 0;
                            }
                            if (kind_read(k2)) p2 += l2;
                        }
                    }
                }
                if (!is_call_filter)
                {
                    is_call_filter = max_pass < del;
                    is_tier2_call_filter = use_t2 ? (max_pass2 < del) : is_call_filter;
                }
                const int mis = static_cast<int>(P[q + 1]) - static_cast<int>(P[q]);
                is_neighbor_mismatch = (del - mis) > 0;
            }
            const bool current_call_filter = tier1 ? is_call_filter : is_tier2_call_filter;
            const bool is_tier_specific_filter = tier1 && is_call_filter && !is_tier2_call_filter;
            v16 = min(qscore, 63u) | (min(call_id, 4u) << 6) | fwd_bit | ((is_neighbor_mismatch ? 1u : 0u) << 11) | ((current_call_filter ? 1u : 0u) << 12) |
                  ((is_tier_specific_filter ? 1u : 0u) << 13);
        }
        // four calls per 64-bit store (positions outside the MATCH segments hold 0: nobody reads them)
        acc |= static_cast<unsigned long long>(v16) << (16u * (q & 3u));
        if ((q & 3u) == 3u)
        {
            row[q >> 2] = acc;
            acc = 0;
        }
    }
    if (re > rb && (re & 3u) != 0u) row[(re - 1u) >> 2] = acc;
    rec[r] = out;
#undef K4_SEG_ADVANCE
}

constexpr uint32_t K4G_CHUNK = 8; // 32-site blocks per warp: its read range advances with the blocks

__global__ void __launch_bounds__(128) k4_gather_kernel(k4_args A, const k4_rrec* __restrict__ rec, const uint16_t* __restrict__ bc, uint32_t Ls, uint32_t reach_back,
                                                        uint32_t reach_fwd, const uint32_t* __restrict__ site_off, const uint32_t* __restrict__ t2_off,
                                                        uint16_t* __restrict__ calls, uint16_t* __restrict__ t2_calls)
{
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const uint32_t n_blocks = (A.n_sites + 31u) / 32u;
    const uint32_t b0 = gw * K4G_CHUNK;
    if (b0 >= n_blocks) return;
    const uint32_t b1 = min(b0 + K4G_CHUNK, n_blocks);
    // a read can reach site position P only if its buffer position lies in [P - reach_back, P + reach_fwd]
    // (reach_back = longest alignment span + largest |best start - buffer position|, reach_fwd = the latter)
    uint32_t lo = 0, hi = 0;
    if (lane == 0) lo = lower_bound_pos(A, static_cast<int64_t>(A.report_begin) + static_cast<int64_t>(b0) * 32 - reach_back);
    lo = __shfl_sync(FULL, lo, 0);
    hi = lo;
    for (uint32_t b = b0; b < b1; ++b)
    {
        const int64_t P0 = static_cast<int64_t>(A.report_begin) + static_cast<int64_t>(b) * 32;
        const int64_t want_lo = P0 - reach_back, want_hi = P0 + 31 + reach_fwd; // buffer positions in [want_lo, want_hi]
        while (lo < A.n_reads && bpos_of(A, lo) < want_lo) ++lo; // warp-uniform
        if (hi < lo) hi = lo;
        while (hi < A.n_reads && bpos_of(A, hi) <= want_hi) ++hi;
        const uint32_t s = b * 32u + lane;
        const bool live = s < A.n_sites;
        uint32_t c1 = live ? site_off[s] : 0u, c2 = live ? t2_off[s] : 0u;
        const int32_t si = live ? static_cast<int32_t>(s) : -0x40000000;
        for (uint32_t r = lo; r < hi; ++r)
        {
            const uint4* q4 = reinterpret_cast<const uint4*>(rec + r); // warp-uniform loads
            const uint4 hdr = q4[1];                                   // len[2] | p_lo[0] << 16, p_lo[1] | p_lo[2] << 16, n_iv, padding
            const uint32_t n_iv = hdr.z & 0xffu;
            if (n_iv == 0u) continue;
            const uint4 lo4 = q4[0]; // site_lo[0..2], len[0] | len[1] << 16
            uint32_t hit = 0xffffffffu;
            if (n_iv <= K4_REC_IV)
            {
                const uint32_t d0 = static_cast<uint32_t>(si - static_cast<int32_t>(lo4.x));
                if (d0 < (lo4.w & 0xffffu)) hit = (hdr.x >> 16) + d0;
                if (n_iv > 1u)
                {
                    const uint32_t d1 = static_cast<uint32_t>(si - static_cast<int32_t>(lo4.y));
                    if (d1 < (lo4.w >> 16)) hit = (hdr.y & 0xffffu) + d1;
                    if (n_iv > 2u)
                    {
                        const uint32_t d2 = static_cast<uint32_t>(si - static_cast<int32_t>(lo4.z));
                        if (d2 < (hdr.x & 0xffffu)) hit = (hdr.y >> 16) + d2;
                    }
                }
            }
            else
            {
                // more MATCH intervals than a record holds: the path itself
                const uint32_t rw = lo4.y, rbb = rw & 0xffffu, ree = rw >> 16, ns = (hdr.z >> 8) & 0x7fffffu;
                const sx_aln_seg* path = A.segs + lo4.z;
                int32_t ref_head = static_cast<int32_t>(lo4.x);
                uint32_t read_head = 0;
                for (uint32_t i = 0; i < ns; ++i)
                {
                    const uint32_t k = path[i].kind, len = path[i].len;
                    if (k == SX_SEG_MATCH)
                    {
                        const uint32_t a = max(read_head, rbb), e = min(read_head + len, ree);
                        if (a < e)
                        {
                            const uint32_t d = static_cast<uint32_t>(si - (ref_head + static_cast<int32_t>(a - read_head)));
                            if (d < e - a) hit = a + d;
                        }
                    }
                    if (kind_read(k)) read_head += len;
                    if (kind_ref(k)) ref_head += static_cast<int32_t>(len);
                }
            }
            if (hit != 0xffffffffu)
            {
                const uint16_t v = bc[static_cast<size_t>(r) * Ls + hit];
                if (hdr.z & 0x80000000u) calls[c1++] = v;
                else t2_calls[c2++] = v;
            }
        }
    }
}

int upload(sx_ctx* ctx, int slot, const void* src, size_t bytes, const void** dst, cudaStream_t st)
{
    void* p = nullptr;
    int rc = sx_ensure(ctx, slot, bytes + 64, &p);
    if (rc) return rc;
    if (bytes) SX_CUDA(ctx, cudaMemcpyAsync(p, src, bytes, cudaMemcpyHostToDevice, st));
    *dst = p;
    return SX_OK;
}
} // namespace

extern "C" void sx_default_pileup_opts(sx_pileup_opts* o)
{
    o->isBasecallQualAdjustedForMapq = 1;         // starling_common/starling_base_shared.hh:225
    o->minBasecallErrorPhredProb = 17;            // blt_common/blt_shared.hh:107
    o->mismatchDensityFilterFlankSize = 20;       // applications/starling/starling_shared.hh:37
    o->mismatchDensityFilterMaxMismatchCount = 2; // :36
    o->useTier2Evidence = 0;                      // starling_base_shared.hh:227
    o->tier2MismatchDensityFilterMaxMismatchCount = 10; // starling_common/Tier2Options.hh:37
    o->minDistanceFromReadEdge = 0;               // starling_base_shared.hh:252
    o->reserved_ = 0;
}

// all pointers (batch arrays and output columns) are device pointers; enqueues the three passes (one 8-byte round trip between the scans
// and the fill checks the capacities) and returns without waiting for the fill
int sx_k4_run(sx_ctx* ctx, const sx_pileup_reads_batch* d, const sx_pileup_columns* out, unsigned* launches_out)
{
    if (!d || !out || !out->site_off || !out->t2_off || !out->n_spandel || !out->n_submapped || !out->calls || !out->t2_calls)
        return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_reads_dev: NULL argument");
    if (d->report_end < d->report_begin) return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_reads_dev: empty report range");
    const uint32_t n_sites = static_cast<uint32_t>(d->report_end - d->report_begin);
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->s_compute;
    if (d->qual_bits != 0 && d->qual_bits != 8 && d->qual_bits != 4) return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_reads: qual_bits must be 0, 8 or 4");
    const uint32_t shift = d->buffer_pos ? d->max_pos_shift : 0u;
    const uint32_t W = std::max<uint32_t>(64, (d->max_ref_span + shift + 31u) & ~31u);
    const uint32_t Lcap = std::max<uint32_t>(64, (std::min<uint32_t>(d->max_read_len ? d->max_read_len : K4_MAX_READ, K4_MAX_READ) + 15u) & ~15u);
    if (W > K4_MAX_W)
        return sx_fail(ctx, SX_ERR_UNSUPPORTED, "sx_pileup_reads: max_ref_span %u exceeds the %u positions a window can hold (spliced alignments are not accelerated)",
                       d->max_ref_span, K4_MAX_W);
    k4_args A;
    A.reads = d->reads;
    A.bpos = d->buffer_pos;
    A.qual_bits = d->qual_bits;
    memcpy(A.qual_dict, d->qual_dict, 16);
    A.seq4 = d->seq4;
    A.qual = d->qual;
    A.segs = d->segs;
    A.ref = d->ref;
    A.cand_snv = d->cand_snv;
    A.n_reads = d->n_reads;
    A.n_cand_snv = d->n_cand_snv;
    A.ref_len = d->ref_len;
    A.ref_begin = d->ref_begin;
    A.report_begin = d->report_begin;
    A.report_end = d->report_end;
    A.origin = d->report_begin - static_cast<int32_t>(W);
    A.W = W;
    A.Lcap = Lcap;
    A.span_max = d->max_ref_span;
    A.shift_max = shift;
    A.n_windows = static_cast<uint32_t>((static_cast<int64_t>(d->report_end) - A.origin + W - 1) / W);
    A.n_sites = n_sites;
    A.opt = d->opts;

    // working arrays: the two offset arrays and the two count arrays are scanned in place in the caller's buffers
    int* d1 = reinterpret_cast<int*>(out->site_off);
    int* d2 = reinterpret_cast<int*>(out->t2_off);
    int* dsd = reinterpret_cast<int*>(out->n_spandel);
    int* dsm = reinterpret_cast<int*>(out->n_submapped);
    int *s1 = nullptr, *s2 = nullptr, *b1 = nullptr, *b2 = nullptr, *tile_sums = nullptr;
    int rc;
    const uint32_t tiles = (n_sites + 1 + SCAN_TILE - 1) / SCAN_TILE;
    if ((rc = sx_ensure(ctx, 26, (size_t)(n_sites + 1) * 8 + 64, reinterpret_cast<void**>(&s1)))) return rc;
    s2 = s1 + (n_sites + 1);
    if ((rc = sx_ensure(ctx, 64, (size_t)(n_sites + 1) * 8 + 64, reinterpret_cast<void**>(&b1)))) return rc;
    b2 = b1 + (n_sites + 1);
    if ((rc = sx_ensure(ctx, 27, (size_t)tiles * 8 * sizeof(int) + 64, reinterpret_cast<void**>(&tile_sums)))) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(d1, 0, (size_t)(n_sites + 1) * 4, st));
    SX_CUDA(ctx, cudaMemsetAsync(d2, 0, (size_t)(n_sites + 1) * 4, st));
    SX_CUDA(ctx, cudaMemsetAsync(dsd, 0, (size_t)n_sites * 4, st));
    SX_CUDA(ctx, cudaMemsetAsync(dsm, 0, (size_t)n_sites * 4, st));
    SX_CUDA(ctx, cudaMemsetAsync(s1, 0, (size_t)(n_sites + 1) * 8, st));
    SX_CUDA(ctx, cudaMemsetAsync(b1, 0, (size_t)(n_sites + 1) * 8, st));
    unsigned launches = 0;
    if (d->n_reads)
    {
        k4_count_kernel<<<(d->n_reads + 127) / 128, 128, 0, st>>>(A, d1, d2, s1, s2, b1, b2, dsd, dsm, ctx->d_status);
        SX_CUDA(ctx, cudaGetLastError());
        ++launches;
    }
    auto run_scans = [&](const scan_job& J, int n_arrays) -> int {
        const dim3 grid(tiles, n_arrays);
        k4_scan_tile_sums<<<grid, SCAN_THREADS, 0, st>>>(J, tile_sums, tiles);
        k4_scan_of_sums<<<n_arrays, SCAN_THREADS, 0, st>>>(J, tile_sums, tiles);
        k4_scan_tiles<<<grid, SCAN_THREADS, 0, st>>>(J, tile_sums, tiles);
        SX_CUDA(ctx, cudaGetLastError());
        launches += 3;
        return SX_OK;
    };
    {
        scan_job J{}; // differences -> counts
        int* arr[8] = {d1, d2, s1, s2, dsd, dsm, b1, b2};
        const uint32_t n[8] = {n_sites + 1, n_sites + 1, n_sites, n_sites, n_sites, n_sites, n_sites, n_sites};
        for (int k = 0; k < 8; ++k)
        {
            J.data[k] = arr[k];
            J.n[k] = n[k];
            J.exclusive[k] = 0;
        }
        if ((rc = run_scans(J, 8))) return rc;
        scan_job K{}; // counts -> CSR offsets
        K.data[0] = d1;
        K.data[1] = d2;
        K.n[0] = K.n[1] = n_sites + 1;
        K.exclusive[0] = K.exclusive[1] = 1;
        if ((rc = run_scans(K, 2))) return rc;
    }
    uint32_t totals[2] = {0, 0};
    SX_CUDA(ctx, cudaMemcpyAsync(&totals[0], out->site_off + n_sites, 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(&totals[1], out->t2_off + n_sites, 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    if (totals[0] > out->calls_capacity || totals[1] > out->t2_capacity)
        return sx_fail(ctx, SX_ERR_NOMEM, "sx_pileup_reads: the columns hold %u + %u calls, capacities are %llu + %llu", totals[0], totals[1],
                       (unsigned long long)out->calls_capacity, (unsigned long long)out->t2_capacity);
    // pass 3: thread per read + warp per 32 sites (default), or SX_K4_PLAN=1: one warp per window, reads in turn
    const size_t bc_bytes = (size_t)d->n_reads * Lcap * 2;
    const bool gather_plan = (getenv("SX_K4_PLAN") && atoi(getenv("SX_K4_PLAN")) == 2) && bc_bytes <= ((size_t)12 << 30); // (opt-in: the windowed fill is the default)
    if (d->n_reads && gather_plan)
    {
        k4_rrec* rec = nullptr;
        uint16_t* bc = nullptr;
        if ((rc = sx_ensure(ctx, 30, (size_t)(d->n_reads + 1) * sizeof(k4_rrec) + 64, reinterpret_cast<void**>(&rec)))) return rc;
        if ((rc = sx_ensure(ctx, 31, bc_bytes + 64, reinterpret_cast<void**>(&bc)))) return rc;
        const size_t smem = (size_t)K4B_THREADS * (Lcap + 2u) * 2u;
        if (smem > 48 * 1024) SX_CUDA(ctx, cudaFuncSetAttribute(k4_bases_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ctx->smem_optin)));
        k4_bases_kernel<<<(d->n_reads + K4B_THREADS - 1) / K4B_THREADS, K4B_THREADS, smem, st>>>(A, rec, bc, Lcap, ctx->d_tables, ctx->d_status);
        SX_CUDA(ctx, cudaGetLastError());
        const uint32_t n_warps = ((n_sites + 31u) / 32u + K4G_CHUNK - 1u) / K4G_CHUNK;
        k4_gather_kernel<<<(n_warps + 3u) / 4u, 128, 0, st>>>(A, rec, bc, Lcap, d->max_ref_span + shift, shift, out->site_off, out->t2_off, out->calls, out->t2_calls);
        SX_CUDA(ctx, cudaGetLastError());
        launches += 2;
    }
    else if (d->n_reads)
    {
        const size_t smem = (size_t)k4_warp_smem(W, Lcap) * K4_WARPS;
        if (smem > 48 * 1024) SX_CUDA(ctx, cudaFuncSetAttribute(k4_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(ctx->smem_optin)));
        k4_fill_kernel<<<(A.n_windows + K4_WARPS - 1) / K4_WARPS, K4_WARPS * 32, smem, st>>>(A, out->site_off, out->t2_off, s1, s2, b1, b2, out->calls, out->t2_calls, ctx->d_tables,
                                                                                         ctx->d_status);
        SX_CUDA(ctx, cudaGetLastError());
        ++launches;
    }
    *launches_out += launches;
    return SX_OK;
}

extern "C" int sx_pileup_reads_dev(sx_ctx* ctx, const sx_pileup_reads_batch* d, sx_pileup_columns* out)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    sx_kernel_timer t(ctx);
    unsigned launches = 0;
    int rc = sx_k4_run(ctx, d, out, &launches);
    if (rc) return rc;
    t.stop(launches);
    rc = t.finish();
    if (rc) return rc;
    return sx_check_status(ctx, "sx_pileup_reads");
}

extern "C" int sx_pileup_reads(sx_ctx* ctx, const sx_pileup_reads_batch* b, sx_pileup_columns* out)
{
    if (!ctx) return SX_ERR_ARG;
    if (!b || !out || !b->reads || !out->site_off || !out->t2_off || !out->n_spandel || !out->n_submapped)
        return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_reads: NULL argument");
    if (b->report_end < b->report_begin) return sx_fail(ctx, SX_ERR_ARG, "sx_pileup_reads: empty report range");
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->s_compute;
    const uint32_t n_sites = static_cast<uint32_t>(b->report_end - b->report_begin);
    sx_pileup_reads_batch d = *b;
    int rc;
    const sx_pileup_read& end = b->reads[b->n_reads];
    if ((rc = upload(ctx, 0, b->reads, (size_t)(b->n_reads + 1) * sizeof(sx_pileup_read), reinterpret_cast<const void**>(&d.reads), st))) return rc;
    if ((rc = upload(ctx, 1, b->seq4, end.seq_off, reinterpret_cast<const void**>(&d.seq4), st))) return rc;
    if ((rc = upload(ctx, 2, b->qual, end.qual_off, reinterpret_cast<const void**>(&d.qual), st))) return rc;
    if ((rc = upload(ctx, 3, b->segs, (size_t)b->n_segs * sizeof(sx_aln_seg), reinterpret_cast<const void**>(&d.segs), st))) return rc;
    if ((rc = upload(ctx, 4, b->ref, b->ref_len, reinterpret_cast<const void**>(&d.ref), st))) return rc;
    if ((rc = upload(ctx, 5, b->cand_snv, (size_t)b->n_cand_snv * 4, reinterpret_cast<const void**>(&d.cand_snv), st))) return rc;
    if (b->buffer_pos && (rc = upload(ctx, 9, b->buffer_pos, (size_t)b->n_reads * 4, reinterpret_cast<const void**>(&d.buffer_pos), st))) return rc;
    sx_pileup_columns dc = *out;
    void* p = nullptr;
    if ((rc = sx_ensure(ctx, 6, (size_t)(n_sites + 1) * 4 * 4 + 64, &p))) return rc;
    dc.site_off = static_cast<uint32_t*>(p);
    dc.t2_off = dc.site_off + (n_sites + 1);
    dc.n_spandel = dc.t2_off + (n_sites + 1);
    dc.n_submapped = dc.n_spandel + (n_sites + 1);
    if ((rc = sx_ensure(ctx, 7, (size_t)out->calls_capacity * 2 + 64, &p))) return rc;
    dc.calls = static_cast<uint16_t*>(p);
    if ((rc = sx_ensure(ctx, 8, (size_t)out->t2_capacity * 2 + 64, &p))) return rc;
    dc.t2_calls = static_cast<uint16_t*>(p);
    rc = sx_pileup_reads_dev(ctx, &d, &dc);
    if (rc && rc != SX_ERR_NOMEM) return rc;
    // offsets and counts are valid even when a capacity was too small (the caller can size and retry)
    SX_CUDA(ctx, cudaMemcpyAsync(out->site_off, dc.site_off, (size_t)(n_sites + 1) * 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out->t2_off, dc.t2_off, (size_t)(n_sites + 1) * 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out->n_spandel, dc.n_spandel, (size_t)n_sites * 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out->n_submapped, dc.n_submapped, (size_t)n_sites * 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    if (rc) return rc;
    const uint32_t n1 = out->site_off[n_sites], n2 = out->t2_off[n_sites];
    if (n1) SX_CUDA(ctx, cudaMemcpyAsync(out->calls, dc.calls, (size_t)n1 * 2, cudaMemcpyDeviceToHost, st));
    if (n2) SX_CUDA(ctx, cudaMemcpyAsync(out->t2_calls, dc.t2_calls, (size_t)n2 * 2, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    return SX_OK;
}
