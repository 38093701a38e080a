// k7_enumerate.cu -- K7: candidate-alignment enumeration, one read per thread.
//
// Replaces (include/strelka_b200.h, "K7 enumerate_alignments"; SURVEY 8a row a3 / 8f3)
//   starling_common/starling_read_align.cpp:1816-1994  getCandidateAlignments
//   starling_common/starling_read_align.cpp:857-1277   candidate_alignment_search (+ the helpers listed in the header)
// and produces the alignment lists K1 scores and K6 evaluates, in the order both expect (std::set<CandidateAlignment>).
//
// Shape of the work: per read an irregular depth-first search over a handful of indels (typically 2-6, capped at 64), integer
// only, with a variable-size result.  There is no reuse between reads and nothing GEMM-like; the algorithmic floor is reading the
// window and the input alignment once and writing the alignments once.  The reference's by-value containers become an explicit
// frame stack with position-indexed bit masks (k7_core.cuh), so a read's whole working set is a fixed-size block of a per-thread
// arena.  The result size is unknown until the search has run, and the output must be a dense CSR in read order (it IS the next
// kernels' input), so the search runs twice with a scan in between:
//   k7_count_kernel : search -> per read (alignments, segments, keys) + status
//   scan            : three exclusive prefix sums over reads (one block per 2048 reads + a single-block pass over the block sums)
//   k7_write_kernel : search again (deterministic) -> the set, in its order, at the read's offsets
// Searching twice costs less than a second arena large enough to keep every read's set between the passes, and keeps the output
// independent of scheduling.  Persistent grid: resident blocks x SM count, a thread strides over reads.

#include "k7_core.cuh"
#include "sx_internal.h"
#include "sx_regroup.cuh"
#include "sx_scan3.cuh"

#include <algorithm>
#include <cstdlib>

namespace
{
constexpr int K7_THREADS = 64;
constexpr int K7_ST_SHIFT = 14; // device status bit 16384: an output capacity is too small (reported as SX_ERR_CAPACITY by the host)

struct k7_counts // per read, then (after the scan) its exclusive offsets
{
    uint32_t* aln;
    uint32_t* seg;
    uint32_t* key;
};

__global__ void __launch_bounds__(K7_THREADS) k7_count_kernel(const k7_view v, unsigned char* __restrict__ arena, const size_t per_thread, const uint32_t maxA,
                                                              const uint32_t maxF, const uint32_t* __restrict__ read_region, uint8_t* __restrict__ status, const k7_counts c)
{
    const uint32_t t(blockIdx.x * blockDim.x + threadIdx.x), nthr(gridDim.x * blockDim.x);
    k7_scratch S(k7_scratch_at(arena + (size_t)t * per_thread, maxA, maxF));
    for (uint32_t r = t; r < v.b.n_reads; r += nthr)
    {
        const uint32_t st(k7_enumerate_read(v, read_region[r], r, S));
        uint32_t na, ns, nk;
        k7_count(S, st, na, ns, nk);
        status[r] = (uint8_t)st;
        c.aln[r] = na;
        c.seg[r] = ns;
        c.key[r] = nk;
    }
}

// region of every read (reads of a region are consecutive): one thread per region fills its reads' entries; and the largest window of
// the batch -- a search can hold at most as many indels as its region's window has entries, so that many + 1 frames always suffice
__global__ void k7_read_region_kernel(const uint32_t n_regions, const uint32_t* __restrict__ region_read_off, const uint32_t* __restrict__ region_key_off,
                                      uint32_t* __restrict__ read_region, uint32_t* __restrict__ max_window)
{
    uint32_t m(0);
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < n_regions; g += gridDim.x * blockDim.x)
    {
        for (uint32_t r = region_read_off[g]; r < region_read_off[g + 1]; ++r) read_region[r] = g;
        m = max(m, region_key_off[g + 1] - region_key_off[g]);
    }
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0 && m) atomicMax(max_window, m);
}

// frames a search of this batch can need (see k7_read_region_kernel): one host round trip of 4 bytes sizes the arena
int k7_frames_needed(sx_ctx* ctx, const sx_enum_batch* d, uint32_t* read_region, uint32_t* max_window_dev, uint32_t* frames)
{
    cudaStream_t st(ctx->s_compute);
    SX_CUDA(ctx, cudaMemsetAsync(max_window_dev, 0, 4, st));
    const int g0(std::max(1, std::min<int>((int)((d->n_regions + 127) / 128), ctx->sm_count * 8)));
    k7_read_region_kernel<<<g0, 128, 0, st>>>(d->n_regions, d->region_read_off, d->region_key_off, read_region, max_window_dev);
    SX_CUDA(ctx, cudaGetLastError());
    uint32_t h(0);
    SX_CUDA(ctx, cudaMemcpyAsync(&h, max_window_dev, 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    *frames = std::min<uint32_t>(K7_MAX_INDELS, h) + 1u;
    return SX_OK;
}

// phase 2 of the scan + the batch-wide closing entries; flags the capacity overflow
__global__ void __launch_bounds__(K7_SCAN_THREADS) k7_scan_finish(const uint32_t n, const k7_counts c, const uint32_t* __restrict__ sums, const uint32_t n_tiles,
                                                                  const uint32_t* __restrict__ totals, const sx_enum_out o, int* __restrict__ status)
{
    const uint32_t tile(blockIdx.x);
    const uint32_t base(tile * K7_SCAN_THREADS * K7_SCAN_ITEMS + threadIdx.x * K7_SCAN_ITEMS);
    const uint32_t oa(sums[tile]), os(sums[(size_t)n_tiles + tile]), ok(sums[(size_t)2 * n_tiles + tile]);
    for (int i = 0; i < K7_SCAN_ITEMS; ++i)
        if (base + i < n)
        {
            const uint32_t a(c.aln[base + i] + oa);
            c.aln[base + i] = a;
            c.seg[base + i] += os;
            c.key[base + i] += ok;
            o.aln_off[base + i] = a;
        }
    if (blockIdx.x == 0 && threadIdx.x == 0)
    {
        o.aln_off[n] = totals[0];
        o.totals[0] = totals[0];
        o.totals[1] = totals[1];
        o.totals[2] = totals[2];
        if (totals[0] > o.cap_alns || totals[1] > o.cap_segs || totals[2] > o.cap_keys) atomicOr(status, 1 << K7_ST_SHIFT);
        else
        {
            o.aln_seg_off[totals[0]] = totals[1];
            o.aln_key_off[totals[0]] = totals[2];
        }
    }
}

__global__ void __launch_bounds__(K7_THREADS) k7_write_kernel(const k7_view v, unsigned char* __restrict__ arena, const size_t per_thread, const uint32_t maxA,
                                                              const uint32_t maxF, const uint32_t* __restrict__ read_region, const uint8_t* __restrict__ status,
                                                              const k7_counts c, const sx_enum_out o, const uint32_t* __restrict__ totals)
{
    if (totals[0] > o.cap_alns || totals[1] > o.cap_segs || totals[2] > o.cap_keys) return; // reported by k7_scan_finish
    const uint32_t t(blockIdx.x * blockDim.x + threadIdx.x), nthr(gridDim.x * blockDim.x);
    k7_scratch S(k7_scratch_at(arena + (size_t)t * per_thread, maxA, maxF));
    for (uint32_t r = t; r < v.b.n_reads; r += nthr)
    {
        if (status[r] & (SX_ENUM_ST_EXCEPTION | SX_ENUM_ST_LIMIT)) continue;
        const uint32_t na((r + 1 < v.b.n_reads ? c.aln[r + 1] : totals[0]) - c.aln[r]);
        if (na == 0) continue;
        k7_enumerate_read(v, read_region[r], r, S);
        k7_write(S, o, c.aln[r], c.seg[r], c.key[r]);
    }
}

// ---------------------------------------------------------------------------------------------------------------------------
// SX_ENUM_F_FAST: one search per read.  Tier 1 keeps the scratch in LOCAL memory (the hardware interleaves it per lane, so a converged
// warp touches one line where the arena touches 32 sectors) sized for ordinary reads; a read that needs more frames or slots is
// marked and searched again by tier 2 in the global arena.  Either tier appends the read's alignments to a log (bump allocator) and
// records where; after the scan k7_gather_kernel copies every blob to its place in read order -- the output is independent of
// which thread got which piece of the log.
// ---------------------------------------------------------------------------------------------------------------------------
// The local tier comes in two sizes (SX_K7_LOCAL_ALNS=16|40, default 40): local memory a thread never touches costs nothing but address
// space, while every read the tier passes on is searched a second time from the start in the slower arena.
constexpr uint32_t K7_LOCAL_FRAMES = 12;
constexpr uint32_t K7_MID_ALNS = 96; // per-read capacity of the first arena tier
__host__ __device__ constexpr uint32_t k7_local_bytes(const uint32_t alns) // k7_scratch_bytes(alns, K7_LOCAL_FRAMES), as a constant expression (checked in k7_run_fast)
{
    return (uint32_t)(((((size_t)K7_MAX_INDELS * 2 + 15) & ~(size_t)15) + ((sizeof(k7_frame) * K7_LOCAL_FRAMES + 15) & ~(size_t)15) +
                       ((sizeof(k7_cal) * ((size_t)alns + 1) + 15) & ~(size_t)15) + (((size_t)alns * 2 + 15) & ~(size_t)15) + 255) & ~(size_t)255);
}

struct k7_log
{
    uint32_t* words;             // the log
    unsigned long long* cursor;  // next free word
    uint32_t cap;                // words available
    uint32_t* blob_off;          // [n_reads] where a read's blob starts (UINT32_MAX: it did not fit -- then the output does not either)
};

__device__ __forceinline__ void k7_log_append(const k7_log& L, const k7_scratch& S, const uint32_t r)
{
    const uint32_t w(k7_blob_words(S));
    uint32_t off(UINT32_MAX);
    if (w)
    {
        const unsigned long long at(atomicAdd(L.cursor, (unsigned long long)w));
        if (at + w <= (unsigned long long)L.cap)
        {
            off = (uint32_t)at;
            k7_blob_write(S, L.words + off);
        }
    }
    L.blob_off[r] = off;
}

// the reads a tier could not finish: a dense list for the next tier (which thread appends where does not matter: the output is placed by the scan)
struct k7_retry
{
    uint32_t* list1; // [n_reads] reads the local tier passed on
    uint32_t* list2; // [n_reads] reads the small-arena tier passed on
    uint32_t* n;     // [3] their counts; n[2]: the reads of list0
    uint32_t* list0; // [n_reads] or NULL: the reads the gates let through (batches with a gate array: about half of a 30x window's reads
                     // never reach the search, and a thread that returns at once idles while its warp-mates search)
};

// dense list of the reads that go into the search, in read order within a warp's 32 (neighbouring list entries share their region's window)
__global__ void k7_active_reads_kernel(const uint32_t n_reads, const uint8_t* __restrict__ gate, uint32_t* __restrict__ list0, uint32_t* __restrict__ count)
{
    const uint32_t lane(threadIdx.x & 31u);
    for (uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) - lane; b < n_reads; b += gridDim.x * blockDim.x)
    {
        const uint32_t r(b + lane);
        const bool on(r < n_reads && (gate[r] & SX_GATE_REALIGN));
        const unsigned m(__ballot_sync(0xffffffffu, on));
        uint32_t at(0);
        if (lane == 0 && m) at = atomicAdd(count, (uint32_t)__popc(m));
        at = __shfl_sync(0xffffffffu, at, 0);
        if (on) list0[at + __popc(m & ((1u << lane) - 1u))] = r;
    }
}

// ---- reads of one shape side by side.  The active list is in read order: a warp's 32 reads are one region's reads at neighbouring positions,
// and they differ in WHICH of the window's entries they reach -- so their searches have different trees and the warp executes every tree in turn
// (about half of the 32 lanes active).  A read's shape class = the window entries (first four of its region) its input alignment's range is adjacent
// to (bp_adjacent: what add_indels_in_range will put into indel_order) + which of them the alignment already contains.  The list is regrouped
// by class with a block-local counting sort; which thread searches which read does not matter (the output is placed by the scan).
constexpr uint32_t K7_N_CLASS = SX_RG_CLASSES;
constexpr int K7_CLS_THREADS = SX_RG_THREADS, K7_CLS_ITEMS = SX_RG_ITEMS;

__device__ __forceinline__ uint32_t k7_read_class(const sx_enum_batch& b, const uint32_t region, const uint32_t r)
{
    const uint32_t k0(b.region_key_off[region]), nw(min(b.region_key_off[region + 1] - k0, 4u));
    const uint32_t s0(b.in_seg_off[r]), ns(b.in_seg_off[r + 1] - s0);
    // get_soft_clip_alignment_range of the input alignment (k7_soft_clip_range)
    uint32_t lead(0), trail(0), ref_len(0);
    bool in_lead(true);
    for (uint32_t i = 0; i < ns; ++i)
    {
        const unsigned t(b.in_segs[s0 + i].kind);
        const uint32_t len(b.in_segs[s0 + i].len);
        if (k7_seg_ref_len(t)) ref_len += len;
        if (t == SX_AP_HARD_CLIP || t == SX_AP_SOFT_CLIP) continue;
        if (t == SX_AP_INSERT)
        {
            if (in_lead) lead += len;
            else trail += len;
        }
        else
        {
            in_lead = false;
            trail = 0;
        }
    }
    const int32_t eb(b.in_pos[r] - (int32_t)lead), ee(b.in_pos[r] + (int32_t)ref_len + (int32_t)trail);
    uint32_t cls(0);
    for (uint32_t k = 0; k < nw; ++k)
        if (k7_bp_adjacent(eb, ee, b.keys[k0 + k])) cls |= 1u << k;
    for (uint32_t i = b.in_key_off[r]; i < b.in_key_off[r + 1]; ++i)
        if (b.in_keys[i] < 4u) cls |= 16u << b.in_keys[i];
    return cls & (K7_N_CLASS - 1u);
}

__global__ void __launch_bounds__(K7_CLS_THREADS) k7_class_count_kernel(const k7_view v, const uint32_t* __restrict__ read_region, const uint32_t* __restrict__ list, const uint32_t* __restrict__ n_list,
                                                                        uint8_t* __restrict__ cls, uint32_t* __restrict__ hist)
{
    __shared__ uint32_t s_cnt[K7_N_CLASS];
    s_cnt[threadIdx.x] = 0;
    __syncthreads();
    const uint32_t n(*n_list);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    {
        const uint32_t r(list[i]);
        const uint32_t c(k7_read_class(v.b, read_region[r], r));
        cls[i] = (uint8_t)c;
        atomicAdd(&s_cnt[c], 1u);
    }
    __syncthreads();
    if (s_cnt[threadIdx.x]) atomicAdd(&hist[threadIdx.x], s_cnt[threadIdx.x]);
}

template <uint32_t K7_LOCAL_ALNS, int K7_MIN_BLOCKS>
__global__ void __launch_bounds__(K7_THREADS, K7_MIN_BLOCKS) k7_search_local_kernel(const k7_view v, const uint32_t* __restrict__ read_region, uint8_t* __restrict__ status,
                                                                     const k7_retry R, const k7_counts c, const k7_log L)
{
    __align__(16) unsigned char local[k7_local_bytes(K7_LOCAL_ALNS)];
    k7_scratch S(k7_scratch_at(local, K7_LOCAL_ALNS, K7_LOCAL_FRAMES, K7_ST_RETRY));
    const uint32_t t(blockIdx.x * blockDim.x + threadIdx.x), nthr(gridDim.x * blockDim.x);
    const uint32_t n_work(R.list0 ? R.n[2] : v.b.n_reads); // (with a list: the counts / status of the other reads were zeroed by the host side)
    for (uint32_t i = t; i < n_work; i += nthr)
    {
        const uint32_t r(R.list0 ? R.list0[i] : i);
        const uint32_t st(k7_enumerate_read(v, read_region[r], r, S));
        const bool retry((st & K7_ST_RETRY) != 0);
        uint32_t na(0), ns(0), nk(0);
        if (!retry)
        {
            k7_count(S, st, na, ns, nk);
            status[r] = (uint8_t)st;
            if (na) k7_log_append(L, S, r);
        }
        else R.list1[atomicAdd(&R.n[0], 1u)] = r;
        c.aln[r] = na;
        c.seg[r] = ns;
        c.key[r] = nk;
    }
}

// level 1: the reads of list1 in a modest per-thread arena (most of them need a few dozen alignments); what still does not fit goes to list2.
// level 2: the reads of list2 with the caller's full per-read capacity (the reference's own bound is 5000 alignments), few threads.
__global__ void __launch_bounds__(K7_THREADS) k7_search_arena_kernel(const k7_view v, unsigned char* __restrict__ arena, const size_t per_thread, const uint32_t maxA,
                                                                     const uint32_t maxF, const uint32_t* __restrict__ read_region, uint8_t* __restrict__ status,
                                                                     const k7_retry R, const int level, const int pass_on, const k7_counts c, const k7_log L)
{
    const uint32_t t(blockIdx.x * blockDim.x + threadIdx.x), nthr(gridDim.x * blockDim.x);
    k7_scratch S(k7_scratch_at(arena + (size_t)t * per_thread, maxA, maxF, pass_on ? K7_ST_RETRY : SX_ENUM_ST_LIMIT));
    const uint32_t* list(level == 1 ? R.list1 : R.list2);
    const uint32_t cnt(R.n[level - 1]);
    for (uint32_t i = t; i < cnt; i += nthr)
    {
        const uint32_t r(list[i]);
        const uint32_t st(k7_enumerate_read(v, read_region[r], r, S));
        if (st & K7_ST_RETRY) // (only with pass_on)
        {
            R.list2[atomicAdd(&R.n[1], 1u)] = r;
            continue;
        }
        uint32_t na, ns, nk;
        k7_count(S, st, na, ns, nk);
        status[r] = (uint8_t)st;
        if (na) k7_log_append(L, S, r);
        c.aln[r] = na;
        c.seg[r] = ns;
        c.key[r] = nk;
    }
}

__global__ void k7_gather_kernel(const uint32_t n_reads, const k7_counts c, const k7_log L, const sx_enum_out o, const uint32_t* __restrict__ totals,
                                 const uint32_t* __restrict__ list, const uint32_t* __restrict__ n_list)
{
    if (totals[0] > o.cap_alns || totals[1] > o.cap_segs || totals[2] > o.cap_keys) return; // reported by k7_scan_finish
    // with a list (in read order: the CSR output is written in read order): only the searched reads have a blob
    const uint32_t n_work(list ? *n_list : n_reads);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_work; i += gridDim.x * blockDim.x)
    {
        const uint32_t r(list ? list[i] : i);
        const uint32_t na((r + 1 < n_reads ? c.aln[r + 1] : totals[0]) - c.aln[r]);
        if (na == 0 || L.blob_off[r] == UINT32_MAX) continue;
        k7_blob_gather(L.words + L.blob_off[r], na, o, c.aln[r], c.seg[r], c.key[r]);
    }
}

// the reference's table: starling_align_limit (starling_align_limit.cpp:53-88).  Every quantity is an integer far below 2^24 until
// the running sum passes max_alignments, so the float arithmetic of the reference is exact there and doubles reproduce it.
unsigned k7_max_candidate_alignment_toggle(const unsigned n_indel, const unsigned max_alignments)
{
    const double max(max_alignments);
    double sum(1.);
    for (unsigned i = 0; i < n_indel; ++i)
    {
        const unsigned k(i + 1);
        double binom(1.);
        for (unsigned j = 1; j <= k; ++j) binom = binom * (double)(n_indel - k + j) / (double)j; // exact: each partial product is an integer
        sum += std::ldexp(1., (int)k) * std::floor(binom + 0.5);
        if (sum > max) return i;
    }
    return n_indel;
}

int k7_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* o, unsigned* launches)
{
    cudaStream_t st(ctx->s_compute);
    const uint32_t n(d->n_reads);
    const uint32_t maxA(d->opts.max_alns_per_read ? std::min<uint32_t>(d->opts.max_alns_per_read, 65535u) : 64u);
    int rc;
    uint32_t* read_region(nullptr);
    if ((rc = sx_ensure(ctx, 41, (size_t)n * 4 + 32, reinterpret_cast<void**>(&read_region)))) return rc;
    uint32_t maxF(K7_MAX_INDELS + 1);
    if ((rc = k7_frames_needed(ctx, d, read_region, read_region + n + 1, &maxF))) return rc; // (also fills read_region)
    const size_t per_thread((k7_scratch_bytes(maxA, maxF) + 255) & ~(size_t)255);
    int per_sm(1);
    SX_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k7_count_kernel, K7_THREADS, 0));
    per_sm = std::max(1, per_sm);
    size_t blocks(std::min<size_t>(((size_t)n + K7_THREADS - 1) / K7_THREADS, (size_t)ctx->sm_count * per_sm));
    const size_t arena_cap((size_t)4 << 30);
    while (blocks > 1 && blocks * K7_THREADS * per_thread > arena_cap) blocks = (blocks + 1) / 2;
    unsigned char* arena(nullptr);
    if ((rc = sx_ensure(ctx, 40, blocks * K7_THREADS * per_thread, reinterpret_cast<void**>(&arena)))) return rc;
    k7_counts c;
    if ((rc = sx_ensure(ctx, 42, (size_t)n * 4 + 16, reinterpret_cast<void**>(&c.aln)))) return rc;
    if ((rc = sx_ensure(ctx, 43, (size_t)n * 4 + 16, reinterpret_cast<void**>(&c.seg)))) return rc;
    if ((rc = sx_ensure(ctx, 44, (size_t)n * 4 + 16, reinterpret_cast<void**>(&c.key)))) return rc;
    const uint32_t tile(K7_SCAN_THREADS * K7_SCAN_ITEMS), n_tiles((n + tile - 1) / tile);
    uint32_t* sums(nullptr);
    if ((rc = sx_ensure(ctx, 45, ((size_t)3 * n_tiles + 4) * 4, reinterpret_cast<void**>(&sums)))) return rc;
    uint32_t* totals(sums + (size_t)3 * n_tiles);

    k7_view v;
    v.b = *d;
    k7_count_kernel<<<(unsigned)blocks, K7_THREADS, 0, st>>>(v, arena, per_thread, maxA, maxF, read_region, o->status, c);
    SX_CUDA(ctx, cudaGetLastError());
    k7_scan_tiles<<<n_tiles, K7_SCAN_THREADS, 0, st>>>(n, c.aln, c.seg, c.key, sums, n_tiles);
    SX_CUDA(ctx, cudaGetLastError());
    k7_scan_sums<<<1, K7_SCAN_THREADS, 0, st>>>(sums, n_tiles, totals);
    SX_CUDA(ctx, cudaGetLastError());
    k7_scan_finish<<<n_tiles, K7_SCAN_THREADS, 0, st>>>(n, c, sums, n_tiles, totals, *o, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    k7_write_kernel<<<(unsigned)blocks, K7_THREADS, 0, st>>>(v, arena, per_thread, maxA, maxF, read_region, o->status, c, *o, totals);
    SX_CUDA(ctx, cudaGetLastError());
    *launches = 6;
    return SX_OK;
}

int k7_run_fast(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* o, unsigned* launches)
{
    static_assert(K7_LOCAL_FRAMES <= K7_MAX_INDELS + 1, "local tier sizes");
    bool small_local(false);
    if (const char* e = getenv("SX_K7_LOCAL_ALNS")) small_local = atoi(e) <= 16;
    // the same kernel compiled for 16 / 24 / 32 resident blocks per SM (64 / 40 / 32 registers; its state lives in local memory, so the smaller
    // register budgets spill next to nothing): more warps to hide its latency
    // 16 on an H100: K7 103 vs 119 ms per step at 16 vs 24 (bench.py, 300k cfg2 loci, two runs each; H100 80GB HBM3, 400 W power limit)
    const int min_blocks(getenv("SX_K7_MIN_BLOCKS") ? atoi(getenv("SX_K7_MIN_BLOCKS")) : 16);
    const auto local_kernel(small_local ? k7_search_local_kernel<16, 16>
                            : min_blocks >= 32 ? k7_search_local_kernel<40, 32>
                            : min_blocks >= 24 ? k7_search_local_kernel<40, 24>
                                               : k7_search_local_kernel<40, 16>);
    if (k7_scratch_bytes(small_local ? 16 : 40, K7_LOCAL_FRAMES) > k7_local_bytes(small_local ? 16 : 40)) return sx_fail(ctx, SX_ERR_ARG, "k7: local scratch smaller than its contents");
    cudaStream_t st(ctx->s_compute);
    const uint32_t n(d->n_reads);
    const uint32_t maxA(d->opts.max_alns_per_read ? std::min<uint32_t>(d->opts.max_alns_per_read, 65535u) : 64u);
    int rc;
    uint32_t* read_region(nullptr);
    if ((rc = sx_ensure(ctx, 41, (size_t)n * 4 + 32, reinterpret_cast<void**>(&read_region)))) return rc;
    uint32_t maxF(K7_MAX_INDELS + 1);
    if ((rc = k7_frames_needed(ctx, d, read_region, read_region + n + 1, &maxF))) return rc; // (also fills read_region)
    const size_t per_thread((k7_scratch_bytes(maxA, maxF) + 255) & ~(size_t)255);
    int per_sm(1), per_sm_local(1);
    SX_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k7_search_arena_kernel, K7_THREADS, 0));
    SX_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_local, local_kernel, K7_THREADS, 0));
    per_sm = std::max(1, per_sm);
    per_sm_local = std::max(1, per_sm_local);
    const size_t n_blocks(((size_t)n + K7_THREADS - 1) / K7_THREADS);
    // (SX_K7_LOCAL_BLOCKS_PER_SM: tuning knob -- fewer resident threads keep the tier's local-memory scratch closer to the L2's size)
    if (const char* e = getenv("SX_K7_LOCAL_BLOCKS_PER_SM")) per_sm_local = std::max(1, std::min(per_sm_local, atoi(e)));
    const size_t blocks_local(std::min<size_t>(n_blocks, (size_t)ctx->sm_count * per_sm_local));
    // two arena tiers: a modest one (K7_MID_ALNS alignments per read, the whole device) for the reads the local tier passes on, and -- only when the
    // caller allows more per read -- one with the caller's capacity for the few that still do not fit (few threads: its per-thread scratch is large)
    const uint32_t maxA1(std::min<uint32_t>(maxA, K7_MID_ALNS));
    const bool two_levels(maxA > maxA1);
    const size_t per_thread1((k7_scratch_bytes(maxA1, maxF) + 255) & ~(size_t)255);
    size_t blocks1(std::min<size_t>(n_blocks, (size_t)ctx->sm_count * per_sm));
    const size_t arena_cap((size_t)1 << 30);
    while (blocks1 > 1 && blocks1 * K7_THREADS * per_thread1 > arena_cap) blocks1 = (blocks1 + 1) / 2;
    size_t blocks(std::min<size_t>(n_blocks, std::max<size_t>(1, (size_t)ctx->sm_count * per_sm / 4)));
    while (blocks > 1 && blocks * K7_THREADS * per_thread > arena_cap) blocks = (blocks + 1) / 2;
    unsigned char *arena(nullptr), *arena1(nullptr);
    if ((rc = sx_ensure(ctx, 40, blocks1 * K7_THREADS * per_thread1, reinterpret_cast<void**>(&arena1)))) return rc;
    if (two_levels && (rc = sx_ensure(ctx, 65, blocks * K7_THREADS * per_thread, reinterpret_cast<void**>(&arena)))) return rc;
    k7_counts c;
    if ((rc = sx_ensure(ctx, 42, (size_t)n * 4 + 16, reinterpret_cast<void**>(&c.aln)))) return rc;
    if ((rc = sx_ensure(ctx, 43, (size_t)n * 4 + 16, reinterpret_cast<void**>(&c.seg)))) return rc;
    if ((rc = sx_ensure(ctx, 44, (size_t)n * 4 + 16, reinterpret_cast<void**>(&c.key)))) return rc;
    const uint32_t tile(K7_SCAN_THREADS * K7_SCAN_ITEMS), n_tiles((n + tile - 1) / tile);
    uint32_t* sums(nullptr);
    if ((rc = sx_ensure(ctx, 45, ((size_t)3 * n_tiles + 4) * 4, reinterpret_cast<void**>(&sums)))) return rc;
    uint32_t* totals(sums + (size_t)3 * n_tiles);
    // the log holds whatever the output arrays can hold: 3 words + segments + ceil(keys / 2) words per alignment
    const unsigned long long want_words((unsigned long long)o->cap_alns * 4ull + o->cap_segs + (o->cap_keys + 1ull) / 2ull + 16ull);
    k7_log L;
    L.cap = (uint32_t)std::min<unsigned long long>(want_words, 0xFFFFFFF0ull);
    k7_retry R;
    if ((rc = sx_ensure(ctx, 54, (size_t)L.cap * 4 + 16, reinterpret_cast<void**>(&L.words)))) return rc;
    if ((rc = sx_ensure(ctx, 55, (size_t)n * 4 + 16, reinterpret_cast<void**>(&L.blob_off)))) return rc;
    if ((rc = sx_ensure(ctx, 56, 16, reinterpret_cast<void**>(&L.cursor)))) return rc;
    if ((rc = sx_ensure(ctx, 57, (size_t)n * 4 + 16, reinterpret_cast<void**>(&R.list1)))) return rc;
    if ((rc = sx_ensure(ctx, 66, (size_t)n * 4 + 16, reinterpret_cast<void**>(&R.list2)))) return rc;
    if ((rc = sx_ensure(ctx, 67, 16, reinterpret_cast<void**>(&R.n)))) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(L.cursor, 0, 16, st));
    SX_CUDA(ctx, cudaMemsetAsync(R.n, 0, 16, st));
    R.list0 = nullptr;
    unsigned extra(0);
    if (d->gate)
    {
        if ((rc = sx_ensure(ctx, 68, (size_t)n * 4 + 16, reinterpret_cast<void**>(&R.list0)))) return rc;
        SX_CUDA(ctx, cudaMemsetAsync(c.aln, 0, (size_t)n * 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(c.seg, 0, (size_t)n * 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(c.key, 0, (size_t)n * 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(o->status, 0, (size_t)n, st));
        k7_active_reads_kernel<<<std::max(1, std::min<int>((int)((n + 255) / 256), ctx->sm_count * 8)), 256, 0, st>>>(n, d->gate, R.list0, R.n + 2);
        SX_CUDA(ctx, cudaGetLastError());
        extra = 1;
    }

    k7_view v;
    v.b = *d;
    if (R.list0 && !getenv("SX_K7_NO_CLASS_SORT"))
    {
        // the active list regrouped by shape class (see k7_read_class)
        uint8_t* cls(nullptr);
        uint32_t *hist(nullptr), *list0b(nullptr);
        if ((rc = sx_ensure(ctx, 32, (size_t)n + 16, reinterpret_cast<void**>(&cls)))) return rc;
        if ((rc = sx_ensure(ctx, 33, (size_t)K7_N_CLASS * 4 + 16, reinterpret_cast<void**>(&hist)))) return rc;
        if ((rc = sx_ensure(ctx, 34, (size_t)n * 4 + 16, reinterpret_cast<void**>(&list0b)))) return rc;
        SX_CUDA(ctx, cudaMemsetAsync(hist, 0, (size_t)K7_N_CLASS * 4, st));
        const int gc(std::max(1, std::min<int>((int)((n + K7_CLS_THREADS * K7_CLS_ITEMS - 1) / (K7_CLS_THREADS * K7_CLS_ITEMS)), ctx->sm_count * 8)));
        k7_class_count_kernel<<<gc, K7_CLS_THREADS, 0, st>>>(v, read_region, R.list0, R.n + 2, cls, hist);
        SX_CUDA(ctx, cudaGetLastError());
        sx_regroup_scan_kernel<<<1, SX_RG_CLASSES, 0, st>>>(hist);
        SX_CUDA(ctx, cudaGetLastError());
        sx_regroup_scatter_kernel<<<gc, SX_RG_THREADS, 0, st>>>(R.list0, R.n + 2, cls, hist, list0b);
        SX_CUDA(ctx, cudaGetLastError());
        R.list0 = list0b;
        extra += 3;
    }
    local_kernel<<<(unsigned)blocks_local, K7_THREADS, 0, st>>>(v, read_region, o->status, R, c, L);
    SX_CUDA(ctx, cudaGetLastError());
    k7_search_arena_kernel<<<(unsigned)blocks1, K7_THREADS, 0, st>>>(v, arena1, per_thread1, maxA1, maxF, read_region, o->status, R, 1, two_levels ? 1 : 0, c, L);
    SX_CUDA(ctx, cudaGetLastError());
    if (two_levels)
    {
        k7_search_arena_kernel<<<(unsigned)blocks, K7_THREADS, 0, st>>>(v, arena, per_thread, maxA, maxF, read_region, o->status, R, 2, 0, c, L);
        SX_CUDA(ctx, cudaGetLastError());
    }
    k7_scan_tiles<<<n_tiles, K7_SCAN_THREADS, 0, st>>>(n, c.aln, c.seg, c.key, sums, n_tiles);
    SX_CUDA(ctx, cudaGetLastError());
    k7_scan_sums<<<1, K7_SCAN_THREADS, 0, st>>>(sums, n_tiles, totals);
    SX_CUDA(ctx, cudaGetLastError());
    k7_scan_finish<<<n_tiles, K7_SCAN_THREADS, 0, st>>>(n, c, sums, n_tiles, totals, *o, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    const int g1(std::max(1, std::min<int>((int)((n + 127) / 128), ctx->sm_count * 16)));
    k7_gather_kernel<<<g1, 128, 0, st>>>(n, c, L, *o, totals, nullptr, nullptr); // (every read, in read order: walking the active list instead, in read or class order, was slower)
    SX_CUDA(ctx, cudaGetLastError());
    *launches = (two_levels ? 8 : 7) + extra;
    return SX_OK;
}

int k7_check_args(sx_ctx* ctx, const sx_enum_batch* b, const sx_enum_out* o, const char* what)
{
    if (!b || !o) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (!o->totals || !o->aln_off) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    if (b->n_reads == 0) return SX_OK;
    if (!b->region_read_off || !b->region_key_off || !b->realign_begin || !b->realign_end || !b->in_pos || !b->in_seg_off || !b->in_segs || !b->in_key_off ||
        !b->use_key_off || !b->in_lead_key || !b->in_trail_key || !b->read_len || !o->status || !o->aln_pos || !o->aln_seg_off || !o->segs || !o->aln_key_off ||
        !o->aln_keys || !o->aln_lead_key || !o->aln_trail_key)
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL array", what);
    if ((b->n_keys && !b->keys) || b->n_regions == 0) return sx_fail(ctx, SX_ERR_ARG, "%s: reads without a region / keys without a table", what);
    if (b->opts.n_samples == 0 || b->opts.n_samples > SX_ENUM_MAX_SAMPLES || b->opts.sample_id >= b->opts.n_samples)
        return sx_fail(ctx, SX_ERR_ARG, "%s: n_samples outside 1..%d or sample_id outside the samples", what, SX_ENUM_MAX_SAMPLES);
    if (b->opts.n_max_toggle > 100) return sx_fail(ctx, SX_ERR_ARG, "%s: n_max_toggle above 100", what);
    if (b->opts.max_read_indel_toggle < 0 || b->opts.max_read_indel_toggle > 127) return sx_fail(ctx, SX_ERR_RANGE, "%s: max_read_indel_toggle outside 0..127", what);
    return SX_OK;
}

int k7_finish(sx_ctx* ctx, const char* what, const uint32_t* totals_host)
{
    int st(0);
    SX_CUDA(ctx, cudaMemcpyAsync(&st, ctx->d_status, sizeof(int), cudaMemcpyDeviceToHost, ctx->s_compute));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    if (st & (1 << K7_ST_SHIFT))
    {
        cudaMemsetAsync(ctx->d_status, 0, sizeof(int), ctx->s_compute);
        if (totals_host)
            return sx_fail(ctx, SX_ERR_CAPACITY, "%s: output capacity too small: the batch produces %u alignments, %u segments, %u keys", what, totals_host[0],
                           totals_host[1], totals_host[2]);
        return sx_fail(ctx, SX_ERR_CAPACITY, "%s: output capacity too small (totals[] holds the needed sizes)", what);
    }
    return sx_check_status(ctx, what);
}
} // namespace

extern "C" void sx_default_enum_opts(sx_enum_opts* o)
{
    if (!o) return;
    o->max_indel_size = 49;                 // starling_base_shared.hh:124
    o->max_read_indel_toggle = 5;           // :139
    o->max_candidate_indel_density = 0.15;  // :145
    // starling_align_limit(opt.max_realignment_candidates = 5000), starling_align_limit.cpp:77-88
    o->n_max_toggle = 0;
    for (unsigned i = 0; i < 100; ++i)
    {
        const unsigned mt(k7_max_candidate_alignment_toggle(i, 5000));
        if (i > 1 && mt < 2) break;
        o->max_toggle[o->n_max_toggle++] = (uint8_t)mt;
    }
    for (unsigned i = o->n_max_toggle; i < 100; ++i) o->max_toggle[i] = 1;
    o->is_haplotyping_enabled = 0;          // starling_base_shared.hh:99 (the germline workflow switches it on)
    o->n_samples = 1;
    o->sample_id = 0;
    o->max_alns_per_read = 64;
    o->flags = SX_ENUM_F_FAST; // the default launch plan; 0 = the two-pass arena plan
}

extern "C" int sx_enumerate_alignments_dev(sx_ctx* ctx, const sx_enum_batch* d, sx_enum_out* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k7_check_args(ctx, d, out_dev, "sx_enumerate_alignments_dev"))) return rc;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    if (d->n_reads == 0)
    {
        SX_CUDA(ctx, cudaMemsetAsync(out_dev->totals, 0, 12, ctx->s_compute));
        SX_CUDA(ctx, cudaMemsetAsync(out_dev->aln_off, 0, 4, ctx->s_compute));
        SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
        return SX_OK;
    }
    sx_kernel_timer t(ctx);
    unsigned launches(0);
    if ((rc = (d->opts.flags & SX_ENUM_F_FAST) ? k7_run_fast(ctx, d, out_dev, &launches) : k7_run(ctx, d, out_dev, &launches))) return rc;
    t.stop(launches);
    if ((rc = t.finish())) return rc;
    return k7_finish(ctx, "sx_enumerate_alignments", nullptr);
}

extern "C" int sx_enumerate_alignments(sx_ctx* ctx, const sx_enum_batch* b, sx_enum_out* out_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k7_check_args(ctx, b, out_host, "sx_enumerate_alignments"))) return rc;
    if (b->n_reads == 0)
    {
        out_host->totals[0] = out_host->totals[1] = out_host->totals[2] = 0;
        out_host->aln_off[0] = 0;
        return SX_OK;
    }
    if (b->region_read_off[b->n_regions] != b->n_reads || b->region_key_off[b->n_regions] != b->n_keys)
        return sx_fail(ctx, SX_ERR_ARG, "sx_enumerate_alignments: offset arrays do not end at n_reads / n_keys");
    for (uint32_t g = 0; g < b->n_regions; ++g)
        if (b->region_key_off[g + 1] - b->region_key_off[g] > 65535u) return sx_fail(ctx, SX_ERR_RANGE, "sx_enumerate_alignments: more than 65535 window entries in a region");
    for (uint32_t k = 0; k < b->n_keys; ++k)
        if (b->keys[k].type > SX_INDEL_TYPE_MISMATCH) return sx_fail(ctx, SX_ERR_UNSUPPORTED, "sx_enumerate_alignments: breakend entries are not supported");
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st(ctx->s_compute);
    SX_CUDA(ctx, cudaEventRecord(ctx->ev_a, st));
    sx_enum_batch d(*b);
    void* p(nullptr);
    const size_t n_segs(b->in_seg_off[b->n_reads]), n_ikeys(b->in_key_off[b->n_reads]), n_ukeys(b->use_key_off[b->n_reads]);
#define SX_UP(slot, field, type, bytes)                                                        \
    if ((rc = sx_ensure(ctx, slot, (size_t)(bytes) + 16, &p))) return rc;                       \
    if (bytes) SX_CUDA(ctx, cudaMemcpyAsync(p, b->field, (bytes), cudaMemcpyHostToDevice, st)); \
    d.field = static_cast<type>(p);
    SX_UP(0, region_read_off, const uint32_t*, (size_t)(b->n_regions + 1) * 4)
    SX_UP(1, region_key_off, const uint32_t*, (size_t)(b->n_regions + 1) * 4)
    SX_UP(2, keys, const sx_indel_key*, (size_t)b->n_keys * sizeof(sx_indel_key))
    if (b->key_hap)
    {
        SX_UP(3, key_hap, const sx_key_hap*, (size_t)b->n_keys * sizeof(sx_key_hap))
    }
    SX_UP(4, realign_begin, const int32_t*, (size_t)b->n_regions * 4)
    SX_UP(5, realign_end, const int32_t*, (size_t)b->n_regions * 4)
    SX_UP(6, in_pos, const int32_t*, (size_t)b->n_reads * 4)
    SX_UP(7, in_seg_off, const uint32_t*, (size_t)(b->n_reads + 1) * 4)
    SX_UP(8, in_segs, const sx_aln_seg*, n_segs * sizeof(sx_aln_seg))
    SX_UP(9, in_key_off, const uint32_t*, (size_t)(b->n_reads + 1) * 4)
    SX_UP(10, in_keys, const uint16_t*, n_ikeys * 2)
    SX_UP(11, use_key_off, const uint32_t*, (size_t)(b->n_reads + 1) * 4)
    SX_UP(12, use_keys, const uint16_t*, n_ukeys * 2)
    SX_UP(13, in_lead_key, const uint16_t*, (size_t)b->n_reads * 2)
    SX_UP(14, in_trail_key, const uint16_t*, (size_t)b->n_reads * 2)
    SX_UP(15, read_len, const uint16_t*, (size_t)b->n_reads * 2)
    if (b->gate)
    {
        SX_UP(26, gate, const uint8_t*, (size_t)b->n_reads)
    }
#undef SX_UP
    sx_enum_out o(*out_host);
    if ((rc = sx_ensure(ctx, 16, 16, reinterpret_cast<void**>(&o.totals)))) return rc;
    if ((rc = sx_ensure(ctx, 17, (size_t)(b->n_reads + 1) * 4, reinterpret_cast<void**>(&o.aln_off)))) return rc;
    if ((rc = sx_ensure(ctx, 18, (size_t)b->n_reads + 16, reinterpret_cast<void**>(&o.status)))) return rc;
    if ((rc = sx_ensure(ctx, 19, (size_t)o.cap_alns * 4 + 16, reinterpret_cast<void**>(&o.aln_pos)))) return rc;
    if ((rc = sx_ensure(ctx, 20, ((size_t)o.cap_alns + 1) * 4 + 16, reinterpret_cast<void**>(&o.aln_seg_off)))) return rc;
    if ((rc = sx_ensure(ctx, 21, (size_t)o.cap_segs * sizeof(sx_aln_seg) + 16, reinterpret_cast<void**>(&o.segs)))) return rc;
    if ((rc = sx_ensure(ctx, 22, ((size_t)o.cap_alns + 1) * 4 + 16, reinterpret_cast<void**>(&o.aln_key_off)))) return rc;
    if ((rc = sx_ensure(ctx, 23, (size_t)o.cap_keys * 2 + 16, reinterpret_cast<void**>(&o.aln_keys)))) return rc;
    if ((rc = sx_ensure(ctx, 24, (size_t)o.cap_alns * 2 + 16, reinterpret_cast<void**>(&o.aln_lead_key)))) return rc;
    if ((rc = sx_ensure(ctx, 25, (size_t)o.cap_alns * 2 + 16, reinterpret_cast<void**>(&o.aln_trail_key)))) return rc;
    unsigned launches(0);
    if ((rc = (d.opts.flags & SX_ENUM_F_FAST) ? k7_run_fast(ctx, &d, &o, &launches) : k7_run(ctx, &d, &o, &launches))) return rc;
    // the totals decide how much comes back
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->totals, o.totals, 12, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->aln_off, o.aln_off, (size_t)(b->n_reads + 1) * 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->status, o.status, (size_t)b->n_reads, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    const uint32_t nA(out_host->totals[0]), nS(out_host->totals[1]), nK(out_host->totals[2]);
    if (nA <= o.cap_alns && nS <= o.cap_segs && nK <= o.cap_keys)
    {
        SX_CUDA(ctx, cudaMemcpyAsync(out_host->aln_pos, o.aln_pos, (size_t)nA * 4, cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaMemcpyAsync(out_host->aln_seg_off, o.aln_seg_off, ((size_t)nA + 1) * 4, cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaMemcpyAsync(out_host->segs, o.segs, (size_t)nS * sizeof(sx_aln_seg), cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaMemcpyAsync(out_host->aln_key_off, o.aln_key_off, ((size_t)nA + 1) * 4, cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaMemcpyAsync(out_host->aln_keys, o.aln_keys, (size_t)nK * 2, cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaMemcpyAsync(out_host->aln_lead_key, o.aln_lead_key, (size_t)nA * 2, cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaMemcpyAsync(out_host->aln_trail_key, o.aln_trail_key, (size_t)nA * 2, cudaMemcpyDeviceToHost, st));
    }
    SX_CUDA(ctx, cudaEventRecord(ctx->ev_b, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    float ms(0);
    cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b);
    ctx->timing.kernel_ms = ms;
    ctx->timing.launches = launches;
    ctx->total_launches += launches;
    return k7_finish(ctx, "sx_enumerate_alignments", out_host->totals);
}

// asynchronous launcher for the device-resident pipeline (sx_pipeline.cu)
int sx_k7_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* o, unsigned* launches)
{
    unsigned l(0);
    const int rc((d->opts.flags & SX_ENUM_F_FAST) ? k7_run_fast(ctx, d, o, &l) : k7_run(ctx, d, o, &l));
    *launches += l;
    return rc;
}
