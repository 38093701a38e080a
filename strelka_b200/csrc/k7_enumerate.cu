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
//   scan            : three exclusive prefix sums over reads (sx_scan), the alignment offsets straight into aln_off
//   k7_write_kernel : search again (deterministic) -> the set, in its order, at the read's offsets
// Searching twice costs less than a second arena large enough to keep every read's set between the passes, and keeps the output
// independent of scheduling.  Persistent grid: resident blocks x SM count, a thread strides over reads.

#include "k7_core.cuh"
#include "sx_internal.h"
#include "sx_regroup.cuh"

#include <algorithm>
#include <cstdlib>

namespace
{
constexpr int K7_THREADS = 64;

struct k7_counts // per read, then (after the scan) its exclusive offsets
{
    uint32_t* aln; // the output's aln_off
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

// the scan's totals against the capacities: block 0 raises SX_ST_K7_CAP, or closes the per-alignment offset arrays
__device__ __forceinline__ bool k7_fits(const sx_enum_out& o, int* __restrict__ status)
{
    const bool fits(o.totals[0] <= o.cap_alns && o.totals[1] <= o.cap_segs && o.totals[2] <= o.cap_keys);
    if (blockIdx.x == 0 && threadIdx.x == 0)
    {
        if (!fits) atomicOr(status, SX_ST_K7_CAP);
        else
        {
            o.aln_seg_off[o.totals[0]] = o.totals[1];
            o.aln_key_off[o.totals[0]] = o.totals[2];
        }
    }
    return fits;
}

__global__ void __launch_bounds__(K7_THREADS) k7_write_kernel(const k7_view v, unsigned char* __restrict__ arena, const size_t per_thread, const uint32_t maxA,
                                                              const uint32_t maxF, const uint32_t* __restrict__ read_region, const uint8_t* __restrict__ status,
                                                              const k7_counts c, const sx_enum_out o, int* __restrict__ d_status)
{
    if (!k7_fits(o, d_status)) return;
    const uint32_t t(blockIdx.x * blockDim.x + threadIdx.x), nthr(gridDim.x * blockDim.x);
    k7_scratch S(k7_scratch_at(arena + (size_t)t * per_thread, maxA, maxF));
    for (uint32_t r = t; r < v.b.n_reads; r += nthr)
    {
        if (status[r] & (SX_ENUM_ST_EXCEPTION | SX_ENUM_ST_LIMIT)) continue;
        const uint32_t na(c.aln[r + 1] - c.aln[r]);
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
// The local tier holds 40 alignments: local memory a thread never touches costs nothing but address space, while every read the tier
// passes on is searched a second time from the start in the slower arena (DESIGN.md section 6 has the sweep over 16 / 40 alignments
// and 16 / 24 / 32 resident blocks per SM behind these constants).
constexpr uint32_t K7_LOCAL_ALNS = 40;
constexpr uint32_t K7_LOCAL_FRAMES = 12;
static_assert(K7_LOCAL_FRAMES <= K7_MAX_INDELS + 1, "local tier sizes");
constexpr uint32_t K7_LOCAL_BYTES = (uint32_t)((k7_scratch_bytes(K7_LOCAL_ALNS, K7_LOCAL_FRAMES) + 255) & ~(size_t)255); // one thread's local scratch
// 16 resident blocks per SM (64 registers; its state lives in local memory): on an H100, K7 103 vs 119 ms per step at 16 vs 24 (bench.py,
// 300k cfg2 loci, two runs each; H100 80GB HBM3, 400 W power limit) -- fewer resident threads keep the local scratch closer to the L2's size
constexpr int K7_LOCAL_MIN_BLOCKS = 16;
constexpr uint32_t K7_MID_ALNS = 96; // per-read capacity of the first arena tier

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

__global__ void __launch_bounds__(K7_THREADS, K7_LOCAL_MIN_BLOCKS) k7_search_local_kernel(const k7_view v, const uint32_t* __restrict__ read_region, uint8_t* __restrict__ status,
                                                                           const k7_retry R, const k7_counts c, const k7_log L)
{
    __align__(16) unsigned char local[K7_LOCAL_BYTES];
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

__global__ void k7_gather_kernel(const uint32_t n_reads, const k7_counts c, const k7_log L, const sx_enum_out o, int* __restrict__ d_status,
                                 const uint32_t* __restrict__ list, const uint32_t* __restrict__ n_list)
{
    if (!k7_fits(o, d_status)) return;
    // with a list (in read order: the CSR output is written in read order): only the searched reads have a blob
    const uint32_t n_work(list ? *n_list : n_reads);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_work; i += gridDim.x * blockDim.x)
    {
        const uint32_t r(list ? list[i] : i);
        const uint32_t na(c.aln[r + 1] - c.aln[r]);
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

// the per-read counts: alignments in the output's aln_off, segments and keys in the stage's scratch
int k7_take_counts(sx_ctx* ctx, const uint32_t n, const sx_enum_out* o, k7_counts* c)
{
    int rc;
    c->aln = o->aln_off;
    if ((rc = sx_take(ctx, SX_SLOT_K7_CNT_SEG, n, c->seg, 16))) return rc;
    return sx_take(ctx, SX_SLOT_K7_CNT_KEY, n, c->key, 16);
}

// counts -> exclusive offsets, aln_off[n] and the three totals
int k7_offsets(sx_ctx* ctx, const uint32_t n, const sx_enum_out* o, const k7_counts& c, unsigned* launches)
{
    const sx_scan_set J = {3,
                           {{c.aln, n, SX_SCAN_EXCLUSIVE | SX_SCAN_CLOSE, o->totals},
                            {c.seg, n, SX_SCAN_EXCLUSIVE, o->totals + 1},
                            {c.key, n, SX_SCAN_EXCLUSIVE, o->totals + 2}}};
    return sx_scan(ctx, SX_SLOT_K7_SUMS, J, launches);
}

int k7_plan_two_pass(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* o, unsigned* launches)
{
    cudaStream_t st(ctx->s_compute);
    const uint32_t n(d->n_reads);
    const uint32_t maxA(d->opts.max_alns_per_read ? std::min<uint32_t>(d->opts.max_alns_per_read, 65535u) : 64u);
    int rc;
    uint32_t* read_region(nullptr);
    if ((rc = sx_take(ctx, SX_SLOT_K7_READ_REGION, n, read_region, 32))) return rc;
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
    if ((rc = sx_take(ctx, SX_SLOT_K7_ARENA, blocks * K7_THREADS * per_thread, arena, 0))) return rc;
    k7_counts c;
    if ((rc = k7_take_counts(ctx, n, o, &c))) return rc;

    k7_view v;
    v.b = *d;
    k7_count_kernel<<<(unsigned)blocks, K7_THREADS, 0, st>>>(v, arena, per_thread, maxA, maxF, read_region, o->status, c);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 2; // (with the frame count)
    if ((rc = k7_offsets(ctx, n, o, c, launches))) return rc;
    k7_write_kernel<<<(unsigned)blocks, K7_THREADS, 0, st>>>(v, arena, per_thread, maxA, maxF, read_region, o->status, c, *o, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

int k7_plan_fast(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* o, unsigned* launches)
{
    cudaStream_t st(ctx->s_compute);
    const uint32_t n(d->n_reads);
    const uint32_t maxA(d->opts.max_alns_per_read ? std::min<uint32_t>(d->opts.max_alns_per_read, 65535u) : 64u);
    int rc;
    uint32_t* read_region(nullptr);
    if ((rc = sx_take(ctx, SX_SLOT_K7_READ_REGION, n, read_region, 32))) return rc;
    uint32_t maxF(K7_MAX_INDELS + 1);
    if ((rc = k7_frames_needed(ctx, d, read_region, read_region + n + 1, &maxF))) return rc; // (also fills read_region)
    const size_t per_thread((k7_scratch_bytes(maxA, maxF) + 255) & ~(size_t)255);
    int per_sm(1), per_sm_local(1);
    SX_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k7_search_arena_kernel, K7_THREADS, 0));
    SX_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_local, k7_search_local_kernel, K7_THREADS, 0));
    per_sm = std::max(1, per_sm);
    per_sm_local = std::max(1, per_sm_local);
    const size_t n_blocks(((size_t)n + K7_THREADS - 1) / K7_THREADS);
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
    if ((rc = sx_take(ctx, SX_SLOT_K7_ARENA, blocks1 * K7_THREADS * per_thread1, arena1, 0))) return rc;
    if (two_levels && (rc = sx_take(ctx, SX_SLOT_K7_ARENA_DEEP, blocks * K7_THREADS * per_thread, arena, 0))) return rc;
    k7_counts c;
    if ((rc = k7_take_counts(ctx, n, o, &c))) return rc;
    // the log holds whatever the output arrays can hold: 3 words + segments + ceil(keys / 2) words per alignment
    const unsigned long long want_words((unsigned long long)o->cap_alns * 4ull + o->cap_segs + (o->cap_keys + 1ull) / 2ull + 16ull);
    k7_log L;
    L.cap = (uint32_t)std::min<unsigned long long>(want_words, 0xFFFFFFF0ull);
    k7_retry R;
    if ((rc = sx_take(ctx, SX_SLOT_K7_LOG, L.cap, L.words, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K7_LOG_OFF, n, L.blob_off, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K7_LOG_CURSOR, 2, L.cursor, 0))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K7_RETRY1, n, R.list1, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K7_RETRY2, n, R.list2, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K7_RETRY_N, 4, R.n, 0))) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(L.cursor, 0, 16, st));
    SX_CUDA(ctx, cudaMemsetAsync(R.n, 0, 16, st));
    R.list0 = nullptr;
    unsigned extra(0);
    if (d->gate)
    {
        if ((rc = sx_take(ctx, SX_SLOT_K7_ACTIVE, n, R.list0, 16))) return rc;
        SX_CUDA(ctx, cudaMemsetAsync(c.aln, 0, (size_t)n * 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(c.seg, 0, (size_t)n * 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(c.key, 0, (size_t)n * 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(o->status, 0, (size_t)n, st));
        if ((rc = sx_k7_active_reads(ctx, n, d->gate, R.list0, R.n + 2))) return rc;
        extra = 1;
    }

    k7_view v;
    v.b = *d;
    if (R.list0 && !getenv("SX_K7_NO_CLASS_SORT"))
    {
        // the active list regrouped by shape class (see k7_read_class)
        uint8_t* cls(nullptr);
        uint32_t *hist(nullptr), *list0b(nullptr);
        if ((rc = sx_take(ctx, SX_SLOT_K7_CLASS, n, cls, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K7_HIST, K7_N_CLASS, hist, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K7_ACTIVE_BY_CLASS, n, list0b, 16))) return rc;
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
    k7_search_local_kernel<<<(unsigned)blocks_local, K7_THREADS, 0, st>>>(v, read_region, o->status, R, c, L);
    SX_CUDA(ctx, cudaGetLastError());
    k7_search_arena_kernel<<<(unsigned)blocks1, K7_THREADS, 0, st>>>(v, arena1, per_thread1, maxA1, maxF, read_region, o->status, R, 1, two_levels ? 1 : 0, c, L);
    SX_CUDA(ctx, cudaGetLastError());
    if (two_levels)
    {
        k7_search_arena_kernel<<<(unsigned)blocks, K7_THREADS, 0, st>>>(v, arena, per_thread, maxA, maxF, read_region, o->status, R, 2, 0, c, L);
        SX_CUDA(ctx, cudaGetLastError());
    }
    *launches += (two_levels ? 4 : 3) + extra; // (with the frame count)
    if ((rc = k7_offsets(ctx, n, o, c, launches))) return rc;
    const int g1(std::max(1, std::min<int>((int)((n + 127) / 128), ctx->sm_count * 16)));
    k7_gather_kernel<<<g1, 128, 0, st>>>(n, c, L, *o, ctx->d_status, nullptr, nullptr); // (every read, in read order: walking the active list instead, in read or class order, was slower)
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
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

} // namespace

// K7's launcher: the batch's options pick the launch plan
int sx_k7_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* o, unsigned* launches)
{
    return (d->opts.flags & SX_ENUM_F_FAST) ? k7_plan_fast(ctx, d, o, launches) : k7_plan_two_pass(ctx, d, o, launches);
}

int sx_k7_active_reads(sx_ctx* ctx, const uint32_t n_reads, const uint8_t* gate, uint32_t* list, uint32_t* count)
{
    k7_active_reads_kernel<<<std::max(1, std::min<int>((int)((n_reads + 255) / 256), ctx->sm_count * 8)), 256, 0, ctx->s_compute>>>(n_reads, gate, list, count);
    SX_CUDA(ctx, cudaGetLastError());
    return SX_OK;
}

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
    if (d->n_reads == 0)
    {
        SX_CUDA(ctx, cudaSetDevice(ctx->device));
        SX_CUDA(ctx, cudaMemsetAsync(out_dev->totals, 0, 12, ctx->s_compute));
        SX_CUDA(ctx, cudaMemsetAsync(out_dev->aln_off, 0, 4, ctx->s_compute));
        SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
        return SX_OK;
    }
    if ((rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k7_run(ctx, d, out_dev, launches); }))) return rc;
    return sx_check_status(ctx, "sx_enumerate_alignments", SX_ST_K7_CAP);
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
    sx_call_timer t(ctx);
    sx_enum_batch d(*b);
    const size_t n(b->n_reads), nr(b->n_regions), n_segs(b->in_seg_off[b->n_reads]), n_ikeys(b->in_key_off[b->n_reads]), n_ukeys(b->use_key_off[b->n_reads]);
    if ((rc = sx_upload(ctx, sx_host_slot(0), b->region_read_off, nr + 1, d.region_read_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(1), b->region_key_off, nr + 1, d.region_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(2), b->keys, b->n_keys, d.keys, 16))) return rc;
    if (b->key_hap && (rc = sx_upload(ctx, sx_host_slot(3), b->key_hap, b->n_keys, d.key_hap, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(4), b->realign_begin, nr, d.realign_begin, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(5), b->realign_end, nr, d.realign_end, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(6), b->in_pos, n, d.in_pos, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(7), b->in_seg_off, n + 1, d.in_seg_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(8), b->in_segs, n_segs, d.in_segs, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(9), b->in_key_off, n + 1, d.in_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(10), b->in_keys, n_ikeys, d.in_keys, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(11), b->use_key_off, n + 1, d.use_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(12), b->use_keys, n_ukeys, d.use_keys, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(13), b->in_lead_key, n, d.in_lead_key, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(14), b->in_trail_key, n, d.in_trail_key, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(15), b->read_len, n, d.read_len, 16))) return rc;
    if (b->gate && (rc = sx_upload(ctx, sx_host_slot(26), b->gate, n, d.gate, 16))) return rc;
    sx_enum_out o(*out_host);
    if ((rc = sx_take(ctx, sx_host_slot(16), 4, o.totals, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(17), n + 1, o.aln_off, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(18), n, o.status, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(19), o.cap_alns, o.aln_pos, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(20), (size_t)o.cap_alns + 1, o.aln_seg_off, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(21), o.cap_segs, o.segs, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(22), (size_t)o.cap_alns + 1, o.aln_key_off, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(23), o.cap_keys, o.aln_keys, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(24), o.cap_alns, o.aln_lead_key, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(25), o.cap_alns, o.aln_trail_key, 16))) return rc;
    unsigned launches(0);
    if ((rc = sx_k7_run(ctx, &d, &o, &launches))) return rc;
    // the totals decide how much comes back
    if ((rc = sx_download(ctx, out_host->totals, o.totals, 3))) return rc;
    if ((rc = sx_download(ctx, out_host->aln_off, o.aln_off, n + 1))) return rc;
    if ((rc = sx_download(ctx, out_host->status, o.status, n))) return rc;
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    const uint32_t nA(out_host->totals[0]), nS(out_host->totals[1]), nK(out_host->totals[2]);
    if (nA <= o.cap_alns && nS <= o.cap_segs && nK <= o.cap_keys)
    {
        if ((rc = sx_download(ctx, out_host->aln_pos, o.aln_pos, nA))) return rc;
        if ((rc = sx_download(ctx, out_host->aln_seg_off, o.aln_seg_off, (size_t)nA + 1))) return rc;
        if ((rc = sx_download(ctx, out_host->segs, o.segs, nS))) return rc;
        if ((rc = sx_download(ctx, out_host->aln_key_off, o.aln_key_off, (size_t)nA + 1))) return rc;
        if ((rc = sx_download(ctx, out_host->aln_keys, o.aln_keys, nK))) return rc;
        if ((rc = sx_download(ctx, out_host->aln_lead_key, o.aln_lead_key, nA))) return rc;
        if ((rc = sx_download(ctx, out_host->aln_trail_key, o.aln_trail_key, nA))) return rc;
    }
    if ((rc = t.finish(launches))) return rc;
    return sx_check_status(ctx, "sx_enumerate_alignments", SX_ST_K7_CAP, out_host->totals);
}
