// k6_lists.cuh -- the list builder of K6b and K6g: K6's read-major sx_read_indel_score records regrouped into lists sorted by read id, in
// device memory.  Included by k6b_indel_reads.cu and k6g_allele_groups.cu; device-only (the CPU tests mirror it in tests/cpp/k6_lists_host.h).
//
// A link's records go to its owners through the view's id -> owner table (k6b_view::locus_of): K6b's owners are its loci and it has two
// samples, K6g's are the ids some allele group names (locus_of[x] = x) and it has one.  Owner o's list of sample s is the segment
// Hook::n_samples * o + s.
//   k6l_count_kernel    one thread per read of either sample: integer atomics on cnt[segment], and the 64-bit total of what they add
//   scan                -> off, copied to the scatter's cursors; one 12-byte round trip sizes the triples (and refuses more than 2^32 - 1)
//   k6l_scatter_kernel  (read id, record, read) triples at atomic cursors: the order inside a segment is arbitrary here
//   k6l_sort_kernel     one warp per owner: each segment sorted by read id (k6b_sort_by_key, in shared memory up to K6L_SMEM_SORT entries, in
//                       the scratch itself beyond -- no depth cap), the sorted ids left in place and `order` beside them; equal neighbours
//                       = a duplicate id.  The link's hook sees each segment, then the owner's end with the duplicate flag.
// Read ids of an unflagged segment are distinct, so the sorted order -- and every byte a link writes from it -- is the same whatever order
// the atomics ran in.
#pragma once

#include "k6b_core.cuh"
#include "sx_internal.h"

#include <algorithm>

constexpr int K6L_THREADS = 128;
constexpr int K6L_WARPS = K6L_THREADS / 32;
constexpr uint32_t K6L_SMEM_SORT = 512; // entries of one segment sorted in shared memory: 4 KiB per warp

struct k6l_pairs // the scatter's output, segment i at off[i]
{
    uint32_t* id;    // read id, sorted in place by k6l_sort_kernel
    uint32_t* rec;   // record index in the sample's recs
    uint32_t* read;  // read index in the sample
    uint32_t* order; // order[p] = which of the segment's triples is p-th by read id
};

inline unsigned k6l_grid(const sx_ctx* ctx, const uint32_t m, const uint32_t per)
{
    return (unsigned)std::max(1, std::min<int>((int)((m + per - 1) / per), ctx->sm_count * 16));
}

// `total` is the 64-bit count of what the 32-bit counts and their scan hold: the launcher refuses a batch whose entries do not fit 32 bits
template <uint32_t NS>
__global__ void __launch_bounds__(K6L_THREADS) k6l_count_kernel(const k6b_view v, uint32_t* __restrict__ cnt, unsigned long long* __restrict__ total, int* __restrict__ status)
{
    const uint32_t n0(v.s[0].n_reads), n(n0 + v.s[1].n_reads);
    uint32_t st(0);
    unsigned long long mine(0);
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x)
    {
        const uint32_t sample(t < n0 ? 0u : 1u);
        st |= k6b_for_each_entry(v, sample, t - (sample ? n0 : 0u), [&](const uint32_t o, uint32_t) {
            atomicAdd(cnt + NS * o + sample, 1u);
            ++mine;
        });
    }
    for (int d = 16; d > 0; d >>= 1) mine += __shfl_down_sync(0xffffffffu, mine, d);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(total, mine);
    if (st) atomicOr(status, SX_ST_K6B_ID);
}

template <uint32_t NS> __global__ void __launch_bounds__(K6L_THREADS) k6l_scatter_kernel(const k6b_view v, uint32_t* __restrict__ cursor, const k6l_pairs P)
{
    const uint32_t n0(v.s[0].n_reads), n(n0 + v.s[1].n_reads);
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < n; t += gridDim.x * blockDim.x)
    {
        const uint32_t sample(t < n0 ? 0u : 1u), r(t - (sample ? n0 : 0u));
        const uint32_t id(k6b_read_id(v.s[sample], r));
        k6b_for_each_entry(v, sample, r, [&](const uint32_t o, const uint32_t i) {
            const uint32_t at(atomicAdd(cursor + NS * o + sample, 1u));
            P.id[at] = id;
            P.rec[at] = i;
            P.read[at] = r;
        });
    }
}

// One warp per owner.  Hook (a link's) has n_samples, a per-warp shared struct warp_smem, and the warp-wide calls
//   begin(ws, lane)                                 before the owner's first segment
//   segment(ws, owner, sample, base, n, P, lane)    after a segment is sorted (positions base .. base + n of P); returns the status bits
//                                                   of the ids it looked up (K6B_ST_BAD_ID, raised as SX_ST_K6B_ID like the count's)
//   end(ws, owner, dup, off, lane)                  dup: a read id twice in one of the owner's segments
template <typename Hook>
__global__ void __launch_bounds__(K6L_THREADS) k6l_sort_kernel(const uint32_t n_owners, const uint32_t* __restrict__ off, const k6l_pairs P, const Hook hook,
                                                               int* __restrict__ status)
{
    __shared__ uint32_t s_key[K6L_WARPS][K6L_SMEM_SORT], s_val[K6L_WARPS][K6L_SMEM_SORT];
    __shared__ typename Hook::warp_smem s_hook[K6L_WARPS];
    const uint32_t lane(threadIdx.x & 31), warp(threadIdx.x >> 5);
    const auto sync = [] { __syncwarp(); };
    uint32_t bad(0);
    for (uint32_t x = blockIdx.x * K6L_WARPS + warp; x < n_owners; x += gridDim.x * K6L_WARPS)
    {
        hook.begin(s_hook[warp], lane);
        bool dup(false);
        for (uint32_t sample = 0; sample < Hook::n_samples; ++sample)
        {
            const uint32_t base(off[Hook::n_samples * x + sample]), n(off[Hook::n_samples * x + sample + 1] - base);
            const uint32_t* key(P.id + base);
            if (n <= K6L_SMEM_SORT)
            {
                for (uint32_t i = lane; i < n; i += 32)
                {
                    s_key[warp][i] = P.id[base + i];
                    s_val[warp][i] = i;
                }
                __syncwarp();
                k6b_sort_by_key(s_key[warp], s_val[warp], n, lane, 32u, sync);
                for (uint32_t i = lane; i < n; i += 32)
                {
                    P.id[base + i] = s_key[warp][i];
                    P.order[base + i] = s_val[warp][i];
                }
                key = s_key[warp];
            }
            else
            {
                for (uint32_t i = lane; i < n; i += 32) P.order[base + i] = i;
                __syncwarp();
                k6b_sort_by_key(P.id + base, P.order + base, n, lane, 32u, sync);
            }
            for (uint32_t i = lane; i + 1 < n; i += 32) dup |= key[i] == key[i + 1];
            bad |= hook.segment(s_hook[warp], x, sample, base, n, P, lane);
            __syncwarp(); // s_key is loaded again for the next segment
        }
        hook.end(s_hook[warp], x, __any_sync(0xffffffffu, dup), off, lane);
    }
    if (bad) atomicOr(status, SX_ST_K6B_ID);
}

// The builder's scratch in the SX_SLOT_K6L_* buffers: the segments' offsets (Hook::n_samples * n_owners + 1) and the sorted triples
struct k6l_lists
{
    const uint32_t* off;
    k6l_pairs P;
};

// The lists of the records `v` walks, for the n_owners owners of v.locus_of (filled by the link before this on the compute stream); the sort
// kernel runs `hook`.  Enqueued on the compute stream with one round trip (the triples' total).
template <typename Hook> int k6l_build(sx_ctx* ctx, const char* what, const k6b_view& v, const uint32_t n_owners, const Hook& hook, k6l_lists* L, unsigned* launches)
{
    constexpr uint32_t NS(Hook::n_samples);
    cudaStream_t st(ctx->s_compute);
    const uint32_t n_seg(NS * n_owners), n_reads(v.s[0].n_reads + v.s[1].n_reads);
    uint32_t *off(nullptr), *cursor(nullptr);
    unsigned long long* total64(nullptr);
    int rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6L_OFF, (size_t)n_seg + 1, off, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6L_CURSOR, n_seg, cursor, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6L_TOTAL64, 1, total64, 0))) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(off, 0, (size_t)n_seg * 4, st));
    SX_CUDA(ctx, cudaMemsetAsync(total64, 0, 8, st));
    k6l_count_kernel<NS><<<k6l_grid(ctx, n_reads, K6L_THREADS), K6L_THREADS, 0, st>>>(v, off, total64, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    const sx_scan_set segs = {1, {{off, n_seg, SX_SCAN_EXCLUSIVE | SX_SCAN_CLOSE, nullptr}}};
    if ((rc = sx_scan(ctx, SX_SLOT_K6L_SUMS, segs, launches))) return rc;
    SX_CUDA(ctx, cudaMemcpyAsync(cursor, off, (size_t)n_seg * 4, cudaMemcpyDeviceToDevice, st));
    uint32_t n_pairs(0);
    unsigned long long n_pairs64(0);
    SX_CUDA(ctx, cudaMemcpyAsync(&n_pairs, off + n_seg, 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(&n_pairs64, total64, 8, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    if (n_pairs64 != n_pairs) return sx_fail(ctx, SX_ERR_RANGE, "%s: %llu list entries: the offsets are 32-bit", what, n_pairs64);

    k6l_pairs P;
    if ((rc = sx_take(ctx, SX_SLOT_K6L_ID, n_pairs, P.id, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6L_REC, n_pairs, P.rec, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6L_READ, n_pairs, P.read, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6L_ORDER, n_pairs, P.order, 16))) return rc;
    k6l_scatter_kernel<NS><<<k6l_grid(ctx, n_reads, K6L_THREADS), K6L_THREADS, 0, st>>>(v, cursor, P);
    SX_CUDA(ctx, cudaGetLastError());
    k6l_sort_kernel<Hook><<<k6l_grid(ctx, n_owners, K6L_WARPS), K6L_THREADS, 0, st>>>(n_owners, off, P, hook, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 2;
    *L = k6l_lists{off, P};
    return SX_OK;
}

// The body of a link's _dev entry: `run(launches)` under sx_run_timed.  The timer finishes whatever the link returns, since its totals stand
// even when a capacity is too small; then the link's own status bits (`own`) outrank SX_ERR_CAPACITY: a bad id or group may have inflated it.
template <typename F> int k6l_link_dev(sx_ctx* ctx, const char* what, const int own, F&& run)
{
    bool ran(false);
    int rc_link(SX_OK);
    const int rc(sx_run_timed(ctx, [&](unsigned* launches) {
        ran = true;
        rc_link = run(launches);
        return SX_OK;
    }));
    if (!ran) return rc; // (the device could not be set)
    if (rc_link == SX_ERR_CAPACITY || rc_link == SX_OK)
    {
        const int rc_st(sx_check_status(ctx, what, own));
        if (rc_st) return rc_st;
    }
    return rc_link ? rc_link : rc;
}
