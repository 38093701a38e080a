// sx_scan.cu -- in-place prefix sums of 1..SX_SCAN_MAX uint32 arrays: how every stage turns per-item counts into CSR offsets.
//
// Reduce-then-scan in three launches, the arrays side by side on blockIdx.y (a tile past an array's end returns at once):
//   sx_scan_reduce_kernel  each SX_SCAN_TILE-element tile's sum
//   sx_scan_carry_kernel   one block per array: exclusive scan of its tile sums, SX_SCAN_THREADS of them per round; the total to
//                          data[n] (SX_SCAN_CLOSE) and to *total
//   sx_scan_tiles_kernel   each tile scanned from its carry-in, the final values written in place
// Every element is read twice and written once.  Unsigned addition wraps, so an int array passed as uint32_t scans to the same bits.
#include "sx_internal.h"

#include <algorithm>

namespace
{
constexpr uint32_t PER = SX_SCAN_TILE / SX_SCAN_THREADS; // consecutive elements per thread in the last pass
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ uint32_t tiles_of(const uint32_t n) { return (n + SX_SCAN_TILE - 1) / SX_SCAN_TILE; }

// inclusive scan across the block's SX_SCAN_THREADS threads (warp_sums: SX_SCAN_THREADS / 32 words of shared memory)
__device__ __forceinline__ uint32_t block_scan_incl(uint32_t v, uint32_t* warp_sums)
{
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1)
    {
        const uint32_t y = __shfl_up_sync(FULL, v, d);
        if (lane >= (uint32_t)d) v += y;
    }
    if (lane == 31) warp_sums[wid] = v;
    __syncthreads();
    if (wid == 0)
    {
        uint32_t s = lane < SX_SCAN_THREADS / 32 ? warp_sums[lane] : 0;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1)
        {
            const uint32_t y = __shfl_up_sync(FULL, s, d);
            if (lane >= (uint32_t)d) s += y;
        }
        if (lane < SX_SCAN_THREADS / 32) warp_sums[lane] = s;
    }
    __syncthreads();
    if (wid > 0) v += warp_sums[wid - 1];
    return v;
}

__global__ void __launch_bounds__(SX_SCAN_THREADS) sx_scan_reduce_kernel(const sx_scan_set J, uint32_t* __restrict__ sums, const uint32_t tiles_per_array)
{
    const sx_scan_array& A = J.a[blockIdx.y];
    const uint32_t base = blockIdx.x * SX_SCAN_TILE;
    if (base >= A.n) return;
    uint32_t s = 0;
    for (uint32_t i = base + threadIdx.x; i < min(base + SX_SCAN_TILE, A.n); i += SX_SCAN_THREADS) s += A.data[i];
    __shared__ uint32_t ws[SX_SCAN_THREADS / 32];
    const uint32_t incl = block_scan_incl(s, ws);
    if (threadIdx.x == SX_SCAN_THREADS - 1) sums[blockIdx.y * tiles_per_array + blockIdx.x] = incl;
}

__global__ void __launch_bounds__(SX_SCAN_THREADS) sx_scan_carry_kernel(const sx_scan_set J, uint32_t* __restrict__ sums, const uint32_t tiles_per_array)
{
    const sx_scan_array& A = J.a[blockIdx.x];
    uint32_t* s = sums + blockIdx.x * tiles_per_array;
    const uint32_t nt = tiles_of(A.n);
    __shared__ uint32_t ws[SX_SCAN_THREADS / 32];
    __shared__ uint32_t carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (uint32_t b = 0; b < nt; b += SX_SCAN_THREADS)
    {
        const uint32_t i = b + threadIdx.x;
        const uint32_t v = i < nt ? s[i] : 0;
        const uint32_t incl = block_scan_incl(v, ws);
        const uint32_t carry = carry_s;
        if (i < nt) s[i] = carry + incl - v; // the tile's carry-in
        __syncthreads();
        if (threadIdx.x == SX_SCAN_THREADS - 1) carry_s = carry + incl;
        __syncthreads();
    }
    if (threadIdx.x == 0)
    {
        if (A.flags & SX_SCAN_CLOSE) A.data[A.n] = carry_s;
        if (A.total) *A.total = carry_s;
    }
}

__global__ void __launch_bounds__(SX_SCAN_THREADS) sx_scan_tiles_kernel(const sx_scan_set J, const uint32_t* __restrict__ sums, const uint32_t tiles_per_array)
{
    const sx_scan_array& A = J.a[blockIdx.y];
    const uint32_t base = blockIdx.x * SX_SCAN_TILE, n = A.n;
    if (base >= n) return;
    __shared__ uint32_t ws[SX_SCAN_THREADS / 32];
    const uint32_t carry = sums[blockIdx.y * tiles_per_array + blockIdx.x];
    const bool exclusive = (A.flags & SX_SCAN_EXCLUSIVE) != 0;
    uint32_t v[PER];
    uint32_t s = 0;
    const uint32_t i0 = base + threadIdx.x * PER;
#pragma unroll
    for (uint32_t e = 0; e < PER; ++e)
    {
        v[e] = (i0 + e) < n ? A.data[i0 + e] : 0;
        s += v[e];
    }
    uint32_t run = carry + block_scan_incl(s, ws) - s;
#pragma unroll
    for (uint32_t e = 0; e < PER; ++e)
    {
        const uint32_t out = exclusive ? run : run + v[e];
        run += v[e];
        if ((i0 + e) < n) A.data[i0 + e] = out;
    }
}
} // namespace

int sx_scan(sx_ctx* ctx, const sx_slot sums_slot, const sx_scan_set& J, unsigned* launches)
{
    if (J.n_arrays < 1 || J.n_arrays > SX_SCAN_MAX) return sx_fail(ctx, SX_ERR_ARG, "sx_scan: %d arrays, not 1..%d", J.n_arrays, SX_SCAN_MAX);
    uint32_t n_max = 0;
    for (int k = 0; k < J.n_arrays; ++k) n_max = std::max(n_max, J.a[k].n);
    const uint32_t tiles = std::max(1u, (n_max + SX_SCAN_TILE - 1) / SX_SCAN_TILE);
    uint32_t* sums = nullptr;
    int rc;
    if ((rc = sx_take(ctx, sums_slot, (size_t)tiles * J.n_arrays, sums, 0))) return rc;
    cudaStream_t st = ctx->s_compute;
    const dim3 grid(tiles, J.n_arrays);
    sx_scan_reduce_kernel<<<grid, SX_SCAN_THREADS, 0, st>>>(J, sums, tiles);
    sx_scan_carry_kernel<<<J.n_arrays, SX_SCAN_THREADS, 0, st>>>(J, sums, tiles);
    sx_scan_tiles_kernel<<<grid, SX_SCAN_THREADS, 0, st>>>(J, sums, tiles);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 3;
    return SX_OK;
}
