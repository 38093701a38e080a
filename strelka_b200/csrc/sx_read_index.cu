// sx_read_index.cu -- the read index: each read's region and the byte offsets of its packed bases and qualities, in one pass.
//
// A warp per region walks the region's reads 32 at a time: a lane per read, the byte offsets by a warp scan of the reads' sizes from the
// region's seq_off / qual_off (reads of a region back to back, each on a byte boundary).  The window pass builds it once and hands it to K7g,
// K7a, K7b and K9 (and reads the per-read facts only it needs -- 'N' counts, buffer positions, pin bits -- off the offsets, sx_pipeline.cu);
// the entry points of K7a and K7b, which have no window pass in front of them, build the part they read with the same kernel.

#include "sx_internal.h"

#include <algorithm>
#include <cstring>

namespace
{
__global__ void __launch_bounds__(128) sx_read_index_kernel(const sx_read_index_in in, const sx_read_index o)
{
    const uint32_t lane(threadIdx.x & 31u), n_warps((gridDim.x * blockDim.x) >> 5);
    for (uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; g < in.n_regions; g += n_warps)
    {
        const uint32_t r0(in.region_read_off[g]), r1(in.region_read_off[g + 1]);
        unsigned long long sb(in.regions ? in.regions[g].seq_off : 0ull), qb(in.regions ? in.regions[g].qual_off : 0ull);
        for (uint32_t base = r0; base < r1; base += 32)
        {
            const uint32_t r(base + lane);
            const bool live(r < r1);
            const uint32_t len(live && in.read_len ? in.read_len[r] : 0u), packed((len + 1u) / 2u), qbytes(in.qual_bits == 4 ? packed : len);
            uint32_t s_inc(packed), q_inc(qbytes); // inclusive scans of the 32 reads' sizes
            for (uint32_t d = 1; d < 32; d <<= 1)
            {
                const uint32_t s(__shfl_up_sync(0xffffffffu, s_inc, d)), q(__shfl_up_sync(0xffffffffu, q_inc, d));
                if (lane >= d)
                {
                    s_inc += s;
                    q_inc += q;
                }
            }
            if (live)
            {
                const unsigned long long so(sb + s_inc - packed), qo(qb + q_inc - qbytes);
                if (o.region) o.region[r] = g;
                if (o.seq_off) o.seq_off[r] = (uint32_t)so;
                if (o.qual_off) o.qual_off[r] = (uint32_t)qo;
            }
            sb += __shfl_sync(0xffffffffu, s_inc, 31);
            qb += __shfl_sync(0xffffffffu, q_inc, 31);
        }
        if (g + 1 == in.n_regions && lane == 0)
        {
            if (o.seq_off) o.seq_off[in.n_reads] = (uint32_t)sb;
            if (o.qual_off) o.qual_off[in.n_reads] = (uint32_t)qb;
        }
    }
}
} // namespace

int sx_read_index_run(sx_ctx* ctx, const sx_read_index_in* in, const sx_read_index* o, unsigned* launches)
{
    if (in->n_reads == 0 || in->n_regions == 0) return SX_OK;
    const unsigned grid((unsigned)std::max(1, std::min<int>((int)((in->n_regions + 3) / 4), ctx->sm_count * 16))); // 4 warps a block
    sx_read_index_kernel<<<grid, 128, 0, ctx->s_compute>>>(*in, *o);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

int sx_read_region_run(sx_ctx* ctx, const uint32_t n_regions, const uint32_t n_reads, const uint32_t* region_read_off, uint32_t* region, unsigned* launches)
{
    sx_read_index_in in;
    memset(&in, 0, sizeof(in));
    in.n_regions = n_regions;
    in.n_reads = n_reads;
    in.region_read_off = region_read_off;
    sx_read_index o;
    memset(&o, 0, sizeof(o));
    o.region = region;
    return sx_read_index_run(ctx, &in, &o, launches);
}
