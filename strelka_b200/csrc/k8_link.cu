// k8_link.cu -- K7b link_alignments: K7's candidate alignments -> the alignment part of K1's batch, in device memory.
//
// Replaces (include/strelka_b200.h, "K7b link_alignments") the per-alignment host work in front of K1: the segment walk of
// scoreCandidateAlignment (starling_common/starling_read_align_score.cpp:289-499) with getMatchingIndelKey :177-224, the insert
// sequence / leading-edge tail rule :334-338, :394-398 and the candidacy look-up :473-475 resolved.  Per-alignment body: k8_core.cuh.
//
// Shape of the work: a streaming relabel -- every K7 segment is read once, every K1 segment and insert byte written once; the only
// structure is K1's staging rule (each region's first segment a multiple of 8, its first insert byte a multiple of 16), which turns
// the offsets into a two-level prefix sum: within a region (one thread per region walks its alignments' sizes) and over regions
// (sx_scan3.cuh).  Launches: sizes (thread per alignment) -> region sums -> scan -> write (thread per alignment) + region records.

#include "k8_core.cuh"
#include "sx_internal.h"
#include "sx_scan3.cuh"

#include <algorithm>

namespace
{
constexpr int K8_ST_SHIFT = 15;      // device status bits 32768 (no key) / 65536 (segment kind)
constexpr int K8_CAP_BIT = 1 << 17;  // an output capacity is too small

// alignment -> read (K7 lists a read's alignments consecutively)
__global__ void k8_aln_read_kernel(const uint32_t n_reads, const uint32_t* __restrict__ aln_off, uint32_t* __restrict__ aln_read)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n_reads; r += gridDim.x * blockDim.x)
        for (uint32_t a = aln_off[r]; a < aln_off[r + 1]; ++a) aln_read[a] = r;
}

__global__ void k8_read_region_kernel(const uint32_t n_regions, const uint32_t* __restrict__ region_read_off, uint32_t* __restrict__ read_region)
{
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < n_regions; g += gridDim.x * blockDim.x)
        for (uint32_t r = region_read_off[g]; r < region_read_off[g + 1]; ++r) read_region[r] = g;
}

__global__ void k8_size_kernel(const k8_view v, const uint32_t n_alns, const uint32_t* __restrict__ aln_read, const uint32_t* __restrict__ read_region,
                               uint32_t* __restrict__ seg_n, uint32_t* __restrict__ ins_n, int* __restrict__ status)
{
    uint32_t st(0);
    for (uint32_t a = blockIdx.x * blockDim.x + threadIdx.x; a < n_alns; a += gridDim.x * blockDim.x)
    {
        uint32_t ns, ni;
        st |= k8_walk(v, read_region[aln_read[a]], a, ns, ni, nullptr, nullptr);
        seg_n[a] = ns;
        ins_n[a] = ni;
    }
    if (st) atomicOr(status, (int)(st << K8_ST_SHIFT));
}

// per region: exclusive offsets of its alignments within the region (in place) and the region's padded totals.  One WARP per region: a region
// of a 30x window holds a few hundred alignments, and one thread walking them was most of the link's time
__global__ void k8_region_kernel(const k8_view v, uint32_t* __restrict__ seg_n, uint32_t* __restrict__ ins_n, uint32_t* __restrict__ reg_seg,
                                 uint32_t* __restrict__ reg_ins, uint32_t* __restrict__ reg_zero)
{
    const uint32_t lane(threadIdx.x & 31u), wpb(blockDim.x >> 5);
    for (uint32_t g = blockIdx.x * wpb + (threadIdx.x >> 5); g < v.b.n_regions; g += gridDim.x * wpb)
    {
        const uint32_t a0(v.e.aln_off[v.b.region_read_off[g]]), a1(v.e.aln_off[v.b.region_read_off[g + 1]]);
        uint32_t s(0), n(0);
        for (uint32_t b = a0; b < a1; b += 32)
        {
            const uint32_t a(b + lane);
            const uint32_t ds(a < a1 ? seg_n[a] : 0u), dn(a < a1 ? ins_n[a] : 0u);
            uint32_t is(ds), in(dn);
#pragma unroll
            for (uint32_t d = 1; d < 32; d <<= 1)
            {
                const uint32_t t(__shfl_up_sync(0xffffffffu, is, d)), u(__shfl_up_sync(0xffffffffu, in, d));
                if (lane >= d)
                {
                    is += t;
                    in += u;
                }
            }
            if (a < a1)
            {
                seg_n[a] = s + is - ds;
                ins_n[a] = n + in - dn;
            }
            s += __shfl_sync(0xffffffffu, is, 31);
            n += __shfl_sync(0xffffffffu, in, 31);
        }
        if (lane == 0)
        {
            reg_seg[g] = (s + 7u) & ~7u;
            reg_ins[g] = (n + 15u) & ~15u;
            reg_zero[g] = 0;
        }
    }
}

// region offsets after the scan; region records; capacity check; sentinels
__global__ void __launch_bounds__(K7_SCAN_THREADS) k8_finish_kernel(const k8_view v, const uint32_t n_alns, uint32_t* __restrict__ reg_seg, uint32_t* __restrict__ reg_ins,
                                                                   const uint32_t* __restrict__ sums, const uint32_t n_tiles, const uint32_t* __restrict__ totals,
                                                                   const sx_link_out o, int* __restrict__ status)
{
    const uint32_t n(v.b.n_regions), tile(blockIdx.x);
    const uint32_t base(tile * K7_SCAN_THREADS * K7_SCAN_ITEMS + threadIdx.x * K7_SCAN_ITEMS);
    const uint32_t os(sums[tile]), on(sums[(size_t)n_tiles + tile]);
    for (int i = 0; i < K7_SCAN_ITEMS; ++i)
        if (base + i < n)
        {
            const uint32_t g(base + i);
            const uint32_t s(reg_seg[g] + os), b(reg_ins[g] + on);
            reg_seg[g] = s;
            reg_ins[g] = b;
            o.regions[g].aln_begin = v.e.aln_off[v.b.region_read_off[g]];
            o.regions[g].seg_begin = s;
            o.regions[g].ins_begin = b;
        }
    if (blockIdx.x == 0 && threadIdx.x == 0)
    {
        o.totals[0] = totals[0];
        o.totals[1] = totals[1];
        o.regions[n].aln_begin = n_alns;
        o.regions[n].seg_begin = totals[0];
        o.regions[n].ins_begin = totals[1];
        o.regions[n].read_begin = v.b.n_reads;
        if (totals[0] > o.cap_segs || totals[1] > o.cap_ins) atomicOr(status, K8_CAP_BIT);
        else o.alns[n_alns] = sx_aln{v.b.n_reads, 0, totals[0], totals[1]};
    }
}

__global__ void k8_write_kernel(const k8_view v, const uint32_t n_alns, const uint32_t* __restrict__ aln_read, const uint32_t* __restrict__ read_region,
                                const uint32_t* __restrict__ seg_rel, const uint32_t* __restrict__ ins_rel, const uint32_t* __restrict__ reg_seg,
                                const uint32_t* __restrict__ reg_ins, const uint32_t* __restrict__ totals, const sx_link_out o)
{
    if (totals[0] > o.cap_segs || totals[1] > o.cap_ins) return; // reported by k8_finish_kernel
    for (uint32_t a = blockIdx.x * blockDim.x + threadIdx.x; a < n_alns; a += gridDim.x * blockDim.x)
    {
        const uint32_t r(aln_read[a]), g(read_region[r]);
        const uint32_t s(reg_seg[g] + seg_rel[a]), b(reg_ins[g] + ins_rel[a]);
        o.alns[a] = sx_aln{r, v.e.aln_pos[a], s, b};
        uint32_t ns, ni;
        k8_walk(v, g, a, ns, ni, o.segs + s, o.ins + b);
        if (o.k6_segs)
            for (uint32_t q = v.e.aln_seg_off[a]; q < v.e.aln_seg_off[a + 1]; ++q) o.k6_segs[q] = sx_aln_seg{v.e.segs[q].len, k8_k6_kind(v.e.segs[q].kind), 0};
    }
}

// the pads between a region's last used segment / insert byte and the next region's first
__global__ void k8_pad_kernel(const k8_view v, const uint32_t* __restrict__ seg_rel, const uint32_t* __restrict__ ins_rel, const uint32_t* __restrict__ reg_seg,
                              const uint32_t* __restrict__ reg_ins, const uint32_t* __restrict__ totals, const sx_link_out o)
{
    if (totals[0] > o.cap_segs || totals[1] > o.cap_ins) return;
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < v.b.n_regions; g += gridDim.x * blockDim.x)
    {
        const uint32_t a0(v.e.aln_off[v.b.region_read_off[g]]), a1(v.e.aln_off[v.b.region_read_off[g + 1]]);
        const uint32_t seg_end(g + 1 < v.b.n_regions ? reg_seg[g + 1] : totals[0]), ins_end(g + 1 < v.b.n_regions ? reg_ins[g + 1] : totals[1]);
        uint32_t s(reg_seg[g]), b(reg_ins[g]);
        if (a1 > a0) // the end of the region's last alignment
        {
            uint32_t ns, ni;
            k8_walk(v, g, a1 - 1, ns, ni, nullptr, nullptr);
            s += seg_rel[a1 - 1] + ns;
            b += ins_rel[a1 - 1] + ni;
        }
        for (; s < seg_end; ++s) o.segs[s] = sx_aln_seg{0, SX_SEG_HARDCLIP, 0};
        for (; b < ins_end; ++b) o.ins[b] = 0;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) // K1 loads 16-byte slices: up to 16 no-op segments of slack after the last one, where they fit
        for (uint32_t s = totals[0]; s < o.cap_segs && s < totals[0] + 16u; ++s) o.segs[s] = sx_aln_seg{0, SX_SEG_HARDCLIP, 0};
}

int k8_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* e, const uint32_t n_alns, const uint32_t* key_ins_off, const char* key_ins, const sx_link_out* o,
           unsigned* launches)
{
    cudaStream_t st(ctx->s_compute);
    int rc;
    uint32_t *aln_read(nullptr), *read_region(nullptr), *seg_n(nullptr), *ins_n(nullptr), *reg_seg(nullptr), *reg_ins(nullptr), *reg_zero(nullptr), *sums(nullptr);
    const uint32_t nr(d->n_regions);
    if ((rc = sx_ensure(ctx, 46, (size_t)n_alns * 4 + 16, reinterpret_cast<void**>(&aln_read)))) return rc;
    if ((rc = sx_ensure(ctx, 47, (size_t)d->n_reads * 4 + 16, reinterpret_cast<void**>(&read_region)))) return rc;
    if ((rc = sx_ensure(ctx, 48, (size_t)n_alns * 4 + 16, reinterpret_cast<void**>(&seg_n)))) return rc;
    if ((rc = sx_ensure(ctx, 49, (size_t)n_alns * 4 + 16, reinterpret_cast<void**>(&ins_n)))) return rc;
    if ((rc = sx_ensure(ctx, 50, (size_t)nr * 4 + 16, reinterpret_cast<void**>(&reg_seg)))) return rc;
    if ((rc = sx_ensure(ctx, 51, (size_t)nr * 4 + 16, reinterpret_cast<void**>(&reg_ins)))) return rc;
    if ((rc = sx_ensure(ctx, 52, (size_t)nr * 4 + 16, reinterpret_cast<void**>(&reg_zero)))) return rc;
    const uint32_t tile(K7_SCAN_THREADS * K7_SCAN_ITEMS), n_tiles((nr + tile - 1) / tile);
    if ((rc = sx_ensure(ctx, 53, ((size_t)3 * n_tiles + 4) * 4, reinterpret_cast<void**>(&sums)))) return rc;
    uint32_t* totals(sums + (size_t)3 * n_tiles);
    k8_view v;
    v.b = *d;
    v.e = *e;
    v.key_ins_off = key_ins_off;
    v.key_ins = key_ins;
    const int cap(ctx->sm_count * 16);
    const auto grid = [cap](const uint32_t n) { return (unsigned)std::max(1, std::min<int>((int)((n + 127) / 128), cap)); };
    k8_read_region_kernel<<<grid(nr), 128, 0, st>>>(nr, d->region_read_off, read_region);
    SX_CUDA(ctx, cudaGetLastError());
    k8_aln_read_kernel<<<grid(d->n_reads), 128, 0, st>>>(d->n_reads, e->aln_off, aln_read);
    SX_CUDA(ctx, cudaGetLastError());
    k8_size_kernel<<<grid(n_alns), 128, 0, st>>>(v, n_alns, aln_read, read_region, seg_n, ins_n, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    k8_region_kernel<<<grid((uint32_t)std::min<uint64_t>((uint64_t)nr * 32u, 0xffffff00u)), 128, 0, st>>>(v, seg_n, ins_n, reg_seg, reg_ins, reg_zero);
    SX_CUDA(ctx, cudaGetLastError());
    k7_scan_tiles<<<n_tiles, K7_SCAN_THREADS, 0, st>>>(nr, reg_seg, reg_ins, reg_zero, sums, n_tiles);
    SX_CUDA(ctx, cudaGetLastError());
    k7_scan_sums<<<1, K7_SCAN_THREADS, 0, st>>>(sums, n_tiles, totals);
    SX_CUDA(ctx, cudaGetLastError());
    k8_finish_kernel<<<n_tiles, K7_SCAN_THREADS, 0, st>>>(v, n_alns, reg_seg, reg_ins, sums, n_tiles, totals, *o, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    k8_write_kernel<<<grid(n_alns), 128, 0, st>>>(v, n_alns, aln_read, read_region, seg_n, ins_n, reg_seg, reg_ins, totals, *o);
    SX_CUDA(ctx, cudaGetLastError());
    k8_pad_kernel<<<grid(nr), 128, 0, st>>>(v, seg_n, ins_n, reg_seg, reg_ins, totals, *o);
    SX_CUDA(ctx, cudaGetLastError());
    *launches = 9;
    return SX_OK;
}

int k8_finish(sx_ctx* ctx, const char* what, const uint32_t* totals_host)
{
    int st(0);
    SX_CUDA(ctx, cudaMemcpyAsync(&st, ctx->d_status, sizeof(int), cudaMemcpyDeviceToHost, ctx->s_compute));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    if (st & (K8_CAP_BIT | (3 << K8_ST_SHIFT)))
    {
        cudaMemsetAsync(ctx->d_status, 0, sizeof(int), ctx->s_compute);
        if (st & (K8_ST_NOKEY << K8_ST_SHIFT))
            return sx_fail(ctx, SX_ERR_ARG, "%s: a path gap matches no indel key of its alignment (getMatchingIndelKey would assert)", what);
        if (st & (K8_ST_KIND << K8_ST_SHIFT)) return sx_fail(ctx, SX_ERR_ARG, "%s: can't handle cigar code", what);
        if (totals_host) return sx_fail(ctx, SX_ERR_CAPACITY, "%s: output capacity too small: %u segments, %u insert bytes needed", what, totals_host[0], totals_host[1]);
        return sx_fail(ctx, SX_ERR_CAPACITY, "%s: output capacity too small (totals[] holds the needed sizes)", what);
    }
    return sx_check_status(ctx, what);
}

int k8_check_args(sx_ctx* ctx, const sx_enum_batch* b, const sx_enum_out* e, const uint32_t* key_ins_off, const char* key_ins, const sx_link_out* o, const char* what)
{
    if (!b || !e || !o) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (!o->totals || !o->regions || !o->alns) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    if (b->n_regions == 0) return sx_fail(ctx, SX_ERR_ARG, "%s: no regions", what);
    if (!b->region_read_off || !b->region_key_off || (b->n_keys && (!b->keys || !key_ins_off || !key_ins)) || !e->aln_off || !e->aln_pos || !e->aln_seg_off || !e->segs ||
        !e->aln_key_off || !e->aln_keys || !e->aln_lead_key || !e->aln_trail_key || !o->segs || !o->ins)
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL array", what);
    return SX_OK;
}
} // namespace

extern "C" int sx_link_alignments_dev(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* e, uint32_t n_alns, const uint32_t* key_ins_off, const char* key_ins,
                                      sx_link_out* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k8_check_args(ctx, d, e, key_ins_off, key_ins, out_dev, "sx_link_alignments_dev"))) return rc;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_kernel_timer t(ctx);
    unsigned launches(0);
    if ((rc = k8_run(ctx, d, e, n_alns, key_ins_off, key_ins, out_dev, &launches))) return rc;
    t.stop(launches);
    if ((rc = t.finish())) return rc;
    return k8_finish(ctx, "sx_link_alignments", nullptr);
}

extern "C" int sx_link_alignments(sx_ctx* ctx, const sx_enum_batch* b, const sx_enum_out* e, uint32_t n_alns, const uint32_t* key_ins_off, const char* key_ins,
                                  sx_link_out* out_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k8_check_args(ctx, b, e, key_ins_off, key_ins, out_host, "sx_link_alignments"))) return rc;
    if (e->aln_off[b->n_reads] != n_alns) return sx_fail(ctx, SX_ERR_ARG, "sx_link_alignments: n_alns is not the enumeration's alignment count");
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st(ctx->s_compute);
    SX_CUDA(ctx, cudaEventRecord(ctx->ev_a, st));
    sx_enum_batch d(*b);
    sx_enum_out de(*e);
    void* p(nullptr);
    const size_t n_segs(e->aln_seg_off[n_alns]), n_keys(e->aln_key_off[n_alns]);
#define SX_UPX(slot, dst, src, type, bytes)                                                \
    if ((rc = sx_ensure(ctx, slot, (size_t)(bytes) + 16, &p))) return rc;                   \
    if (bytes) SX_CUDA(ctx, cudaMemcpyAsync(p, (src), (bytes), cudaMemcpyHostToDevice, st)); \
    dst = static_cast<type>(p);
    SX_UPX(0, d.region_read_off, b->region_read_off, const uint32_t*, (size_t)(b->n_regions + 1) * 4)
    SX_UPX(1, d.region_key_off, b->region_key_off, const uint32_t*, (size_t)(b->n_regions + 1) * 4)
    SX_UPX(2, d.keys, b->keys, const sx_indel_key*, (size_t)b->n_keys * sizeof(sx_indel_key))
    SX_UPX(3, de.aln_off, e->aln_off, uint32_t*, (size_t)(b->n_reads + 1) * 4)
    SX_UPX(4, de.aln_pos, e->aln_pos, int32_t*, (size_t)n_alns * 4)
    SX_UPX(5, de.aln_seg_off, e->aln_seg_off, uint32_t*, ((size_t)n_alns + 1) * 4)
    SX_UPX(6, de.segs, e->segs, sx_aln_seg*, n_segs * sizeof(sx_aln_seg))
    SX_UPX(7, de.aln_key_off, e->aln_key_off, uint32_t*, ((size_t)n_alns + 1) * 4)
    SX_UPX(8, de.aln_keys, e->aln_keys, uint16_t*, n_keys * 2)
    SX_UPX(9, de.aln_lead_key, e->aln_lead_key, uint16_t*, (size_t)n_alns * 2)
    SX_UPX(10, de.aln_trail_key, e->aln_trail_key, uint16_t*, (size_t)n_alns * 2)
    const uint32_t* d_key_ins_off(nullptr);
    const char* d_key_ins(nullptr);
    const size_t ins_bytes(b->n_keys ? key_ins_off[b->n_keys] : 0);
    SX_UPX(11, d_key_ins_off, key_ins_off, const uint32_t*, b->n_keys ? ((size_t)b->n_keys + 1) * 4 : 0)
    SX_UPX(12, d_key_ins, key_ins, const char*, ins_bytes)
    sx_link_out o(*out_host);
    SX_UPX(13, o.regions, out_host->regions, sx_region*, ((size_t)b->n_regions + 1) * sizeof(sx_region))
#undef SX_UPX
    if ((rc = sx_ensure(ctx, 14, 16, reinterpret_cast<void**>(&o.totals)))) return rc;
    if ((rc = sx_ensure(ctx, 15, ((size_t)n_alns + 1) * sizeof(sx_aln) + 16, reinterpret_cast<void**>(&o.alns)))) return rc;
    if ((rc = sx_ensure(ctx, 16, (size_t)o.cap_segs * sizeof(sx_aln_seg) + 16, reinterpret_cast<void**>(&o.segs)))) return rc;
    if ((rc = sx_ensure(ctx, 17, (size_t)o.cap_ins + SX_POOL_SLACK + 16, reinterpret_cast<void**>(&o.ins)))) return rc;
    if (out_host->k6_segs)
    {
        if ((rc = sx_ensure(ctx, 18, n_segs * sizeof(sx_aln_seg) + 16, reinterpret_cast<void**>(&o.k6_segs)))) return rc;
    }
    unsigned launches(0);
    if ((rc = k8_run(ctx, &d, &de, n_alns, d_key_ins_off, d_key_ins, &o, &launches))) return rc;
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->totals, o.totals, 8, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->regions, o.regions, ((size_t)b->n_regions + 1) * sizeof(sx_region), cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    const uint32_t nS(out_host->totals[0]), nI(out_host->totals[1]);
    if (nS <= o.cap_segs && nI <= o.cap_ins)
    {
        SX_CUDA(ctx, cudaMemcpyAsync(out_host->alns, o.alns, ((size_t)n_alns + 1) * sizeof(sx_aln), cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaMemcpyAsync(out_host->segs, o.segs, (size_t)nS * sizeof(sx_aln_seg), cudaMemcpyDeviceToHost, st));
        SX_CUDA(ctx, cudaMemcpyAsync(out_host->ins, o.ins, (size_t)nI, cudaMemcpyDeviceToHost, st));
        if (out_host->k6_segs) SX_CUDA(ctx, cudaMemcpyAsync(out_host->k6_segs, o.k6_segs, n_segs * sizeof(sx_aln_seg), cudaMemcpyDeviceToHost, st));
    }
    SX_CUDA(ctx, cudaEventRecord(ctx->ev_b, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    float ms(0);
    cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b);
    ctx->timing.kernel_ms = ms;
    ctx->timing.launches = launches;
    ctx->total_launches += launches;
    return k8_finish(ctx, "sx_link_alignments", out_host->totals);
}

// asynchronous launcher for the device-resident pipeline (sx_pipeline.cu)
int sx_k8_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* e, uint32_t n_alns, const uint32_t* key_ins_off, const char* key_ins, const sx_link_out* o,
              unsigned* launches)
{
    unsigned l(0);
    const int rc(k8_run(ctx, d, e, n_alns, key_ins_off, key_ins, o, &l));
    *launches += l;
    return rc;
}
