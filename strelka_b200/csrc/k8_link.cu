// k8_link.cu -- K7b link_alignments: K7's candidate alignments -> the alignment part of K1's batch, in device memory.
//
// Replaces (include/strelka_b200.h, "K7b link_alignments") the per-alignment host work in front of K1: the segment walk of
// scoreCandidateAlignment (starling_common/starling_read_align_score.cpp:289-499) with getMatchingIndelKey :177-224, the insert
// sequence / leading-edge tail rule :334-338, :394-398 and the candidacy look-up :473-475 resolved.  Per-alignment body: k8_core.cuh.
//
// Shape of the work: a streaming relabel -- every K7 segment is read once, every K1 segment and insert byte written once; the only
// structure is K1's staging rule (each region's first segment a multiple of 8, its first insert byte a multiple of 16), which turns
// the offsets into a two-level prefix sum: within a region (one thread per region walks its alignments' sizes) and over regions
// (sx_scan).  Launches: sizes (thread per alignment) -> region sums -> scan -> write (thread per alignment) -> pads + region records.

#include "k8_core.cuh"
#include "sx_internal.h"

#include <algorithm>

namespace
{
constexpr int K8_ST_SHIFT = 15; // K8_ST_* bits are reported as ctx status bits 32768, 65536
static_assert((K8_ST_NOKEY << K8_ST_SHIFT) == SX_ST_K8_NO_KEY && (K8_ST_KIND << K8_ST_SHIFT) == SX_ST_K8_KIND, "K8's shifted status bits are the context's");

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
                                 uint32_t* __restrict__ reg_ins)
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
        }
    }
}

__device__ __forceinline__ bool k8_fits(const sx_link_out& o) { return o.totals[0] <= o.cap_segs && o.totals[1] <= o.cap_ins; }

__global__ void k8_write_kernel(const k8_view v, const uint32_t n_alns, const uint32_t* __restrict__ aln_read, const uint32_t* __restrict__ read_region,
                                const uint32_t* __restrict__ seg_rel, const uint32_t* __restrict__ ins_rel, const uint32_t* __restrict__ reg_seg,
                                const uint32_t* __restrict__ reg_ins, const sx_link_out o)
{
    if (!k8_fits(o)) return; // reported by k8_pad_kernel
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

// the region records (also when a capacity is too small: they say what each region needs), the sentinels, the capacity check, and the
// pads between a region's last used segment / insert byte and the next region's first
__global__ void k8_pad_kernel(const k8_view v, const uint32_t n_alns, const uint32_t* __restrict__ seg_rel, const uint32_t* __restrict__ ins_rel,
                              const uint32_t* __restrict__ reg_seg, const uint32_t* __restrict__ reg_ins, const sx_link_out o, int* __restrict__ status)
{
    const uint32_t nr(v.b.n_regions);
    const uint32_t* totals(o.totals);
    const bool fits(k8_fits(o));
    if (blockIdx.x == 0 && threadIdx.x == 0)
    {
        o.regions[nr].aln_begin = n_alns;
        o.regions[nr].seg_begin = totals[0];
        o.regions[nr].ins_begin = totals[1];
        o.regions[nr].read_begin = v.b.n_reads;
        if (!fits) atomicOr(status, SX_ST_K8_CAP);
        else o.alns[n_alns] = sx_aln{v.b.n_reads, 0, totals[0], totals[1]};
    }
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < nr; g += gridDim.x * blockDim.x)
    {
        const uint32_t a0(v.e.aln_off[v.b.region_read_off[g]]), a1(v.e.aln_off[v.b.region_read_off[g + 1]]);
        o.regions[g].aln_begin = a0;
        o.regions[g].seg_begin = reg_seg[g];
        o.regions[g].ins_begin = reg_ins[g];
        if (!fits) continue;
        const uint32_t seg_end(g + 1 < nr ? reg_seg[g + 1] : totals[0]), ins_end(g + 1 < nr ? reg_ins[g + 1] : totals[1]);
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
    if (fits && blockIdx.x == 0 && threadIdx.x == 0) // K1 loads 16-byte slices: up to 16 no-op segments of slack after the last one, where they fit
        for (uint32_t s = totals[0]; s < o.cap_segs && s < totals[0] + 16u; ++s) o.segs[s] = sx_aln_seg{0, SX_SEG_HARDCLIP, 0};
}
} // namespace

// K7b's launcher
int sx_k8_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* e, const uint32_t n_alns, const uint32_t* key_ins_off, const char* key_ins, const sx_link_out* o,
              unsigned* launches)
{
    cudaStream_t st(ctx->s_compute);
    int rc;
    uint32_t *aln_read(nullptr), *read_region(nullptr), *seg_n(nullptr), *ins_n(nullptr), *reg_seg(nullptr), *reg_ins(nullptr);
    const uint32_t nr(d->n_regions);
    if ((rc = sx_take(ctx, SX_SLOT_K8_ALN_READ, n_alns, aln_read, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K8_READ_REGION, d->n_reads, read_region, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K8_SEG_N, n_alns, seg_n, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K8_INS_N, n_alns, ins_n, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K8_REG_SEG, nr, reg_seg, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K8_REG_INS, nr, reg_ins, 16))) return rc;
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
    k8_region_kernel<<<grid((uint32_t)std::min<uint64_t>((uint64_t)nr * 32u, 0xffffff00u)), 128, 0, st>>>(v, seg_n, ins_n, reg_seg, reg_ins);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 4;
    const sx_scan_set J = {2, {{reg_seg, nr, SX_SCAN_EXCLUSIVE, o->totals}, {reg_ins, nr, SX_SCAN_EXCLUSIVE, o->totals + 1}}};
    if ((rc = sx_scan(ctx, SX_SLOT_K8_SUMS, J, launches))) return rc;
    k8_write_kernel<<<grid(n_alns), 128, 0, st>>>(v, n_alns, aln_read, read_region, seg_n, ins_n, reg_seg, reg_ins, *o);
    SX_CUDA(ctx, cudaGetLastError());
    k8_pad_kernel<<<grid(nr), 128, 0, st>>>(v, n_alns, seg_n, ins_n, reg_seg, reg_ins, *o, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 2;
    return SX_OK;
}

namespace
{
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
    if ((rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k8_run(ctx, d, e, n_alns, key_ins_off, key_ins, out_dev, launches); }))) return rc;
    return sx_check_status(ctx, "sx_link_alignments", SX_ST_K8_NO_KEY | SX_ST_K8_KIND | SX_ST_K8_CAP);
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
    sx_call_timer t(ctx);
    sx_enum_batch d(*b);
    sx_enum_out de(*e);
    const size_t nr(b->n_regions), n_segs(e->aln_seg_off[n_alns]), n_keys(e->aln_key_off[n_alns]);
    if ((rc = sx_upload(ctx, sx_host_slot(0), b->region_read_off, nr + 1, d.region_read_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(1), b->region_key_off, nr + 1, d.region_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(2), b->keys, b->n_keys, d.keys, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(3), e->aln_off, (size_t)b->n_reads + 1, de.aln_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(4), e->aln_pos, n_alns, de.aln_pos, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(5), e->aln_seg_off, (size_t)n_alns + 1, de.aln_seg_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(6), e->segs, n_segs, de.segs, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(7), e->aln_key_off, (size_t)n_alns + 1, de.aln_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(8), e->aln_keys, n_keys, de.aln_keys, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(9), e->aln_lead_key, n_alns, de.aln_lead_key, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(10), e->aln_trail_key, n_alns, de.aln_trail_key, 16))) return rc;
    const uint32_t* d_key_ins_off(nullptr);
    const char* d_key_ins(nullptr);
    if ((rc = sx_upload(ctx, sx_host_slot(11), key_ins_off, b->n_keys ? (size_t)b->n_keys + 1 : 0, d_key_ins_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(12), key_ins, b->n_keys ? key_ins_off[b->n_keys] : 0, d_key_ins, 16))) return rc;
    sx_link_out o(*out_host);
    if ((rc = sx_upload(ctx, sx_host_slot(13), out_host->regions, nr + 1, o.regions, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(14), 4, o.totals, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(15), (size_t)n_alns + 1, o.alns, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(16), o.cap_segs, o.segs, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(17), o.cap_ins, o.ins, SX_POOL_SLACK + 16))) return rc;
    if (out_host->k6_segs && (rc = sx_take(ctx, sx_host_slot(18), n_segs, o.k6_segs, 16))) return rc;
    unsigned launches(0);
    if ((rc = sx_k8_run(ctx, &d, &de, n_alns, d_key_ins_off, d_key_ins, &o, &launches))) return rc;
    if ((rc = sx_download(ctx, out_host->totals, o.totals, 2))) return rc;
    if ((rc = sx_download(ctx, out_host->regions, o.regions, nr + 1))) return rc;
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    const uint32_t nS(out_host->totals[0]), nI(out_host->totals[1]);
    if (nS <= o.cap_segs && nI <= o.cap_ins)
    {
        if ((rc = sx_download(ctx, out_host->alns, o.alns, (size_t)n_alns + 1))) return rc;
        if ((rc = sx_download(ctx, out_host->segs, o.segs, nS))) return rc;
        if ((rc = sx_download(ctx, out_host->ins, o.ins, nI))) return rc;
        if (out_host->k6_segs && (rc = sx_download(ctx, out_host->k6_segs, o.k6_segs, n_segs))) return rc;
    }
    if ((rc = t.finish(launches))) return rc;
    return sx_check_status(ctx, "sx_link_alignments", SX_ST_K8_NO_KEY | SX_ST_K8_KIND | SX_ST_K8_CAP, out_host->totals);
}
