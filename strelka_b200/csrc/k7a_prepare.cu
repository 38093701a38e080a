// k7a_prepare.cu -- K7a alignment_indels: the keys an input alignment already contains, on the device.
//
// Replaces (include/strelka_b200.h, "K7a alignment_indels") the first step of getCandidateAlignments
// (starling_common/starling_read_align.cpp:1853-1858): getCandidateAlignment :1481-1522 + getAlignmentIndels
// (CandidateAlignment.cpp:58-173) -- the per-base host loop in front of K7.  Per-read body: k7a_core.cuh.
//
// Shape of the work: one pass over every aligned read base (a nibble load + a reference byte load + a compare; a binary search of the
// window only at a mismatch) -- HBM-bound at ~1.5 bytes per base, all of it data K1 reads anyway.  One read per thread; the CSR
// output needs the usual count -> scan -> write, and the body is cheap enough to run twice.

#include "k7a_core.cuh"
#include "sx_internal.h"
#include "sx_read_index.cuh"

#include <algorithm>
#include <cstring>

namespace
{
// the byte offset of read r's first packed base from the read index's 32-bit offset: the region's 64-bit seq_off plus the read's place in the
// region (the index's offsets wrap at 4 GiB together with the region's)
__device__ __forceinline__ uint64_t k7a_read_byte(const k7a_view& v, const uint32_t g, const uint32_t* __restrict__ seq_off, const uint32_t r)
{
    const uint64_t b(v.regions[g].seq_off);
    return b + (uint32_t)(seq_off[r] - (uint32_t)b);
}

// The reads the gates turned away (about half of a 30x window's) have no keys: with a gate the two passes below run over the DENSE list of the
// others (full warps instead of about a quarter of the lanes), and the first pass leaves a read's first K7A_STAGE keys in a staging row so that the second
// pass copies them instead of walking the read again.
#define K7A_STAGE 6u

// list == NULL: every read (and the per-read defaults are written here); otherwise the listed reads (the defaults were set by the host side).
// The counts go into in_key_off, which the scan turns into the offsets.
__global__ void k7a_count_kernel(const k7a_view v, const uint32_t* __restrict__ seq_off, const uint32_t* __restrict__ read_region,
                                 const uint32_t* __restrict__ list, const uint32_t* __restrict__ n_list, uint16_t* __restrict__ stage, const sx_prep_out o)
{
    const uint32_t n_work(list ? *n_list : v.b.n_reads);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_work; i += gridDim.x * blockDim.x)
    {
        const uint32_t r(list ? list[i] : i);
        const uint32_t g(read_region[r]);
        uint16_t keys[K7A_MAX_KEYS], lead, trail;
        const uint32_t n(k7a_read(v, g, r, k7a_read_byte(v, g, seq_off, r), keys, lead, trail));
        o.in_key_off[r] = n;
        o.in_lead_key[r] = lead;
        o.in_trail_key[r] = trail;
        if (stage)
            for (uint32_t k = 0; k < n && k < K7A_STAGE; ++k) stage[(size_t)r * K7A_STAGE + k] = keys[k];
    }
}

__global__ void k7a_write_kernel(const k7a_view v, const uint32_t* __restrict__ seq_off, const uint32_t* __restrict__ read_region, const uint32_t* __restrict__ list,
                                 const uint32_t* __restrict__ n_list, const uint16_t* __restrict__ stage, const sx_prep_out o, int* __restrict__ status)
{
    if (o.totals[0] > o.cap_keys)
    {
        if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(status, SX_ST_K7A_CAP);
        return;
    }
    const uint32_t n_work(list ? *n_list : v.b.n_reads);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_work; i += gridDim.x * blockDim.x)
    {
        const uint32_t r(list ? list[i] : i);
        const uint32_t at(o.in_key_off[r]), n_known(o.in_key_off[r + 1] - at);
        if (stage && n_known <= K7A_STAGE)
        {
            for (uint32_t k = 0; k < n_known; ++k) o.in_keys[at + k] = stage[(size_t)r * K7A_STAGE + k];
            continue;
        }
        const uint32_t g(read_region[r]);
        uint16_t keys[K7A_MAX_KEYS], lead, trail;
        const uint32_t n(k7a_read(v, g, r, k7a_read_byte(v, g, seq_off, r), keys, lead, trail));
        for (uint32_t k = 0; k < n; ++k) o.in_keys[at + k] = keys[k];
    }
}

// read_region: the read index's (the window pass), or NULL: a binary search of region_read_off per read (the gates' own entry points)
__global__ void k7g_gates_kernel(const sx_gate_batch b, const sx_gate_out o, const uint32_t* __restrict__ read_region)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < b.n_reads; r += gridDim.x * blockDim.x)
    {
        const uint32_t g(read_region ? read_region[r] : sxi_region_of(b.region_read_off, b.n_regions, r));
        int32_t pos;
        o.gate[r] = (uint8_t)k7g_read(b, g, r, pos, o.in_segs + b.seg_off[r]);
        o.in_pos[r] = pos;
    }
}
} // namespace

// K7a's launcher
int sx_k7a_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_region* regions, const uint8_t* seq4, const char* ref, const uint32_t* key_ins_off, const char* key_ins,
               const sx_prep_out* o, const uint32_t* read_region, const uint32_t* read_seq_off, unsigned* launches)
{
    k7a_view v;
    v.b = *d;
    v.regions = regions;
    v.seq4 = seq4;
    v.ref = ref;
    v.key_ins_off = key_ins_off;
    v.key_ins = key_ins;
    cudaStream_t st(ctx->s_compute);
    const uint32_t n(v.b.n_reads);
    int rc;
    if (!read_region || !read_seq_off) // no window pass in front: the read index's region and packed-base offsets of every read
    {
        uint32_t *region(nullptr), *seq_off(nullptr);
        if ((rc = sx_take(ctx, SX_SLOT_K7A_READ_REGION, n, region, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K7A_K9_READ_WORD, (size_t)n + 1, seq_off, 16))) return rc;
        sx_read_index_in in;
        memset(&in, 0, sizeof(in));
        in.n_regions = v.b.n_regions;
        in.n_reads = n;
        in.region_read_off = v.b.region_read_off;
        in.read_len = v.b.read_len;
        in.regions = regions;
        sx_read_index ix;
        memset(&ix, 0, sizeof(ix));
        ix.region = region;
        ix.seq_off = seq_off;
        if ((rc = sx_read_index_run(ctx, &in, &ix, launches))) return rc;
        read_region = region;
        read_seq_off = seq_off;
    }
    const int cap(ctx->sm_count * 16);
    const auto grid = [cap](const uint32_t m) { return (unsigned)std::max(1, std::min<int>((int)((m + 127) / 128), cap)); };
    uint32_t *list(nullptr), *n_list(nullptr);
    uint16_t* stage(nullptr);
    unsigned extra(0);
    if ((rc = sx_take(ctx, SX_SLOT_K7A_STAGE, (size_t)n * K7A_STAGE, stage, 16))) return rc;
    if (v.b.gate)
    {
        if ((rc = sx_take(ctx, SX_SLOT_K7A_ACTIVE, (size_t)n + 4, list, 0))) return rc;
        n_list = list + n;
        SX_CUDA(ctx, cudaMemsetAsync(n_list, 0, 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(o->in_key_off, 0, (size_t)n * 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(o->in_lead_key, 0xFF, (size_t)n * 2, st)); // SX_NO_KEY
        SX_CUDA(ctx, cudaMemsetAsync(o->in_trail_key, 0xFF, (size_t)n * 2, st));
        if ((rc = sx_k7_active_reads(ctx, n, v.b.gate, list, n_list))) return rc;
        extra = 1;
    }
    k7a_count_kernel<<<grid(n), 128, 0, st>>>(v, read_seq_off, read_region, list, n_list, stage, *o);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1 + extra;
    const sx_scan_set J = {1, {{o->in_key_off, n, SX_SCAN_EXCLUSIVE | SX_SCAN_CLOSE, o->totals}}};
    if ((rc = sx_scan(ctx, SX_SLOT_K7A_K9_SUMS, J, launches))) return rc;
    k7a_write_kernel<<<grid(n), 128, 0, st>>>(v, read_seq_off, read_region, list, n_list, stage, *o, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

// K7g's launcher
int sx_k7g_run(sx_ctx* ctx, const sx_gate_batch* d, const sx_gate_out* o, const uint32_t* read_region, unsigned* launches)
{
    if (d->n_reads == 0) return SX_OK;
    const unsigned grid((unsigned)std::max(1, std::min<int>((int)((d->n_reads + 127) / 128), ctx->sm_count * 16)));
    k7g_gates_kernel<<<grid, 128, 0, ctx->s_compute>>>(*d, *o, read_region);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

namespace
{
int k7a_check_args(sx_ctx* ctx, const sx_enum_batch* b, const sx_region* regions, const uint8_t* seq4, const char* ref, const uint32_t* key_ins_off, const char* key_ins,
                   const sx_prep_out* o, const char* what)
{
    if (!b || !o || !regions || !seq4 || !ref) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (!o->totals || !o->in_key_off) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    if (b->n_reads == 0) return SX_OK;
    if (!b->region_read_off || !b->region_key_off || !b->in_pos || !b->in_seg_off || !b->in_segs || !b->read_len || (b->n_keys && (!b->keys || !key_ins_off || !key_ins)) ||
        !o->in_keys || !o->in_lead_key || !o->in_trail_key)
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL array", what);
    if (b->n_regions == 0) return sx_fail(ctx, SX_ERR_ARG, "%s: reads without a region", what);
    return SX_OK;
}

int k7g_check_args(sx_ctx* ctx, const sx_gate_batch* b, const sx_gate_out* o, const char* what)
{
    if (!b || !o) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (b->n_reads == 0) return SX_OK;
    if (!b->region_read_off || !b->region_key_off || !b->realign_begin || !b->realign_end || !b->raw_pos || !b->seg_off || !b->raw_segs || !b->read_len || !o->gate ||
        !o->in_pos || !o->in_segs)
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL array", what);
    if (b->n_regions == 0) return sx_fail(ctx, SX_ERR_ARG, "%s: reads without a region", what);
    return SX_OK;
}
} // namespace

extern "C" int sx_realign_gates_dev(sx_ctx* ctx, const sx_gate_batch* d, sx_gate_out* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k7g_check_args(ctx, d, out_dev, "sx_realign_gates_dev"))) return rc;
    if (d->n_reads == 0) return SX_OK;
    if ((rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k7g_run(ctx, d, out_dev, nullptr, launches); }))) return rc;
    return sx_check_status(ctx, "sx_realign_gates");
}

extern "C" int sx_realign_gates(sx_ctx* ctx, const sx_gate_batch* b, sx_gate_out* out_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k7g_check_args(ctx, b, out_host, "sx_realign_gates"))) return rc;
    if (b->n_reads == 0) return SX_OK;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer t(ctx);
    sx_gate_batch d(*b);
    const size_t n(b->n_reads), nr(b->n_regions), n_segs(b->seg_off[b->n_reads]), n_win(b->region_key_off[b->n_regions]);
    if ((rc = sx_upload(ctx, sx_host_slot(0), b->region_read_off, nr + 1, d.region_read_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(1), b->region_key_off, nr + 1, d.region_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(2), b->keys, n_win, d.keys, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(3), b->realign_begin, nr, d.realign_begin, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(4), b->realign_end, nr, d.realign_end, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(5), b->raw_pos, n, d.raw_pos, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(6), b->seg_off, n + 1, d.seg_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(7), b->raw_segs, n_segs, d.raw_segs, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(8), b->read_len, n, d.read_len, 16))) return rc;
    if (b->pin_flags && (rc = sx_upload(ctx, sx_host_slot(9), b->pin_flags, n, d.pin_flags, 16))) return rc;
    sx_gate_out o;
    if ((rc = sx_take(ctx, sx_host_slot(10), n, o.gate, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(11), n, o.in_pos, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(12), n_segs, o.in_segs, 16))) return rc;
    unsigned launches(0);
    if ((rc = sx_k7g_run(ctx, &d, &o, nullptr, &launches))) return rc;
    if ((rc = sx_download(ctx, out_host->gate, o.gate, n))) return rc;
    if ((rc = sx_download(ctx, out_host->in_pos, o.in_pos, n))) return rc;
    if ((rc = sx_download(ctx, out_host->in_segs, o.in_segs, n_segs))) return rc;
    if ((rc = t.finish(launches))) return rc;
    return sx_check_status(ctx, "sx_realign_gates");
}

extern "C" int sx_alignment_indels_dev(sx_ctx* ctx, const sx_enum_batch* d, const sx_region* regions, const uint8_t* seq4, const char* ref, const uint32_t* key_ins_off,
                                       const char* key_ins, sx_prep_out* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k7a_check_args(ctx, d, regions, seq4, ref, key_ins_off, key_ins, out_dev, "sx_alignment_indels_dev"))) return rc;
    if (d->n_reads == 0)
    {
        SX_CUDA(ctx, cudaSetDevice(ctx->device));
        SX_CUDA(ctx, cudaMemsetAsync(out_dev->totals, 0, 4, ctx->s_compute));
        SX_CUDA(ctx, cudaMemsetAsync(out_dev->in_key_off, 0, 4, ctx->s_compute));
        SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
        return SX_OK;
    }
    if ((rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k7a_run(ctx, d, regions, seq4, ref, key_ins_off, key_ins, out_dev, nullptr, nullptr, launches); }))) return rc;
    return sx_check_status(ctx, "sx_alignment_indels", SX_ST_K7A_CAP);
}

extern "C" int sx_alignment_indels(sx_ctx* ctx, const sx_enum_batch* b, const sx_region* regions, const uint8_t* seq4, const char* ref, const uint32_t* key_ins_off,
                                   const char* key_ins, sx_prep_out* out_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k7a_check_args(ctx, b, regions, seq4, ref, key_ins_off, key_ins, out_host, "sx_alignment_indels"))) return rc;
    if (b->n_reads == 0)
    {
        out_host->totals[0] = 0;
        out_host->in_key_off[0] = 0;
        return SX_OK;
    }
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer t(ctx);
    sx_enum_batch d(*b);
    const sx_region* d_regions(nullptr);
    const uint8_t* d_seq4(nullptr);
    const char *d_ref(nullptr), *d_key_ins(nullptr);
    const uint32_t* d_key_ins_off(nullptr);
    const size_t n(b->n_reads), nr(b->n_regions), n_segs(b->in_seg_off[b->n_reads]);
    const sx_region& end(regions[b->n_regions]); // the sentinel carries the pool sizes
    if ((rc = sx_upload(ctx, sx_host_slot(0), b->region_read_off, nr + 1, d.region_read_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(1), b->region_key_off, nr + 1, d.region_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(2), b->keys, b->n_keys, d.keys, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(3), b->in_pos, n, d.in_pos, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(4), b->in_seg_off, n + 1, d.in_seg_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(5), b->in_segs, n_segs, d.in_segs, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(6), b->read_len, n, d.read_len, 16))) return rc;
    if (b->gate && (rc = sx_upload(ctx, sx_host_slot(17), b->gate, n, d.gate, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(7), regions, nr + 1, d_regions, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(8), seq4, (size_t)end.seq_off + SX_POOL_SLACK, d_seq4, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(9), ref, (size_t)end.ref_off + SX_POOL_SLACK, d_ref, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(10), key_ins_off, b->n_keys ? (size_t)b->n_keys + 1 : 0, d_key_ins_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(11), key_ins, b->n_keys ? key_ins_off[b->n_keys] : 0, d_key_ins, 16))) return rc;
    sx_prep_out o(*out_host);
    if ((rc = sx_take(ctx, sx_host_slot(12), 4, o.totals, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(13), n + 1, o.in_key_off, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(14), o.cap_keys, o.in_keys, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(15), n, o.in_lead_key, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(16), n, o.in_trail_key, 16))) return rc;
    unsigned launches(0);
    if ((rc = sx_k7a_run(ctx, &d, d_regions, d_seq4, d_ref, d_key_ins_off, d_key_ins, &o, nullptr, nullptr, &launches))) return rc;
    if ((rc = sx_download(ctx, out_host->totals, o.totals, 1))) return rc;
    if ((rc = sx_download(ctx, out_host->in_key_off, o.in_key_off, n + 1))) return rc;
    if ((rc = sx_download(ctx, out_host->in_lead_key, o.in_lead_key, n))) return rc;
    if ((rc = sx_download(ctx, out_host->in_trail_key, o.in_trail_key, n))) return rc;
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    if (out_host->totals[0] <= o.cap_keys && (rc = sx_download(ctx, out_host->in_keys, o.in_keys, out_host->totals[0]))) return rc;
    if ((rc = t.finish(launches))) return rc;
    return sx_check_status(ctx, "sx_alignment_indels", SX_ST_K7A_CAP, out_host->totals);
}
