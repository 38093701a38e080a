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
#include "sx_scan3.cuh"

#include <algorithm>

namespace
{
constexpr int K7A_CAP_BIT = 1 << 18;

// byte offset of every read's first packed base: reads of a region are back to back from its seq_off, each on a byte boundary
__global__ void k7a_read_offsets_kernel(const k7a_view v, unsigned long long* __restrict__ read_byte, uint32_t* __restrict__ read_region)
{
    for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; g < v.b.n_regions; g += gridDim.x * blockDim.x)
    {
        unsigned long long at(v.regions[g].seq_off);
        for (uint32_t r = v.b.region_read_off[g]; r < v.b.region_read_off[g + 1]; ++r)
        {
            read_byte[r] = at;
            read_region[r] = g;
            at += (v.b.read_len[r] + 1u) / 2u;
        }
    }
}

// The reads the gates turned away (about half of a 30x window's) have no keys: with a gate the two passes below run over the DENSE list of the
// others (full warps instead of about a quarter of the lanes), and the first pass leaves a read's first K7A_STAGE keys in a staging row so that the second
// pass copies them instead of walking the read again.
#define K7A_STAGE 6u

__global__ void k7a_active_reads_kernel(const uint32_t n_reads, const uint8_t* __restrict__ gate, uint32_t* __restrict__ list, uint32_t* __restrict__ count)
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
        if (on) list[at + __popc(m & ((1u << lane) - 1u))] = r;
    }
}

// list == NULL: every read (and the per-read defaults are written here); otherwise the listed reads (the defaults were set by the host side)
__global__ void k7a_count_kernel(const k7a_view v, const unsigned long long* __restrict__ read_byte, const uint32_t* __restrict__ read_region, uint32_t* __restrict__ cnt,
                                 uint32_t* __restrict__ zero1, uint32_t* __restrict__ zero2, const uint32_t* __restrict__ list, const uint32_t* __restrict__ n_list,
                                 uint16_t* __restrict__ stage, const sx_prep_out o)
{
    const uint32_t n_work(list ? *n_list : v.b.n_reads);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_work; i += gridDim.x * blockDim.x)
    {
        const uint32_t r(list ? list[i] : i);
        uint16_t keys[K7A_MAX_KEYS], lead, trail;
        const uint32_t n(k7a_read(v, read_region[r], r, read_byte[r], keys, lead, trail));
        cnt[r] = n;
        if (!list) zero1[r] = zero2[r] = 0;
        o.in_lead_key[r] = lead;
        o.in_trail_key[r] = trail;
        if (stage)
            for (uint32_t k = 0; k < n && k < K7A_STAGE; ++k) stage[(size_t)r * K7A_STAGE + k] = keys[k];
    }
}

__global__ void __launch_bounds__(K7_SCAN_THREADS) k7a_finish_kernel(const uint32_t n, uint32_t* __restrict__ cnt, const uint32_t* __restrict__ sums, const uint32_t* __restrict__ totals,
                                                                    const sx_prep_out o, int* __restrict__ status)
{
    const uint32_t tile(blockIdx.x), base(tile * K7_SCAN_THREADS * K7_SCAN_ITEMS + threadIdx.x * K7_SCAN_ITEMS);
    const uint32_t off(sums[tile]);
    for (int i = 0; i < K7_SCAN_ITEMS; ++i)
        if (base + i < n)
        {
            const uint32_t x(cnt[base + i] + off);
            cnt[base + i] = x;
            o.in_key_off[base + i] = x;
        }
    if (blockIdx.x == 0 && threadIdx.x == 0)
    {
        o.in_key_off[n] = totals[0];
        o.totals[0] = totals[0];
        if (totals[0] > o.cap_keys) atomicOr(status, K7A_CAP_BIT);
    }
}

__global__ void k7a_write_kernel(const k7a_view v, const unsigned long long* __restrict__ read_byte, const uint32_t* __restrict__ read_region, const uint32_t* __restrict__ off,
                                 const uint32_t* __restrict__ totals, const uint32_t* __restrict__ list, const uint32_t* __restrict__ n_list, const uint16_t* __restrict__ stage,
                                 const sx_prep_out o)
{
    if (totals[0] > o.cap_keys) return;
    const uint32_t n_work(list ? *n_list : v.b.n_reads);
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_work; i += gridDim.x * blockDim.x)
    {
        const uint32_t r(list ? list[i] : i);
        const uint32_t at(off[r]), n_known(o.in_key_off[r + 1] - at);
        if (stage && n_known <= K7A_STAGE)
        {
            for (uint32_t k = 0; k < n_known; ++k) o.in_keys[at + k] = stage[(size_t)r * K7A_STAGE + k];
            continue;
        }
        uint16_t keys[K7A_MAX_KEYS], lead, trail;
        const uint32_t n(k7a_read(v, read_region[r], r, read_byte[r], keys, lead, trail));
        for (uint32_t k = 0; k < n; ++k) o.in_keys[at + k] = keys[k];
    }
}

__global__ void k7g_gates_kernel(const sx_gate_batch b, const sx_gate_out o, uint32_t* __restrict__ read_region)
{
    // reads of a region are consecutive: a thread finds its read's region by a binary search of region_read_off
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < b.n_reads; r += gridDim.x * blockDim.x)
    {
        uint32_t lo(0), hi(b.n_regions);
        while (lo + 1 < hi)
        {
            const uint32_t mid((lo + hi) / 2);
            if (b.region_read_off[mid] <= r) lo = mid;
            else hi = mid;
        }
        int32_t pos;
        o.gate[r] = (uint8_t)k7g_read(b, lo, r, pos, o.in_segs + b.seg_off[r]);
        o.in_pos[r] = pos;
    }
    (void)read_region;
}

int k7a_run(sx_ctx* ctx, const k7a_view& v, const sx_prep_out* o, unsigned* launches)
{
    cudaStream_t st(ctx->s_compute);
    const uint32_t n(v.b.n_reads);
    int rc;
    unsigned long long* read_byte(nullptr);
    uint32_t *read_region(nullptr), *cnt(nullptr), *z1(nullptr), *z2(nullptr), *sums(nullptr);
    if ((rc = sx_ensure(ctx, 58, (size_t)n * 8 + 16, reinterpret_cast<void**>(&read_byte)))) return rc;
    if ((rc = sx_ensure(ctx, 59, (size_t)n * 4 + 16, reinterpret_cast<void**>(&read_region)))) return rc;
    if ((rc = sx_ensure(ctx, 60, (size_t)n * 4 + 16, reinterpret_cast<void**>(&cnt)))) return rc;
    if ((rc = sx_ensure(ctx, 61, (size_t)n * 4 + 16, reinterpret_cast<void**>(&z1)))) return rc;
    if ((rc = sx_ensure(ctx, 62, (size_t)n * 4 + 16, reinterpret_cast<void**>(&z2)))) return rc;
    const uint32_t tile(K7_SCAN_THREADS * K7_SCAN_ITEMS), n_tiles((n + tile - 1) / tile);
    if ((rc = sx_ensure(ctx, 63, ((size_t)3 * n_tiles + 4) * 4, reinterpret_cast<void**>(&sums)))) return rc;
    uint32_t* totals(sums + (size_t)3 * n_tiles);
    const int cap(ctx->sm_count * 16);
    const auto grid = [cap](const uint32_t m) { return (unsigned)std::max(1, std::min<int>((int)((m + 127) / 128), cap)); };
    k7a_read_offsets_kernel<<<grid(v.b.n_regions), 128, 0, st>>>(v, read_byte, read_region);
    SX_CUDA(ctx, cudaGetLastError());
    uint32_t *list(nullptr), *n_list(nullptr);
    uint16_t* stage(nullptr);
    unsigned extra(0);
    if ((rc = sx_ensure(ctx, 39, (size_t)n * K7A_STAGE * 2 + 16, reinterpret_cast<void**>(&stage)))) return rc;
    if (v.b.gate)
    {
        if ((rc = sx_ensure(ctx, 38, ((size_t)n + 4) * 4, reinterpret_cast<void**>(&list)))) return rc;
        n_list = list + n;
        SX_CUDA(ctx, cudaMemsetAsync(n_list, 0, 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(cnt, 0, (size_t)n * 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(z1, 0, (size_t)n * 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(z2, 0, (size_t)n * 4, st));
        SX_CUDA(ctx, cudaMemsetAsync(o->in_lead_key, 0xFF, (size_t)n * 2, st)); // SX_NO_KEY
        SX_CUDA(ctx, cudaMemsetAsync(o->in_trail_key, 0xFF, (size_t)n * 2, st));
        k7a_active_reads_kernel<<<std::max(1, std::min<int>((int)((n + 255) / 256), ctx->sm_count * 8)), 256, 0, st>>>(n, v.b.gate, list, n_list);
        SX_CUDA(ctx, cudaGetLastError());
        extra = 1;
    }
    k7a_count_kernel<<<grid(n), 128, 0, st>>>(v, read_byte, read_region, cnt, z1, z2, list, n_list, stage, *o);
    SX_CUDA(ctx, cudaGetLastError());
    k7_scan_tiles<<<n_tiles, K7_SCAN_THREADS, 0, st>>>(n, cnt, z1, z2, sums, n_tiles);
    SX_CUDA(ctx, cudaGetLastError());
    k7_scan_sums<<<1, K7_SCAN_THREADS, 0, st>>>(sums, n_tiles, totals);
    SX_CUDA(ctx, cudaGetLastError());
    k7a_finish_kernel<<<n_tiles, K7_SCAN_THREADS, 0, st>>>(n, cnt, sums, totals, *o, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    k7a_write_kernel<<<grid(n), 128, 0, st>>>(v, read_byte, read_region, cnt, totals, list, n_list, stage, *o);
    SX_CUDA(ctx, cudaGetLastError());
    *launches = 6 + extra;
    return SX_OK;
}

int k7a_finish(sx_ctx* ctx, const char* what, const uint32_t* totals_host)
{
    int st(0);
    SX_CUDA(ctx, cudaMemcpyAsync(&st, ctx->d_status, sizeof(int), cudaMemcpyDeviceToHost, ctx->s_compute));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    if (st & K7A_CAP_BIT)
    {
        cudaMemsetAsync(ctx->d_status, 0, sizeof(int), ctx->s_compute);
        if (totals_host) return sx_fail(ctx, SX_ERR_CAPACITY, "%s: cap_keys too small: %u keys needed", what, totals_host[0]);
        return sx_fail(ctx, SX_ERR_CAPACITY, "%s: cap_keys too small (totals[0] holds the needed size)", what);
    }
    return sx_check_status(ctx, what);
}

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
} // namespace

namespace
{
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
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_kernel_timer t(ctx);
    const unsigned grid((unsigned)std::max(1, std::min<int>((int)((d->n_reads + 127) / 128), ctx->sm_count * 16)));
    k7g_gates_kernel<<<grid, 128, 0, ctx->s_compute>>>(*d, *out_dev, nullptr);
    SX_CUDA(ctx, cudaGetLastError());
    t.stop(1);
    if ((rc = t.finish())) return rc;
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
    cudaStream_t st(ctx->s_compute);
    SX_CUDA(ctx, cudaEventRecord(ctx->ev_a, st));
    sx_gate_batch d(*b);
    void* p(nullptr);
    const size_t n_segs(b->seg_off[b->n_reads]), n_win(b->region_key_off[b->n_regions]);
#define SX_UPX(slot, dst, src, type, bytes)                                                \
    if ((rc = sx_ensure(ctx, slot, (size_t)(bytes) + 16, &p))) return rc;                   \
    if (bytes) SX_CUDA(ctx, cudaMemcpyAsync(p, (src), (bytes), cudaMemcpyHostToDevice, st)); \
    dst = static_cast<type>(p);
    SX_UPX(0, d.region_read_off, b->region_read_off, const uint32_t*, (size_t)(b->n_regions + 1) * 4)
    SX_UPX(1, d.region_key_off, b->region_key_off, const uint32_t*, (size_t)(b->n_regions + 1) * 4)
    SX_UPX(2, d.keys, b->keys, const sx_indel_key*, n_win * sizeof(sx_indel_key))
    SX_UPX(3, d.realign_begin, b->realign_begin, const int32_t*, (size_t)b->n_regions * 4)
    SX_UPX(4, d.realign_end, b->realign_end, const int32_t*, (size_t)b->n_regions * 4)
    SX_UPX(5, d.raw_pos, b->raw_pos, const int32_t*, (size_t)b->n_reads * 4)
    SX_UPX(6, d.seg_off, b->seg_off, const uint32_t*, (size_t)(b->n_reads + 1) * 4)
    SX_UPX(7, d.raw_segs, b->raw_segs, const sx_aln_seg*, n_segs * sizeof(sx_aln_seg))
    SX_UPX(8, d.read_len, b->read_len, const uint16_t*, (size_t)b->n_reads * 2)
    if (b->pin_flags)
    {
        SX_UPX(9, d.pin_flags, b->pin_flags, const uint8_t*, (size_t)b->n_reads)
    }
#undef SX_UPX
    sx_gate_out o;
    if ((rc = sx_ensure(ctx, 10, (size_t)b->n_reads + 16, reinterpret_cast<void**>(&o.gate)))) return rc;
    if ((rc = sx_ensure(ctx, 11, (size_t)b->n_reads * 4 + 16, reinterpret_cast<void**>(&o.in_pos)))) return rc;
    if ((rc = sx_ensure(ctx, 12, n_segs * sizeof(sx_aln_seg) + 16, reinterpret_cast<void**>(&o.in_segs)))) return rc;
    const unsigned grid((unsigned)std::max(1, std::min<int>((int)((b->n_reads + 127) / 128), ctx->sm_count * 16)));
    k7g_gates_kernel<<<grid, 128, 0, st>>>(d, o, nullptr);
    SX_CUDA(ctx, cudaGetLastError());
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->gate, o.gate, (size_t)b->n_reads, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->in_pos, o.in_pos, (size_t)b->n_reads * 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->in_segs, o.in_segs, n_segs * sizeof(sx_aln_seg), cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaEventRecord(ctx->ev_b, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    float ms(0);
    cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b);
    ctx->timing.kernel_ms = ms;
    ctx->timing.launches = 1;
    ctx->total_launches += 1;
    return sx_check_status(ctx, "sx_realign_gates");
}

extern "C" int sx_alignment_indels_dev(sx_ctx* ctx, const sx_enum_batch* d, const sx_region* regions, const uint8_t* seq4, const char* ref, const uint32_t* key_ins_off,
                                       const char* key_ins, sx_prep_out* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k7a_check_args(ctx, d, regions, seq4, ref, key_ins_off, key_ins, out_dev, "sx_alignment_indels_dev"))) return rc;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    if (d->n_reads == 0)
    {
        SX_CUDA(ctx, cudaMemsetAsync(out_dev->totals, 0, 4, ctx->s_compute));
        SX_CUDA(ctx, cudaMemsetAsync(out_dev->in_key_off, 0, 4, ctx->s_compute));
        SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
        return SX_OK;
    }
    k7a_view v;
    v.b = *d;
    v.regions = regions;
    v.seq4 = seq4;
    v.ref = ref;
    v.key_ins_off = key_ins_off;
    v.key_ins = key_ins;
    sx_kernel_timer t(ctx);
    unsigned launches(0);
    if ((rc = k7a_run(ctx, v, out_dev, &launches))) return rc;
    t.stop(launches);
    if ((rc = t.finish())) return rc;
    return k7a_finish(ctx, "sx_alignment_indels", nullptr);
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
    cudaStream_t st(ctx->s_compute);
    SX_CUDA(ctx, cudaEventRecord(ctx->ev_a, st));
    k7a_view v;
    v.b = *b;
    void* p(nullptr);
    const size_t n_segs(b->in_seg_off[b->n_reads]);
    const sx_region& end(regions[b->n_regions]); // the sentinel carries the pool sizes
#define SX_UPX(slot, dst, src, type, bytes)                                                \
    if ((rc = sx_ensure(ctx, slot, (size_t)(bytes) + 16, &p))) return rc;                   \
    if (bytes) SX_CUDA(ctx, cudaMemcpyAsync(p, (src), (bytes), cudaMemcpyHostToDevice, st)); \
    dst = static_cast<type>(p);
    SX_UPX(0, v.b.region_read_off, b->region_read_off, const uint32_t*, (size_t)(b->n_regions + 1) * 4)
    SX_UPX(1, v.b.region_key_off, b->region_key_off, const uint32_t*, (size_t)(b->n_regions + 1) * 4)
    SX_UPX(2, v.b.keys, b->keys, const sx_indel_key*, (size_t)b->n_keys * sizeof(sx_indel_key))
    SX_UPX(3, v.b.in_pos, b->in_pos, const int32_t*, (size_t)b->n_reads * 4)
    SX_UPX(4, v.b.in_seg_off, b->in_seg_off, const uint32_t*, (size_t)(b->n_reads + 1) * 4)
    SX_UPX(5, v.b.in_segs, b->in_segs, const sx_aln_seg*, n_segs * sizeof(sx_aln_seg))
    SX_UPX(6, v.b.read_len, b->read_len, const uint16_t*, (size_t)b->n_reads * 2)
    if (b->gate)
    {
        SX_UPX(17, v.b.gate, b->gate, const uint8_t*, (size_t)b->n_reads)
    }
    SX_UPX(7, v.regions, regions, const sx_region*, ((size_t)b->n_regions + 1) * sizeof(sx_region))
    SX_UPX(8, v.seq4, seq4, const uint8_t*, (size_t)end.seq_off + SX_POOL_SLACK)
    SX_UPX(9, v.ref, ref, const char*, (size_t)end.ref_off + SX_POOL_SLACK)
    const size_t ins_bytes(b->n_keys ? key_ins_off[b->n_keys] : 0);
    SX_UPX(10, v.key_ins_off, key_ins_off, const uint32_t*, b->n_keys ? ((size_t)b->n_keys + 1) * 4 : 0)
    SX_UPX(11, v.key_ins, key_ins, const char*, ins_bytes)
#undef SX_UPX
    sx_prep_out o(*out_host);
    if ((rc = sx_ensure(ctx, 12, 16, reinterpret_cast<void**>(&o.totals)))) return rc;
    if ((rc = sx_ensure(ctx, 13, (size_t)(b->n_reads + 1) * 4 + 16, reinterpret_cast<void**>(&o.in_key_off)))) return rc;
    if ((rc = sx_ensure(ctx, 14, (size_t)o.cap_keys * 2 + 16, reinterpret_cast<void**>(&o.in_keys)))) return rc;
    if ((rc = sx_ensure(ctx, 15, (size_t)b->n_reads * 2 + 16, reinterpret_cast<void**>(&o.in_lead_key)))) return rc;
    if ((rc = sx_ensure(ctx, 16, (size_t)b->n_reads * 2 + 16, reinterpret_cast<void**>(&o.in_trail_key)))) return rc;
    unsigned launches(0);
    if ((rc = k7a_run(ctx, v, &o, &launches))) return rc;
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->totals, o.totals, 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->in_key_off, o.in_key_off, (size_t)(b->n_reads + 1) * 4, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->in_lead_key, o.in_lead_key, (size_t)b->n_reads * 2, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaMemcpyAsync(out_host->in_trail_key, o.in_trail_key, (size_t)b->n_reads * 2, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    if (out_host->totals[0] <= o.cap_keys) SX_CUDA(ctx, cudaMemcpyAsync(out_host->in_keys, o.in_keys, (size_t)out_host->totals[0] * 2, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaEventRecord(ctx->ev_b, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    float ms(0);
    cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b);
    ctx->timing.kernel_ms = ms;
    ctx->timing.launches = launches;
    ctx->total_launches += launches;
    return k7a_finish(ctx, "sx_alignment_indels", out_host->totals);
}

// ---- asynchronous launchers for the device-resident pipeline (sx_pipeline.cu): everything is enqueued on ctx->s_compute, nothing waits
int sx_k7g_run(sx_ctx* ctx, const sx_gate_batch* d, const sx_gate_out* o, unsigned* launches)
{
    if (d->n_reads == 0) return SX_OK;
    const unsigned grid((unsigned)std::max(1, std::min<int>((int)((d->n_reads + 127) / 128), ctx->sm_count * 16)));
    k7g_gates_kernel<<<grid, 128, 0, ctx->s_compute>>>(*d, *o, nullptr);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

int sx_k7a_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_region* regions, const uint8_t* seq4, const char* ref, const uint32_t* key_ins_off, const char* key_ins,
               const sx_prep_out* o, unsigned* launches)
{
    k7a_view v;
    v.b = *d;
    v.regions = regions;
    v.seq4 = seq4;
    v.ref = ref;
    v.key_ins_off = key_ins_off;
    v.key_ins = key_ins;
    unsigned l(0);
    const int rc(k7a_run(ctx, v, o, &l));
    *launches += l;
    return rc;
}
