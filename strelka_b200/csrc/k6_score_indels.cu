// k6_score_indels.cu -- K6: the arg-max epilogue of scoreCandidateAlignments and score_indels, one read per thread.
//
// Replaces (include/strelka_b200.h, "K6 score_indels"; SURVEY 8f2)
//   starling_common/starling_read_align.cpp:1573-1593            arg-max with isFirstCandidateAlignmentPreferred
//   starling_common/starling_read_align_score_indels.cpp:454-1079 score_indels
// and consumes K1's scores where K1 wrote them (device memory).
//
// Shape of the work: per read a handful of alignments x a handful of indels of integer bookkeeping and a few fp64 adds and
// compares -- no reuse between reads and nothing GEMM-like; the algorithmic floor is reading every input once.  About half of a
// window's reads have no candidate alignment: k6_max_kernel lists the reads that have one, the host memsets the outputs of the
// others, and k6_score_list_kernel (persistent grid: resident blocks x SM count) runs one listed read per thread on the global
// arrays, the list regrouped by the read's number of alignments so that a warp's reads do similar work.  Per-read state (sort
// order, filter flags, per-indel maxima) is local memory for ordinary reads (<= 40 alignments, <= 4 output slots) and a column of
// an element-major global arena for deep ones.  Output: one 32-byte record per (read, evaluated indel).  The body is k6_core.cuh.

#include "k6_core.cuh"
#include "sx_regroup.cuh"
#include "sx_internal.h"

#include <algorithm>
#include <cstdlib>

namespace
{
constexpr int K6_THREADS = 128;
constexpr int K6_ST_SHIFT = 9; // K6_ST_* bits are reported as ctx status bits 512, 1024, ...
static_assert((K6_ST_SEGKIND << K6_ST_SHIFT) == SX_ST_K6_SEG_KIND && (K6_ST_LIMIT_A << K6_ST_SHIFT) == SX_ST_K6_ALNS && (K6_ST_LIMIT_E << K6_ST_SHIFT) == SX_ST_K6_EVAL &&
                  (K6_ST_RECCAP << K6_ST_SHIFT) == SX_ST_K6_REC_CAP && (K6_ST_BADKEY << K6_ST_SHIFT) == SX_ST_K6_KEY,
              "K6's shifted status bits are the context's");

// sizes the launch needs: out[0] = max alignments of a read, out[1] = max output slots of a read; and the dense list of the reads that
// HAVE candidate alignments -- out[2] = their count --, in read order within a warp's 32
__global__ void k6_max_kernel(const sx_score_indels_batch b, uint32_t* __restrict__ out, uint32_t* __restrict__ list)
{
    uint32_t mA(0), mS(0);
    const uint32_t tid(blockIdx.x * blockDim.x + threadIdx.x), nthr(gridDim.x * blockDim.x), lane(threadIdx.x & 31u);
    for (uint32_t b0 = tid - lane; b0 < b.n_reads; b0 += nthr)
    {
        const uint32_t r(b0 + lane);
        const uint32_t nc(r < b.n_reads ? b.aln_off[r + 1] - b.aln_off[r] : 0u);
        if (r < b.n_reads)
        {
            mA = max(mA, nc);
            mS = max(mS, b.rec_off[r + 1] - b.rec_off[r]);
        }
        const unsigned m(__ballot_sync(0xffffffffu, nc > 0));
        uint32_t at(0);
        if (lane == 0 && m) at = atomicAdd(out + 2, (uint32_t)__popc(m));
        at = __shfl_sync(0xffffffffu, at, 0);
        if (nc > 0) list[at + __popc(m & ((1u << lane) - 1u))] = r;
    }
    mA = __reduce_max_sync(0xffffffffu, mA);
    mS = __reduce_max_sync(0xffffffffu, mS);
    if ((threadIdx.x & 31) == 0)
    {
        atomicMax(out, mA);
        atomicMax(out + 1, mS);
    }
}

// the per-read body over the dense list of reads that have alignments: about half of a 30x window's reads never reach the search, and a kernel
// over all reads would idle their lanes
__global__ void __launch_bounds__(K6_THREADS) k6_score_list_kernel(const k6_view v, const k6_scratch S0, const uint32_t* __restrict__ list, const uint32_t* __restrict__ n_list,
                                                                  int* __restrict__ status)
{
    const uint32_t t(blockIdx.x * blockDim.x + threadIdx.x), nthr(gridDim.x * blockDim.x);
    k6_scratch S(S0);
    S.ord.p += t;
    S.smooth.p += t;
    S.filt.p += t;
    S.ev.p += t;
    S.slot.p += t;
    S.present.p += t;
    S.absent.p += t;
    S.has.p += t;
    S.alt.p += t;
    S.pair.p += t;
    uint32_t st(0);
    const uint32_t n(*n_list);
    for (uint32_t i = t; i < n; i += nthr)
    {
        const uint32_t r(list[i]);
        st |= k6_score_read_tiered(v, k6_region_of(v.b.region_read_off, v.b.n_regions, r), r, S);
    }
    if (st) atomicOr(status, (int)(st << K6_ST_SHIFT));
}

struct k6_layout
{
    size_t off[10];
    size_t bytes;
};

// element-major arena for T threads: array a occupies count_a * T elements
k6_layout k6_plan(const uint32_t maxA, const uint32_t maxE, const size_t T)
{
    const size_t count[10] = {maxA, maxA, maxA, maxE, maxE, maxE, maxE, (size_t)maxE * maxE, (size_t)maxE * maxE, maxE};
    const size_t elem[10] = {4, 8, 1, 2, 4, 4, 1, 4, 1, 2};
    k6_layout L;
    size_t o(0);
    for (int i = 0; i < 10; ++i)
    {
        o = (o + 255) & ~(size_t)255;
        L.off[i] = o;
        o += count[i] * elem[i] * T;
    }
    L.bytes = o;
    return L;
}

int k6_check_args(sx_ctx* ctx, const sx_score_indels_batch* b, const double* lnp, const sx_score_indels_out* out, const char* what)
{
    if (!b || !out) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (b->n_reads == 0) return SX_OK;
    if (!lnp || !b->region_read_off || !b->region_key_off || !b->aln_off || !b->aln_pos || !b->aln_seg_off || !b->aln_key_off || !b->read_len || !b->non_ambig ||
        !b->read_flags || !b->rec_off || !out->recs || !out->n_rec || !out->max_aln || !out->eval_aln)
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL array", what);
    if ((b->n_keys && !b->keys) || b->n_regions == 0) return sx_fail(ctx, SX_ERR_ARG, "%s: reads without a region / keys without a table", what);
    if (b->opts.min_read_bp_flank < 0) return sx_fail(ctx, SX_ERR_ARG, "%s: negative min_read_bp_flank", what);
    return SX_OK;
}
} // namespace

// K6's launcher: one 8-byte round trip sizes the scratch, the kernel itself is only enqueued
int sx_k6_run(sx_ctx* ctx, const sx_score_indels_batch* d, const double* lnp_dev, const sx_score_indels_out* out_dev, unsigned* launches)
{
    if (d->n_reads == 0) return SX_OK;
    cudaStream_t st(ctx->s_compute);
    // sizes of the launch: the deepest read of the batch decides the scratch
    uint32_t* d_max(nullptr);
    int rc;
    if ((rc = sx_take(ctx, SX_SLOT_K6_MAX, 8, d_max, 0))) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(d_max, 0, 12, st));
    uint32_t* list(nullptr);
    if ((rc = sx_take(ctx, SX_SLOT_K6_LIST, d->n_reads, list, 16))) return rc;
    const int grid0(std::max(1, std::min<int>((int)((d->n_reads + 255) / 256), ctx->sm_count * 8)));
    k6_max_kernel<<<grid0, 256, 0, st>>>(*d, d_max, list);
    SX_CUDA(ctx, cudaGetLastError());
    uint32_t h_max[2] = {0, 0};
    SX_CUDA(ctx, cudaMemcpyAsync(h_max, d_max, 8, cudaMemcpyDeviceToHost, st));
    SX_CUDA(ctx, cudaStreamSynchronize(st));
    const uint32_t maxA(std::max(1u, h_max[0])), maxE(std::max(1u, std::min(K6_MAX_EVAL, h_max[1])));
    const int threads(K6_THREADS);
    int per_sm(1);
    SX_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k6_score_list_kernel, threads, 0));
    per_sm = std::max(1, per_sm);

    // threads: one per read, up to the resident blocks of every SM; fewer when a deep batch would make the arena too large
    const size_t n_chunks(((size_t)d->n_reads + threads - 1) / threads);
    size_t T(std::min<size_t>(n_chunks, (size_t)ctx->sm_count * per_sm) * threads);
    const size_t arena_cap((size_t)1 << 30);
    while (T > (size_t)threads && k6_plan(maxA, maxE, T).bytes > arena_cap) T = ((T / 2 + threads - 1) / threads) * threads;
    const k6_layout L(k6_plan(maxA, maxE, T));
    char* arena(nullptr);
    if ((rc = sx_take(ctx, SX_SLOT_K6_ARENA, L.bytes, arena, 0))) return rc;
    k6_scratch S;
    S.ord = {reinterpret_cast<uint32_t*>(arena + L.off[0]), T};
    S.smooth = {reinterpret_cast<double*>(arena + L.off[1]), T};
    S.filt = {reinterpret_cast<uint8_t*>(arena + L.off[2]), T};
    S.ev = {reinterpret_cast<uint16_t*>(arena + L.off[3]), T};
    S.present = {reinterpret_cast<float*>(arena + L.off[4]), T};
    S.absent = {reinterpret_cast<float*>(arena + L.off[5]), T};
    S.has = {reinterpret_cast<uint8_t*>(arena + L.off[6]), T};
    S.alt = {reinterpret_cast<float*>(arena + L.off[7]), T};
    S.pair = {reinterpret_cast<uint8_t*>(arena + L.off[8]), T};
    S.slot = {reinterpret_cast<uint16_t*>(arena + L.off[9]), T};
    S.maxA = maxA;
    S.maxE = maxE;
    k6_view v;
    v.b = *d;
    v.lnp = lnp_dev;
    v.recs = out_dev->recs;
    v.n_rec = out_dev->n_rec;
    v.max_aln = out_dev->max_aln;
    v.eval_aln = out_dev->eval_aln;
    // the reads without alignments answer "no records, no maximum alignment" (what the body writes for them)
    SX_CUDA(ctx, cudaMemsetAsync(out_dev->n_rec, 0, (size_t)d->n_reads * 4, st));
    SX_CUDA(ctx, cudaMemsetAsync(out_dev->max_aln, 0xFF, (size_t)d->n_reads * 4, st));
    SX_CUDA(ctx, cudaMemsetAsync(out_dev->eval_aln, 0xFF, (size_t)d->n_reads * 4, st));
    unsigned extra(0);
    if (!getenv("SX_K6_NO_CLASS_SORT"))
    {
        // the list regrouped by class (sx_regroup.cuh) = the read's number of candidate alignments: score_indels loops over the alignments and the
        // window entries they carry, so warps of reads with equally many alignments stay together
        uint8_t* cls(nullptr);
        uint32_t *hist(nullptr), *list2(nullptr);
        if ((rc = sx_take(ctx, SX_SLOT_K6_CLASS, d->n_reads, cls, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K6_HIST, SX_RG_CLASSES, hist, 16))) return rc;
        if ((rc = sx_take(ctx, SX_SLOT_K6_LIST_BY_CLASS, d->n_reads, list2, 16))) return rc;
        SX_CUDA(ctx, cudaMemsetAsync(hist, 0, (size_t)SX_RG_CLASSES * 4, st));
        const int gc(std::max(1, std::min<int>((int)((d->n_reads + SX_RG_THREADS * SX_RG_ITEMS - 1) / (SX_RG_THREADS * SX_RG_ITEMS)), ctx->sm_count * 8)));
        sx_regroup_class_by_count_kernel<<<gc, SX_RG_THREADS, 0, st>>>(d->aln_off, list, d_max + 2, cls, hist);
        sx_regroup_scan_kernel<<<1, SX_RG_CLASSES, 0, st>>>(hist);
        sx_regroup_scatter_kernel<<<gc, SX_RG_THREADS, 0, st>>>(list, d_max + 2, cls, hist, list2);
        SX_CUDA(ctx, cudaGetLastError());
        list = list2;
        extra = 3;
    }
    k6_score_list_kernel<<<(unsigned)(T / threads), threads, 0, st>>>(v, S, list, d_max + 2, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 2 + extra;
    return SX_OK;
}

extern "C" void sx_default_score_indels_opts(sx_score_indels_opts* o)
{
    if (!o) return;
    o->max_indel_size = 49;                       // starling_base_shared.hh:124
    o->upstream_oligo_size = 0;                   // :206
    o->min_read_bp_flank = 5;                     // :108 default_min_read_bp_flank
    o->is_smoothed_alignments = 1;                // :170
    o->smoothed_lnp_range = 2.302585092994046;    // :171 std::log(10.)
}

extern "C" int sx_score_indels_dev(sx_ctx* ctx, const sx_score_indels_batch* d, const double* lnp_dev, sx_score_indels_out* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k6_check_args(ctx, d, lnp_dev, out_dev, "sx_score_indels_dev"))) return rc;
    if (d->n_reads == 0) return SX_OK;
    if ((rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k6_run(ctx, d, lnp_dev, out_dev, launches); }))) return rc;
    return sx_check_status(ctx, "sx_score_indels");
}

extern "C" int sx_score_indels(sx_ctx* ctx, const sx_score_indels_batch* b, const double* lnp_host, sx_score_indels_out* out_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k6_check_args(ctx, b, lnp_host, out_host, "sx_score_indels"))) return rc;
    if (b->n_reads == 0) return SX_OK;
    // host-side consistency of the offsets the uploads are sized from
    if (b->region_read_off[b->n_regions] != b->n_reads || b->region_key_off[b->n_regions] != b->n_keys || b->aln_off[b->n_reads] != b->n_alns)
        return sx_fail(ctx, SX_ERR_ARG, "sx_score_indels: offset arrays do not end at n_reads / n_keys / n_alns");
    for (uint32_t g = 0; g < b->n_regions; ++g)
        if (b->region_key_off[g + 1] - b->region_key_off[g] > 65535u) return sx_fail(ctx, SX_ERR_RANGE, "sx_score_indels: more than 65535 window entries in a region");
    for (uint32_t k = 0; k < b->n_keys; ++k)
        if (b->keys[k].type > SX_INDEL_TYPE_MISMATCH) return sx_fail(ctx, SX_ERR_UNSUPPORTED, "sx_score_indels: breakend entries are not supported");
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer t(ctx);
    sx_score_indels_batch d(*b);
    const size_t n(b->n_reads), n_segs(b->aln_seg_off[b->n_alns]), n_akeys(b->aln_key_off[b->n_alns]), n_slots(b->rec_off[b->n_reads]);
    if ((rc = sx_upload(ctx, sx_host_slot(0), b->region_read_off, (size_t)b->n_regions + 1, d.region_read_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(1), b->region_key_off, (size_t)b->n_regions + 1, d.region_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(2), b->keys, b->n_keys, d.keys, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(3), b->aln_off, n + 1, d.aln_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(4), b->aln_pos, b->n_alns, d.aln_pos, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(5), b->aln_seg_off, (size_t)b->n_alns + 1, d.aln_seg_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(6), b->segs, n_segs, d.segs, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(7), b->aln_key_off, (size_t)b->n_alns + 1, d.aln_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(8), b->aln_keys, n_akeys, d.aln_keys, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(9), b->read_len, n, d.read_len, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(10), b->non_ambig, n, d.non_ambig, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(11), b->read_flags, n, d.read_flags, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(12), b->rec_off, n + 1, d.rec_off, 16))) return rc;
    if (b->full_len && (rc = sx_upload(ctx, sx_host_slot(13), b->full_len, n, d.full_len, 16))) return rc;
    if (b->full_off && (rc = sx_upload(ctx, sx_host_slot(14), b->full_off, n, d.full_off, 16))) return rc;
    const double* d_lnp(nullptr);
    if ((rc = sx_upload(ctx, sx_host_slot(15), lnp_host, b->n_alns, d_lnp, 16))) return rc;
    sx_score_indels_out o;
    if ((rc = sx_take(ctx, sx_host_slot(16), n_slots + 1, o.recs, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(17), n, o.n_rec, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(18), n, o.max_aln, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(19), n, o.eval_aln, 0))) return rc;
    SX_CUDA(ctx, cudaMemsetAsync(o.recs, 0, (n_slots + 1) * sizeof(sx_read_indel_score), ctx->s_compute)); // unused slots read back as zeros
    unsigned launches(0);
    if ((rc = sx_k6_run(ctx, &d, d_lnp, &o, &launches))) return rc;
    if ((rc = sx_download(ctx, out_host->recs, o.recs, n_slots))) return rc;
    if ((rc = sx_download(ctx, out_host->n_rec, o.n_rec, n))) return rc;
    if ((rc = sx_download(ctx, out_host->max_aln, o.max_aln, n))) return rc;
    if ((rc = sx_download(ctx, out_host->eval_aln, o.eval_aln, n))) return rc;
    if ((rc = t.finish(launches))) return rc;
    return sx_check_status(ctx, "sx_score_indels");
}
