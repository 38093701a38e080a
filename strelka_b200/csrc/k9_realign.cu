// k9_realign.cu -- K9 choose_realignment: from the scored candidate alignments to rseg.realignment, one read per thread.
//
// Replaces (include/strelka_b200.h, "K9 choose_realignment"; SURVEY 8a row a2) the tail of scoreCandidateAlignments
// (starling_common/starling_read_align.cpp:1573-1741) with finishRealignment :1411-1450 and starling_read_align_clipper.cpp.  Per-read
// body: k9_core.cuh.
//
// Shape of the work: per read two or three passes over its few alignments' segments (arg-max, pool preference, conflict marking); the
// conflicts are found on segment overlaps, 32 read positions at a time, so nothing per read position is stored.  Reads in the scores
// where K1 wrote them and the alignments where K7 wrote them; writes one (pos, path) per read where K4 reads a read's best alignment.
// HBM-bound by construction (~40 B per alignment in, ~30 B per read out).  Launches: slots per read -> scan -> choose.

#include "k9_core.cuh"
#include "sx_internal.h"
#include "sx_read_index.cuh"

#include <algorithm>

namespace
{
// the slot counts go into seg_off, which the scan turns into the offsets
__global__ void k9_slots_kernel(const sx_realign_batch b, uint32_t* __restrict__ cnt)
{
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < b.n_reads; r += gridDim.x * blockDim.x) cnt[r] = k9_slots(b, r);
}

// read_region: the read index's (the window pass), or NULL: a binary search of region_read_off per read (K9's own entry points)
__global__ void __launch_bounds__(128) k9_choose_kernel(const k9_view v, const uint32_t* __restrict__ read_region, const sx_realign_out o, int* __restrict__ status)
{
    if (o.totals[0] > o.cap_segs)
    {
        if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(status, SX_ST_K9_CAP);
        return;
    }
    k9_scratch S = {nullptr, nullptr}; // (the reference map is not stored)
    const uint32_t n(v.b.n_reads);
    for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x)
    {
        const uint32_t s0(o.seg_off[r]), s1(o.seg_off[r + 1]);
        int32_t p;
        uint16_t ns;
        uint32_t best;
        const uint32_t g(read_region ? read_region[r] : sxi_region_of(v.b.region_read_off, v.b.n_regions, r));
        const uint32_t st(k9_read(v, g, r, S, o.segs + s0, s1 - s0, p, ns, best));
        if (!(st & SX_REALIGN_ST_REALIGNED)) k9_fallback(v.b, r, o.segs + s0, s1 - s0, p, ns);
        o.pos[r] = p;
        o.n_seg[r] = ns;
        o.status[r] = (uint8_t)st;
        o.best_aln[r] = best;
    }
}
} // namespace

// K9's launcher
int sx_k9_run(sx_ctx* ctx, const sx_realign_batch* d, const double* lnp, const sx_realign_out* o, const uint32_t* read_region, unsigned* launches)
{
    if (d->n_reads == 0) return SX_OK;
    cudaStream_t st(ctx->s_compute);
    const uint32_t n(d->n_reads);
    int rc;
    const int cap(ctx->sm_count * 16);
    const auto grid = [cap](const uint32_t m) { return (unsigned)std::max(1, std::min<int>((int)((m + 127) / 128), cap)); };
    k9_slots_kernel<<<grid(n), 128, 0, st>>>(*d, o->seg_off);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    const sx_scan_set J = {1, {{o->seg_off, n, SX_SCAN_EXCLUSIVE | SX_SCAN_CLOSE, o->totals}}};
    if ((rc = sx_scan(ctx, SX_SLOT_K7A_K9_SUMS, J, launches))) return rc;
    k9_view v;
    v.b = *d;
    v.lnp = lnp;
    k9_choose_kernel<<<grid(n), 128, 0, st>>>(v, read_region, *o, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

namespace
{
int k9_check_args(sx_ctx* ctx, const sx_realign_batch* b, const double* lnp, const sx_realign_out* o, const char* what)
{
    if (!b || !o) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (!o->totals || !o->seg_off) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    if (b->n_reads == 0) return SX_OK;
    if (!b->region_read_off || !b->region_key_off || !b->aln_off || !b->aln_pos || !b->aln_seg_off || !b->segs || !b->aln_key_off || !b->aln_keys || !b->read_len ||
        (b->n_alns && !lnp) || !o->pos || !o->n_seg || !o->status || !o->best_aln || !o->segs)
        return sx_fail(ctx, SX_ERR_ARG, "%s: NULL array", what);
    if (b->n_regions == 0) return sx_fail(ctx, SX_ERR_ARG, "%s: reads without a region", what);
    return SX_OK;
}
} // namespace

extern "C" int sx_choose_realignment_dev(sx_ctx* ctx, const sx_realign_batch* d, const double* lnp_dev, sx_realign_out* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k9_check_args(ctx, d, lnp_dev, out_dev, "sx_choose_realignment_dev"))) return rc;
    if (d->n_reads == 0)
    {
        SX_CUDA(ctx, cudaSetDevice(ctx->device));
        SX_CUDA(ctx, cudaMemsetAsync(out_dev->totals, 0, 4, ctx->s_compute));
        SX_CUDA(ctx, cudaMemsetAsync(out_dev->seg_off, 0, 4, ctx->s_compute));
        SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
        return SX_OK;
    }
    if ((rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k9_run(ctx, d, lnp_dev, out_dev, nullptr, launches); }))) return rc;
    return sx_check_status(ctx, "sx_choose_realignment", SX_ST_K9_CAP);
}

extern "C" int sx_choose_realignment(sx_ctx* ctx, const sx_realign_batch* b, const double* lnp_host, sx_realign_out* out_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = k9_check_args(ctx, b, lnp_host, out_host, "sx_choose_realignment"))) return rc;
    if (b->n_reads == 0)
    {
        out_host->totals[0] = 0;
        out_host->seg_off[0] = 0;
        return SX_OK;
    }
    if (b->aln_off[b->n_reads] != b->n_alns) return sx_fail(ctx, SX_ERR_ARG, "sx_choose_realignment: aln_off does not end at n_alns");
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer t(ctx);
    sx_realign_batch d(*b);
    const size_t n(b->n_reads), n_segs(b->aln_seg_off[b->n_alns]), n_keys(b->aln_key_off[b->n_alns]), n_win(b->region_key_off[b->n_regions]);
    if ((rc = sx_upload(ctx, sx_host_slot(0), b->region_read_off, (size_t)b->n_regions + 1, d.region_read_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(1), b->region_key_off, (size_t)b->n_regions + 1, d.region_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(2), b->keys, n_win, d.keys, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(3), b->aln_off, n + 1, d.aln_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(4), b->aln_pos, b->n_alns, d.aln_pos, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(5), b->aln_seg_off, (size_t)b->n_alns + 1, d.aln_seg_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(6), b->segs, n_segs, d.segs, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(7), b->aln_key_off, (size_t)b->n_alns + 1, d.aln_key_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(8), b->aln_keys, n_keys, d.aln_keys, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(9), b->read_len, n, d.read_len, 16))) return rc;
    if (b->pin_flags && (rc = sx_upload(ctx, sx_host_slot(10), b->pin_flags, n, d.pin_flags, 16))) return rc;
    const double* d_lnp(nullptr);
    if ((rc = sx_upload(ctx, sx_host_slot(11), lnp_host, b->n_alns, d_lnp, 16))) return rc;
    sx_realign_out o(*out_host);
    if ((rc = sx_take(ctx, sx_host_slot(12), 4, o.totals, 0))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(13), n + 1, o.seg_off, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(14), n, o.pos, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(15), n, o.n_seg, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(16), n, o.status, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(17), n, o.best_aln, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(18), o.cap_segs, o.segs, 16))) return rc;
    unsigned launches(0);
    if ((rc = sx_k9_run(ctx, &d, d_lnp, &o, nullptr, &launches))) return rc;
    if ((rc = sx_download(ctx, out_host->totals, o.totals, 1))) return rc;
    if ((rc = sx_download(ctx, out_host->seg_off, o.seg_off, n + 1))) return rc;
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    if (out_host->totals[0] <= o.cap_segs)
    {
        if ((rc = sx_download(ctx, out_host->pos, o.pos, n))) return rc;
        if ((rc = sx_download(ctx, out_host->n_seg, o.n_seg, n))) return rc;
        if ((rc = sx_download(ctx, out_host->status, o.status, n))) return rc;
        if ((rc = sx_download(ctx, out_host->best_aln, o.best_aln, n))) return rc;
        if ((rc = sx_download(ctx, out_host->segs, o.segs, out_host->totals[0]))) return rc;
    }
    if ((rc = t.finish(launches))) return rc;
    return sx_check_status(ctx, "sx_choose_realignment", SX_ST_K9_CAP, out_host->totals);
}
