// k2c_continuous.cu -- K2c site_continuous: the germline caller's continuous-frequency site model (include/strelka_b200.h, "K2c
// site_continuous"; the body is k2c_core.cuh).
//
// Three steps, one warp per site in both kernels:
//   k2c_count_kernel   one pass over each sample's column: CleanPileupFilter (the filter bit, as K2a reads it) and the strand x base, ANY
//                      and raw counts in registers, reduced across the warp; each site's counts to a scratch row and its record count
//   sx_scan            record counts -> offsets (sx_scan.cu); the total comes back to the host for the capacity check
//   k2c_write_kernel   each site's loci from its counts: lane (locus, sample) evaluates that entry's qscore and strand bias, the lane of
//                      sample 0 the locus; records at the site's offset
// Columns of the mitochondrial data are thousands of calls deep, so a whole warp streams each column (as K2a does its deep sites); the
// count pass is the only one that reads the calls, the write pass reads 44 bytes per sample and site.  The output does not depend on
// scheduling: every record's place is fixed by the scan.
#include "k2c_core.cuh"
#include "sx_internal.h"

#include <algorithm>
#include <cmath>

namespace
{
constexpr int K2C_WARPS = 8;
constexpr unsigned FULL = 0xffffffffu;
constexpr uint32_t K2C_WORDS = sizeof(k2c_counts) / 4; // 11
static_assert(sizeof(k2c_counts) == 44, "k2c_counts is 11 words");

__global__ void __launch_bounds__(K2C_WARPS * 32) k2c_count_kernel(const sx_cont_batch b, const double min_het_vf, k2c_counts* __restrict__ counts,
                                                                  uint32_t* __restrict__ n_rec)
{
    __shared__ k2c_counts s_c[K2C_WARPS][SX_CONT_MAX_SAMPLES];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t S = b.n_samples;
    for (uint32_t site = blockIdx.x * K2C_WARPS + warp; site < b.n_sites; site += gridDim.x * K2C_WARPS)
    {
        for (uint32_t s = 0; s < S; ++s)
        {
            const sx_pileup_batch& p = b.sample[s];
            const uint32_t c0 = p.site_off[site], c1 = p.site_off[site + 1];
            uint32_t k[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0}; // index 5 * is_fwd + base
            for (uint32_t i = c0 + lane; i < c1; i += 32)
            {
                const uint32_t c = p.calls[i];
                const uint32_t idx = k2c_is_filtered(c) ? 10u : 5u * k2c_is_fwd(c) + k2c_base_of(c);
#pragma unroll
                for (uint32_t j = 0; j < 10; ++j) k[j] += (idx == j) ? 1u : 0u;
            }
#pragma unroll
            for (uint32_t j = 0; j < 10; ++j) k[j] = __reduce_add_sync(FULL, k[j]);
            if (lane == 0)
            {
                k2c_counts& c = s_c[warp][s];
                for (uint32_t j = 0; j < 10; ++j) c.n[j / 5][j % 5] = k[j];
                c.raw = c1 - c0;
            }
        }
        __syncwarp();
        for (uint32_t i = lane; i < S * K2C_WORDS; i += 32)
            reinterpret_cast<uint32_t*>(counts + (size_t)site * S)[i] = reinterpret_cast<const uint32_t*>(&s_c[warp][0])[i];
        if (lane == 0)
        {
            uint8_t loci[5];
            const bool forced = b.forced_output && b.forced_output[site];
            n_rec[site] = k2c_site_loci(&s_c[warp][0], S, k2c_ref_id(b.sample[0].ref_base[site]), forced, min_het_vf, loci);
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(K2C_WARPS * 32) k2c_write_kernel(const sx_cont_batch b, const sx_cont_opts o, const double err_rate,
                                                                  const k2c_counts* __restrict__ counts, const uint32_t* __restrict__ rec_off,
                                                                  sx_cont_locus* __restrict__ loci_out, sx_cont_sample* __restrict__ samples_out)
{
    __shared__ k2c_counts s_c[K2C_WARPS][SX_CONT_MAX_SAMPLES];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t S = b.n_samples;
    for (uint32_t site = blockIdx.x * K2C_WARPS + warp; site < b.n_sites; site += gridDim.x * K2C_WARPS)
    {
        const uint32_t r0 = rec_off[site];
        if (rec_off[site + 1] == r0) continue; // (warp-uniform)
        for (uint32_t i = lane; i < S * K2C_WORDS; i += 32)
            reinterpret_cast<uint32_t*>(&s_c[warp][0])[i] = reinterpret_cast<const uint32_t*>(counts + (size_t)site * S)[i];
        __syncwarp();
        const uint32_t ref = k2c_ref_id(b.sample[0].ref_base[site]);
        const bool forced = b.forced_output && b.forced_output[site];
        uint8_t loci[5];
        const uint32_t m = k2c_site_loci(&s_c[warp][0], S, ref, forced, o.min_het_vf, loci);
        // lane = locus * S + sample: m * S <= 4 * SX_CONT_MAX_SAMPLES = 32
        const uint32_t li = lane / S, s = lane % S;
        const bool active = li < m;
        int32_t gq = 0;
        if (active)
        {
            const sx_cont_sample e = k2c_entry(s_c[warp][s], ref, loci[li], o, err_rate);
            samples_out[(size_t)(r0 + li) * S + s] = e;
            gq = e.gq;
        }
        int32_t qual = 0;
        for (uint32_t t = 0; t < S; ++t) qual = max(qual, __shfl_sync(FULL, gq, min(li * S + t, 31u)));
        if (active && s == 0)
            loci_out[r0 + li] = k2c_locus(&s_c[warp][0], S, b.pos_begin + static_cast<int32_t>(site), ref, loci[li], forced, qual);
        __syncwarp();
    }
}

__global__ void k2c_qscore_kernel(const uint32_t n_pairs, const uint32_t* __restrict__ a, const uint32_t* __restrict__ n, const double err_rate,
                                  const int32_t max_q, int32_t* __restrict__ gq, uint32_t* __restrict__ status)
{
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_pairs; i += gridDim.x * blockDim.x)
    {
        const k2c_q q = k2c_qscore(a[i], n[i], err_rate, max_q);
        gq[i] = q.gq;
        status[i] = q.status;
    }
}

double err_rate_of(const sx_cont_opts* o) { return std::pow(10., -static_cast<double>(o->expected_qscore) / 10.); } // qphred_to_error_prob

int check_opts(sx_ctx* ctx, const char* what, const sx_cont_opts* o)
{
    if (!o) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL options", what);
    if (!(o->min_het_vf > 0.0 && o->min_het_vf < 0.5)) return sx_fail(ctx, SX_ERR_ARG, "%s: min_het_vf outside (0, 0.5)", what);
    if (!(o->max_abs_sample_strand_bias >= 0.0)) return sx_fail(ctx, SX_ERR_ARG, "%s: max_abs_sample_strand_bias below 0", what);
    if (o->expected_qscore < 0 || o->expected_qscore > SX_MAX_QSCORE) return sx_fail(ctx, SX_ERR_ARG, "%s: expected_qscore outside 0..%d", what, SX_MAX_QSCORE);
    if (o->max_qscore < 0 || o->max_qscore > 1000) return sx_fail(ctx, SX_ERR_ARG, "%s: max_qscore outside 0..1000", what);
    return SX_OK;
}

int check_batch(sx_ctx* ctx, const char* what, const sx_cont_batch* b, const sx_cont_out* o)
{
    if (!b || !o) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (b->n_samples < 1 || b->n_samples > SX_CONT_MAX_SAMPLES) return sx_fail(ctx, SX_ERR_ARG, "%s: n_samples outside 1..%d", what, SX_CONT_MAX_SAMPLES);
    for (uint32_t s = 0; s < b->n_samples; ++s)
    {
        const sx_pileup_batch& p = b->sample[s];
        if (p.n_sites != b->n_sites) return sx_fail(ctx, SX_ERR_ARG, "%s: sample %u has %u sites, the batch %u", what, s, p.n_sites, b->n_sites);
        if (!p.site_off || !p.calls || (s == 0 && !p.ref_base)) return sx_fail(ctx, SX_ERR_ARG, "%s: sample %u: NULL array", what, s);
    }
    if (b->n_sites && ((o->cap_loci && (!o->loci || !o->samples)))) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL output array", what);
    return SX_OK;
}

int grid_of(sx_ctx* ctx, uint32_t n_sites) { return static_cast<int>(std::min<uint32_t>((n_sites + K2C_WARPS - 1) / K2C_WARPS, (uint32_t)ctx->sm_count * 16)); }
} // namespace

// K2c's launcher: count, scan, (host: the total), write.  totals_host[0] = records; SX_ERR_CAPACITY past cap_loci with the offsets written.
int sx_k2c_run(sx_ctx* ctx, const sx_cont_opts* o, const sx_cont_batch* d, const sx_cont_out* out, uint32_t* totals_host, unsigned* launches)
{
    const uint32_t n = d->n_sites, S = d->n_samples;
    k2c_counts* counts = nullptr;
    uint32_t *rec_off = nullptr, *total = nullptr;
    int rc;
    if ((rc = sx_take(ctx, SX_SLOT_K2C_COUNTS, (size_t)n * S, counts, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K2C_REC_OFF, (size_t)n + 1, rec_off, 16))) return rc;
    if ((rc = sx_take(ctx, SX_SLOT_K2C_TOTAL, 1, total, 0))) return rc;
    const int grid = grid_of(ctx, n);
    k2c_count_kernel<<<grid, K2C_WARPS * 32, 0, ctx->s_compute>>>(*d, o->min_het_vf, counts, rec_off);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    sx_scan_set job{};
    job.n_arrays = 1;
    job.a[0] = sx_scan_array{rec_off, n, SX_SCAN_EXCLUSIVE | SX_SCAN_CLOSE, total};
    if ((rc = sx_scan(ctx, SX_SLOT_K2C_SUMS, job, launches))) return rc;
    if (out->site_rec_off) SX_CUDA(ctx, cudaMemcpyAsync(out->site_rec_off, rec_off, ((size_t)n + 1) * 4, cudaMemcpyDeviceToDevice, ctx->s_compute));
    uint32_t t = 0;
    SX_CUDA(ctx, cudaMemcpyAsync(&t, total, 4, cudaMemcpyDeviceToHost, ctx->s_compute));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    if (totals_host) totals_host[0] = t;
    if (t > out->cap_loci) return sx_fail(ctx, SX_ERR_CAPACITY, "sx_site_continuous: cap_loci too small: %u records needed", t);
    if (t == 0) return SX_OK;
    k2c_write_kernel<<<grid, K2C_WARPS * 32, 0, ctx->s_compute>>>(*d, *o, err_rate_of(o), counts, rec_off, out->loci, out->samples);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

extern "C" void sx_default_cont_opts(sx_cont_opts* o)
{
    if (!o) return;
    o->min_het_vf = 0.01;                 // starling_base_options::min_het_vf
    o->max_abs_sample_strand_bias = 99.0; // starling_options::maxAbsSampleVariantStrandBias
    o->expected_qscore = 17;              // continuousFrequencyCallerExpectedObservationQuality
    o->max_qscore = 40;                   // continuousFrequencyCallerMaxQscore
}

extern "C" int sx_site_continuous_dev(sx_ctx* ctx, const sx_cont_opts* opts, const sx_cont_batch* d, const sx_cont_out* out, uint32_t* totals_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = check_opts(ctx, "sx_site_continuous_dev", opts)) || (rc = check_batch(ctx, "sx_site_continuous_dev", d, out))) return rc;
    if (d->n_sites == 0)
    {
        if (totals_host) totals_host[0] = 0;
        if (out->site_rec_off) SX_CUDA(ctx, cudaMemsetAsync(out->site_rec_off, 0, 4, ctx->s_compute));
        SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
        return SX_OK;
    }
    rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k2c_run(ctx, opts, d, out, totals_host, launches); });
    if (rc) return rc;
    return sx_check_status(ctx, "sx_site_continuous_dev");
}

extern "C" int sx_site_continuous(sx_ctx* ctx, const sx_cont_opts* opts, const sx_cont_batch* b, const sx_cont_out* out, uint32_t* totals_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = check_opts(ctx, "sx_site_continuous", opts)) || (rc = check_batch(ctx, "sx_site_continuous", b, out))) return rc;
    const uint32_t n = b->n_sites, S = b->n_samples;
    if (n == 0)
    {
        if (totals_host) totals_host[0] = 0;
        if (out->site_rec_off) out->site_rec_off[0] = 0;
        return SX_OK;
    }
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer timer(ctx);
    sx_cont_batch d = *b;
    for (uint32_t s = 0; s < S; ++s)
    {
        const sx_pileup_batch& p = b->sample[s];
        for (uint32_t i = 0; i < n; ++i)
            if (p.site_off[i + 1] < p.site_off[i]) return sx_fail(ctx, SX_ERR_ARG, "sx_site_continuous: sample %u: site_off not monotone at site %u", s, i);
        if ((rc = sx_upload(ctx, sx_host_slot(2 * s), p.site_off, (size_t)n + 1, d.sample[s].site_off, 16))) return rc;
        if ((rc = sx_upload(ctx, sx_host_slot(2 * s + 1), p.calls, p.site_off[n], d.sample[s].calls, 16))) return rc;
        d.sample[s].t2_off = nullptr;
        d.sample[s].t2_calls = nullptr;
        d.sample[s].ploidy = nullptr;
        d.sample[s].ref_base = nullptr;
    }
    if ((rc = sx_upload(ctx, sx_host_slot(16), b->sample[0].ref_base, n, d.sample[0].ref_base, 16))) return rc;
    if (b->forced_output && (rc = sx_upload(ctx, sx_host_slot(17), b->forced_output, n, d.forced_output, 16))) return rc;
    sx_cont_out o{};
    o.cap_loci = out->cap_loci;
    if ((rc = sx_take(ctx, sx_host_slot(18), o.cap_loci, o.loci, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(19), (size_t)o.cap_loci * S, o.samples, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(20), (size_t)n + 1, o.site_rec_off, 16))) return rc;
    unsigned launches = 0;
    uint32_t t = 0;
    rc = sx_k2c_run(ctx, opts, &d, &o, &t, &launches);
    if (totals_host) totals_host[0] = t;
    if (rc && rc != SX_ERR_CAPACITY) return rc;
    if (out->site_rec_off)
    {
        const int rd = sx_download(ctx, out->site_rec_off, o.site_rec_off, (size_t)n + 1);
        if (rd) return rd;
    }
    if (rc == SX_ERR_CAPACITY)
    {
        SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
        return rc;
    }
    if ((rc = sx_download(ctx, out->loci, o.loci, t))) return rc;
    if ((rc = sx_download(ctx, out->samples, o.samples, (size_t)t * S))) return rc;
    if ((rc = timer.finish(launches))) return rc;
    return sx_check_status(ctx, "sx_site_continuous");
}

namespace
{
int qscore_run(sx_ctx* ctx, const sx_cont_opts* o, uint32_t n_pairs, const uint32_t* a, const uint32_t* n, int32_t* gq, uint32_t* status, unsigned* launches)
{
    const int grid = static_cast<int>(std::min<uint32_t>((n_pairs + 255) / 256, (uint32_t)ctx->sm_count * 16));
    k2c_qscore_kernel<<<grid, 256, 0, ctx->s_compute>>>(n_pairs, a, n, err_rate_of(o), o->max_qscore, gq, status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}
} // namespace

extern "C" int sx_cont_qscore_dev(sx_ctx* ctx, const sx_cont_opts* opts, uint32_t n_pairs, const uint32_t* a, const uint32_t* n, int32_t* gq, uint32_t* status)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = check_opts(ctx, "sx_cont_qscore_dev", opts))) return rc;
    if (n_pairs == 0) return SX_OK;
    if (!a || !n || !gq || !status) return sx_fail(ctx, SX_ERR_ARG, "sx_cont_qscore_dev: NULL argument");
    return sx_run_timed(ctx, [&](unsigned* launches) { return qscore_run(ctx, opts, n_pairs, a, n, gq, status, launches); });
}

extern "C" int sx_cont_qscore(sx_ctx* ctx, const sx_cont_opts* opts, uint32_t n_pairs, const uint32_t* a, const uint32_t* n, int32_t* gq, uint32_t* status)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc;
    if ((rc = check_opts(ctx, "sx_cont_qscore", opts))) return rc;
    if (n_pairs == 0) return SX_OK;
    if (!a || !n || !gq || !status) return sx_fail(ctx, SX_ERR_ARG, "sx_cont_qscore: NULL argument");
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer timer(ctx);
    const uint32_t *da = nullptr, *dn = nullptr;
    int32_t* dq = nullptr;
    uint32_t* ds = nullptr;
    if ((rc = sx_upload(ctx, sx_host_slot(0), a, n_pairs, da, 16)) || (rc = sx_upload(ctx, sx_host_slot(1), n, n_pairs, dn, 16))) return rc;
    if ((rc = sx_take(ctx, sx_host_slot(2), n_pairs, dq, 16)) || (rc = sx_take(ctx, sx_host_slot(3), n_pairs, ds, 16))) return rc;
    unsigned launches = 0;
    if ((rc = qscore_run(ctx, opts, n_pairs, da, dn, dq, ds, &launches))) return rc;
    if ((rc = sx_download(ctx, gq, dq, n_pairs)) || (rc = sx_download(ctx, status, ds, n_pairs))) return rc;
    return timer.finish(launches);
}
