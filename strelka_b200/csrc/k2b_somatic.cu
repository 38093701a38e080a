// k2b_somatic.cu -- K2b site_gl_somatic: somatic SNV strand-grid model, one warp per tumor/normal site pair.
//
// Replaces somatic_snv_caller_strand_grid::position_somatic_snv_call
//   (/root/reference/src/c++/lib/applications/strelka/position_somatic_snv_strand_grid.cpp:228-363) including
//   CleanPileupFilter                       starling_common/PileupCleaner.cpp:30-64 (tier1 and tier1+tier2 views)
//   get_diploid_gt_lhood_cached_simple      position_somatic_snv_strand_grid_lhood_cached.cpp:41-85
//   get_diploid_het_grid_lhood_cached       :133-153
//   get_diploid_strand_grid_lhood_spi       position_somatic_snv_strand_grid.cpp:61-81 / lhood_cached.cpp:164-234
//   calculate_result_set_grid               qscore_calculator.cpp:47-209
//
// Parity contract.  Every likelihood is a float sum, in pileup order, of values that depend only on (quality, grid state,
// match?, strand?) -- the reference memoises exactly those values in het_ratio_cache; here they are host-built tables
// (sx_context.cu) staged in shared memory, and each of the 21 normal + 21 tumor + 2x9 strand sums is accumulated by one
// lane, so the float results are bit-identical.  The posterior (calculate_result_set_grid) is evaluated in double, its
// exp() terms summed in the reference's loop order; exp / log / log10 are the reference's libm functions restated
// (sx_libm_mirror_d.h).  The nine strand-state likelihoods end in a float log-sum (getLogSum<float>: expf, then log1p in double
// below 0.01f or logf), restated the same way, so they and the strandBias feature are the reference's bits as well.
#include "sx_libm_mirror.h"
#include "sx_device_util.cuh"
#include "sx_internal.h"
#include "sx_result_set_grid.cuh"

#include <algorithm>

namespace
{
constexpr int K2B_WARPS = 4;
constexpr unsigned FULL = 0xffffffffu;
constexpr int NQ = SX_MAX_QSCORE + 1;

struct som_tables
{
    float simple[NQ][3];
    float het[9][NQ][2];
    float strand[9][NQ][2];
    float off_ref[NQ], off_alt[NQ];
    double term_lprior[6][44];
    uint8_t term_tf[6][44], term_nf[6][44];
    uint32_t n_terms[6];
    float geno_prior[6];
};

struct tier_rs // snv_result_set
{
    uint32_t ntype, max_gt;
    int qphred, from_ntype_qphred;
    uint32_t normal_alt_id, tumor_alt_id;
    float strandBias;
};

// one sample, one tier: the 21 grid likelihoods (lanes 0..20), optionally the 9 strand states (lanes 21..29 hold fwd and rev sums),
// alt-allele counts, all-reference flag.  Calls are streamed from global memory (every lane reads the same call: one transaction).
struct sample_acc
{
    float lh;      // lanes 0..20: lhood[lane]; lanes 21..29: lhood[PRESTRAND_SIZE + lane - 21] when with_strand
    uint32_t alt_id;
    bool allref;
    uint32_t n_used;
};

__device__ __forceinline__ sample_acc accumulate_sample(const som_tables& T, const uint32_t* __restrict__ site_off, const uint16_t* __restrict__ calls,
                                                        const uint32_t* __restrict__ t2_off, const uint16_t* __restrict__ t2_calls, uint32_t site,
                                                        uint32_t ref_gt, bool include_tier2, bool with_strand, uint32_t lane, float ln_one_half)
{
    // per-lane term selector
    const float* tb = &T.simple[0][0];
    uint32_t stride = 3, o_match = 0, o_mis = 0;
    if (lane == 0) { o_match = 2; o_mis = 0; }                       // REF
    else if (lane == 1) { o_match = 0; o_mis = 2; }                  // HOM
    else if (lane == 2) { o_match = 1; o_mis = 1; }                  // HET
    else if (lane < 12) { tb = &T.het[lane - 3][0][0]; stride = 2; o_match = 1; o_mis = 0; }          // lhood_low of hetIndex = lane-3
    else if (lane < 21) { tb = &T.het[20 - lane][0][0]; stride = 2; o_match = 0; o_mis = 1; }         // lhood_high of hetIndex = 17-(lane-3)
    const bool strand_lane = with_strand && lane >= 21 && lane < 30;
    const float* sb = strand_lane ? &T.strand[lane - 21][0][0] : &T.strand[0][0][0];

    float lh = 0.f, lh_fwd = 0.f, lh_rev = 0.f;
    uint32_t cnt = 0; // lanes 0..3: count of obs == lane (alt allele tally)
    bool allref = true;
    uint32_t n_used = 0;
    for (int pass = 0; pass < (include_tier2 && t2_off ? 2 : 1); ++pass)
    {
        const uint16_t* cl = pass == 0 ? calls : t2_calls;
        const uint32_t a = pass == 0 ? site_off[site] : t2_off[site], b = pass == 0 ? site_off[site + 1] : t2_off[site + 1];
        for (uint32_t i = a; i < b; ++i)
        {
            const uint32_t c = __ldg(cl + i);
            if ((c >> 12) & 1u)
            {
                // CleanPileupFilter: filtered calls survive only in the tier2 view and only if the filter was tier-specific;
                // filtered tier2_calls never survive
                if (pass == 1 || !(include_tier2 && ((c >> 13) & 1u))) continue;
            }
            ++n_used;
            const uint32_t q = c & 63u, obs = (c >> 6) & 15u, fwd = (c >> 10) & 1u;
            const bool match = (obs == ref_gt);
            if (!match) allref = false;
            if (lane < 21)
            {
                lh = f_add(lh, tb[q * stride + (match ? o_match : o_mis)]);
                if (lane == obs) ++cnt;
            }
            else if (strand_lane)
            {
                const float on = sb[q * 2 + (match ? 0 : 1)];
                const float off = match ? T.off_ref[q] : T.off_alt[q];
                lh_fwd = f_add(lh_fwd, fwd ? on : off);
                lh_rev = f_add(lh_rev, fwd ? off : on);
            }
        }
    }
    if (strand_lane)
    {
        // *lhood = getLogSum(lhood_fwd, lhood_rev) + ln_one_half  (float; tolerance field, see header)
        // getLogSum<float> (blt_util/logSumUtil.hh:33-41): std::exp(float) = expf; log1p_switch<float> = boost::math::log1p(float), which promotes to
        // double and calls log1p, below 0.01f, std::log(1 + x) = logf above -- the reference's libm functions, restated (sx_libm_mirror*.h)
        const float x1 = fmaxf(lh_fwd, lh_rev), x2 = fminf(lh_fwd, lh_rev);
        const float e = sx_expf(f_sub(x2, x1));
        const float l = (fabsf(e) < 0.01f) ? static_cast<float>(sx_log1p(static_cast<double>(e))) : sx_logf(f_add(1.0f, e));
        lh = f_add(f_add(x1, l), ln_one_half);
    }
    // get_most_frequent_alt_id  (blt_common/snp_pos_info.hh:175-198): first strict maximum over base ids != ref
    uint32_t alt_id = ref_gt, max_count = 0;
#pragma unroll
    for (uint32_t bid = 0; bid < 4; ++bid)
    {
        const uint32_t cb = __shfl_sync(FULL, cnt, bid);
        if (cb > max_count && bid != ref_gt)
        {
            max_count = cb;
            alt_id = bid;
        }
    }
    sample_acc o;
    o.lh = lh;
    o.alt_id = alt_id;
    o.allref = allref;
    o.n_used = n_used;
    return o;
}

// calculate_result_set_grid's terms (sx_result_set_grid.cuh): every one is a per-call constant of the context's tables
struct k2b_terms
{
    const som_tables& T;
    __device__ __forceinline__ uint32_t n_terms(uint32_t combo) const { return T.n_terms[combo]; }
    __device__ __forceinline__ double lprior(uint32_t combo, uint32_t i) const { return T.term_lprior[combo][i]; }
    __device__ __forceinline__ uint32_t nf(uint32_t combo, uint32_t i) const { return T.term_nf[combo][i]; }
    __device__ __forceinline__ uint32_t tf(uint32_t combo, uint32_t i) const { return T.term_tf[combo][i]; }
    __device__ __forceinline__ float geno_prior(uint32_t combo) const { return T.geno_prior[combo]; }
};

__global__ void __launch_bounds__(K2B_WARPS * 32) k2b_somatic_kernel(const uint32_t* __restrict__ n_off, const uint16_t* __restrict__ n_calls,
                                                                     const uint32_t* __restrict__ n_t2off, const uint16_t* __restrict__ n_t2calls,
                                                                     const uint32_t* __restrict__ t_off, const uint16_t* __restrict__ t_calls,
                                                                     const uint32_t* __restrict__ t_t2off, const uint16_t* __restrict__ t_t2calls,
                                                                     const char* __restrict__ ref_base, const uint8_t* __restrict__ forced_in, uint32_t n_sites,
                                                                     const sx_tables* __restrict__ tables, sx_ssnv_result* __restrict__ out)
{
    __shared__ som_tables T;
    __shared__ float s_nl[K2B_WARPS][2][32];
    __shared__ float s_tl[K2B_WARPS][2][32];
    __shared__ double s_scr[K2B_WARPS][44];
    {
        float* dst = &T.simple[0][0];
        const float* src = &tables->s_simple[0][0];
        for (int i = threadIdx.x; i < NQ * 3; i += blockDim.x) dst[i] = src[i];
        dst = &T.het[0][0][0];
        src = &tables->s_het[0][0][0];
        for (int i = threadIdx.x; i < 9 * NQ * 2; i += blockDim.x) dst[i] = src[i];
        dst = &T.strand[0][0][0];
        src = &tables->s_strand[0][0][0];
        for (int i = threadIdx.x; i < 9 * NQ * 2; i += blockDim.x) dst[i] = src[i];
        for (int i = threadIdx.x; i < NQ; i += blockDim.x)
        {
            T.off_ref[i] = tables->s_off_ref[i];
            T.off_alt[i] = tables->s_off_alt[i];
        }
        for (int i = threadIdx.x; i < 6 * 44; i += blockDim.x)
        {
            (&T.term_lprior[0][0])[i] = (&tables->s_term_lprior[0][0])[i];
            (&T.term_tf[0][0])[i] = (&tables->s_term_tf[0][0])[i];
            (&T.term_nf[0][0])[i] = (&tables->s_term_nf[0][0])[i];
        }
        if (threadIdx.x < 6)
        {
            T.n_terms[threadIdx.x] = tables->s_n_terms[threadIdx.x];
            T.geno_prior[threadIdx.x] = tables->s_geno_prior[threadIdx.x];
        }
    }
    __syncthreads();
    const float ln_one_half = tables->s_ln_one_half;
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t gwarp = blockIdx.x * K2B_WARPS + warp, nwarps = gridDim.x * K2B_WARPS;
    const bool is_tier2 = (n_t2off != nullptr) && (t_t2off != nullptr);

    for (uint32_t site = gwarp; site < n_sites; site += nwarps)
    {
        sx_ssnv_result* res = out + site;
        {
            uint32_t* w = reinterpret_cast<uint32_t*>(res);
            for (uint32_t i = lane; i < sizeof(sx_ssnv_result) / 4; i += 32) w[i] = 0u;
        }
        __syncwarp();
        const char rb = ref_base[site];
        const uint32_t ref_gt = rb == 'A' ? 0u : rb == 'C' ? 1u : rb == 'G' ? 2u : rb == 'T' ? 3u : 4u;
        if (ref_gt == 4u) continue; // 'N': sgt.is_forced_output=false; return
        const bool forced = forced_in != nullptr && forced_in[site] != 0;
        if (lane == 0) res->ref_gt = ref_gt;

        tier_rs trs[2];
        trs[0] = tier_rs{0, 0, 0, 0, 0, 0, 0.f};
        trs[1] = trs[0];
        bool early = false;
        for (int tier = 0; tier < 2; ++tier)
        {
            if (tier == 1)
            {
                if (!is_tier2) continue;
                if (trs[0].qphred == 0)
                {
                    trs[1] = trs[0];
                    if (lane < 30)
                    {
                        s_nl[warp][1][lane] = s_nl[warp][0][lane];
                        s_tl[warp][1][lane] = s_tl[warp][0][lane];
                    }
                    continue;
                }
            }
            const sample_acc na = accumulate_sample(T, n_off, n_calls, n_t2off, n_t2calls, site, ref_gt, tier == 1, false, lane, ln_one_half);
            const sample_acc ta = accumulate_sample(T, t_off, t_calls, t_t2off, t_t2calls, site, ref_gt, tier == 1, true, lane, ln_one_half);
            if (tier == 0 && !forced && na.allref && ta.allref)
            {
                early = true; // is_spi_allref(normal) && is_spi_allref(tumor)
                break;
            }
            s_nl[warp][tier][lane] = (lane < 21) ? na.lh : 0.f;
            s_tl[warp][tier][lane] = (lane < 30) ? ta.lh : 0.f;
            __syncwarp();
            result_set_grid(k2b_terms{T}, s_nl[warp][tier], s_tl[warp][tier], s_scr[warp], lane, trs[tier]);
            // wrapper (strand_grid.cpp:157-226): returns before the strand-bias block when qphred==0 and not forced
            trs[tier].strandBias = 0.f;
            if (forced || trs[tier].qphred != 0)
            {
                float symm = s_tl[warp][tier][3], strand = s_tl[warp][tier][21];
                for (int k = 4; k < 21; ++k) symm = fmaxf(symm, s_tl[warp][tier][k]);
                for (int k = 22; k < 30; ++k) strand = fmaxf(strand, s_tl[warp][tier][k]);
                trs[tier].strandBias = fmaxf(0.f, f_sub(strand, symm));
            }
            trs[tier].normal_alt_id = na.alt_id;
            trs[tier].tumor_alt_id = ta.alt_id;
        }
        if (early) continue;
        if (!forced)
        {
            if ((trs[0].qphred == 0) || (is_tier2 && (trs[1].qphred == 0))) continue;
        }
        uint32_t snv_tier = 0, snv_from_ntype_tier = 0;
        if (is_tier2)
        {
            if (trs[0].qphred > trs[1].qphred) snv_tier = 1;
            if (trs[0].from_ntype_qphred > trs[1].from_ntype_qphred) snv_from_ntype_tier = 1;
        }
        tier_rs rs = trs[snv_from_ntype_tier];
        if (is_tier2 && (trs[0].ntype != trs[1].ntype))
        {
            rs.ntype = 3; // NTYPE::CONFLICT
            rs.from_ntype_qphred = 0;
        }
        rs.qphred = trs[snv_tier].qphred;
        if (lane < 30)
        {
            res->normal_lhood[lane] = s_nl[warp][snv_from_ntype_tier][lane];
            res->tumor_lhood[lane] = s_tl[warp][snv_from_ntype_tier][lane];
        }
        if (lane == 0)
        {
            res->strandBias = rs.strandBias;
            res->is_computed = 1;
            res->snv_tier = snv_tier;
            res->snv_from_ntype_tier = snv_from_ntype_tier;
            res->ntype = rs.ntype;
            res->max_gt = rs.max_gt;
            res->qphred = rs.qphred;
            res->from_ntype_qphred = rs.from_ntype_qphred;
            res->normal_alt_id = rs.normal_alt_id;
            res->tumor_alt_id = rs.tumor_alt_id;
        }
        __syncwarp();
    }
}

} // namespace

int sx_k2b_run(sx_ctx* ctx, const sx_pileup_batch* n, const sx_pileup_batch* t, const uint8_t* forced_dev, sx_ssnv_result* out_dev, unsigned* launches)
{
    const int grid = static_cast<int>(std::min<uint32_t>((n->n_sites + K2B_WARPS - 1) / K2B_WARPS, (uint32_t)ctx->sm_count * 8));
    k2b_somatic_kernel<<<grid, K2B_WARPS * 32, 0, ctx->s_compute>>>(n->site_off, n->calls, n->t2_off, n->t2_calls, t->site_off, t->calls, t->t2_off, t->t2_calls,
                                                                  n->ref_base, forced_dev, n->n_sites, ctx->d_tables, out_dev);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

extern "C" int sx_site_gl_somatic_dev(sx_ctx* ctx, const sx_pileup_batch* n, const sx_pileup_batch* t, const uint8_t* forced_dev, sx_ssnv_result* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!n || !t || !out_dev) return sx_fail(ctx, SX_ERR_ARG, "sx_site_gl_somatic_dev: NULL argument");
    if (n->n_sites != t->n_sites) return sx_fail(ctx, SX_ERR_ARG, "sx_site_gl_somatic_dev: normal and tumor batches differ in n_sites");
    if (n->n_sites == 0) return SX_OK;
    return sx_run_timed(ctx, [&](unsigned* launches) { return sx_k2b_run(ctx, n, t, forced_dev, out_dev, launches); });
}

extern "C" int sx_site_gl_somatic(sx_ctx* ctx, const sx_pileup_batch* n, const sx_pileup_batch* t, const uint8_t* forced_host, sx_ssnv_result* out_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!n || !t || !out_host) return sx_fail(ctx, SX_ERR_ARG, "sx_site_gl_somatic: NULL argument");
    if (n->n_sites != t->n_sites) return sx_fail(ctx, SX_ERR_ARG, "sx_site_gl_somatic: normal and tumor batches differ in n_sites");
    if (n->n_sites == 0) return SX_OK;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer tm(ctx);
    sx_pileup_batch dn, dt;
    uint32_t m = 0;
    int rc = sx_upload_pileup(ctx, n, 9, &dn, &m);
    if (rc) return rc;
    if ((rc = sx_upload_pileup(ctx, t, 15, &dt, &m))) return rc;
    const uint8_t* d_forced = nullptr;
    if (forced_host && (rc = sx_upload(ctx, sx_host_slot(21), forced_host, n->n_sites, d_forced, 0))) return rc;
    sx_ssnv_result* d_out = nullptr;
    if ((rc = sx_take(ctx, sx_host_slot(22), n->n_sites, d_out, 0))) return rc;
    unsigned launches = 0;
    if ((rc = sx_k2b_run(ctx, &dn, &dt, d_forced, d_out, &launches))) return rc;
    if ((rc = sx_download(ctx, out_host, d_out, n->n_sites))) return rc;
    return tm.finish(launches);
}
