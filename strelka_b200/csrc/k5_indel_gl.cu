// k5_indel_gl.cu -- K5 indel_gl: indel genotype log-likelihoods of an orthogonal allele group from per-read allele likelihoods.
//
// Replaces the per-read loop of getVariantAlleleGroupGenotypeLhoodsForSample
//   (/root/reference/src/c++/lib/starling_common/AlleleGroupGenotype.cpp:184-258):
//   updateGenotypeLogLhoodFromAlleleLogLhood :34-111, updateSupportingReadStats :122-152,
//   integrateOutMappingStatus  starling_common/readMappingAdjustmentUtil.hh:46-56,
//   get_het_observed_allele_ratio  starling_common/starling_indel_call_pprob_digt.cpp:40-71.
//
// One warp per locus.  32 reads at a time: each lane evaluates its read's term for every genotype (double log-sum-exp with the
// reference's log1p switch) into shared memory; lanes 0..G-1 then add the 32 terms of "their" genotype in read order, so the double
// sums keep the reference's order.  Supporting-read counts come from ballots.  exp / log / log1p are the libm mirrors of
// sx_libm_mirror_d.h, so the double likelihoods are the reference's bits (tests/test_gpu_parity.py::test_k5_indel_gl compares them bit for
// bit), and the integer counts are exact.
#include "sx_device_util.cuh"
#include "sx_internal.h"
#include "sx_log_sum.cuh"

#include <algorithm>

namespace
{
constexpr int K5_WARPS = 4;
constexpr unsigned FULL = 0xffffffffu;

__global__ void __launch_bounds__(K5_WARPS * 32) k5_indel_gl_kernel(const uint32_t* __restrict__ read_off, const uint32_t* __restrict__ lnp_off,
                                                                    const uint32_t* __restrict__ allele_off, const uint8_t* __restrict__ ploidy,
                                                                    const uint16_t* __restrict__ del_len, const uint16_t* __restrict__ ins_len,
                                                                    const float* __restrict__ allele_lnp, const uint16_t* __restrict__ read_length,
                                                                    const uint16_t* __restrict__ non_ambig, const uint8_t* __restrict__ is_fwd, uint32_t n_loci,
                                                                    const sx_tables* __restrict__ tables, sx_indel_result* __restrict__ out, int* __restrict__ status)
{
    __shared__ double s_term[K5_WARPS][SX_INDEL_MAX_GT][32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double randomBaseMatchLogProb = tables->i_randomBaseMatchLogProb;
    const double correctMappingLogPrior = tables->i_correctMappingLogPrior;
    const double loghalf = tables->i_loghalf;
    const double threshold = tables->i_readSupportThreshold;
    const uint32_t min_overlap = static_cast<uint32_t>(tables->i_min_flank);

    for (uint32_t l = blockIdx.x * K5_WARPS + warp; l < n_loci; l += gridDim.x * K5_WARPS)
    {
        sx_indel_result* res = out + l;
        const uint32_t A = allele_off[l + 1] - allele_off[l];
        const uint32_t pl = ploidy[l];
        if (A < 1 || A > SX_INDEL_MAX_ALLELES || (pl != 1 && pl != 2))
        {
            if (lane == 0) atomicOr(status, SX_ST_INDEL_ALLELES);
            continue;
        }
        const uint32_t nfull = A + 1;
        const uint32_t G = (pl == 1) ? nfull : (nfull * (nfull + 1)) / 2;
        uint32_t dl[SX_INDEL_MAX_ALLELES], il[SX_INDEL_MAX_ALLELES];
#pragma unroll
        for (uint32_t a = 0; a < SX_INDEL_MAX_ALLELES; ++a)
        {
            dl[a] = a < A ? del_len[allele_off[l] + a] : 0;
            il[a] = a < A ? ins_len[allele_off[l] + a] : 0;
        }
        const uint32_t r0 = read_off[l], r1 = read_off[l + 1];
        double gl = 0.0;                        // lanes < G: genotype `lane`
        uint32_t cnt[2][SX_INDEL_MAX_ALLELES + 2]; // warp-uniform counters
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
            for (int a = 0; a < SX_INDEL_MAX_ALLELES + 2; ++a) cnt[s][a] = 0;

        for (uint32_t rb = r0; rb < r1; rb += 32)
        {
            const uint32_t r = rb + lane;
            const bool valid = r < r1;
            uint32_t choice = SX_INDEL_MAX_ALLELES + 1, fwd = 0;
            if (valid)
            {
                const float* lp = allele_lnp + lnp_off[l] + static_cast<size_t>(r - r0) * nfull;
                double L[SX_INDEL_MAX_ALLELES + 1];
#pragma unroll
                for (uint32_t a = 0; a <= SX_INDEL_MAX_ALLELES; ++a) L[a] = a < nfull ? static_cast<double>(lp[a]) : 0.0;
                const uint32_t rlen = read_length[r];
                const uint32_t nonamb = non_ambig[r];
                fwd = is_fwd[r] ? 1u : 0u;
                const double incorrect = d_mul(randomBaseMatchLogProb, static_cast<double>(nonamb)); // getIncorrectMappingLogLikelihood
                // get_het_observed_allele_ratio per allele (het_allele_ratio = 0.5); outputs stay ln(1/2) when total_path_term == 0
                double lr[SX_INDEL_MAX_ALLELES], li[SX_INDEL_MAX_ALLELES];
                const uint32_t base_expect = ((rlen + 1) < (2 * min_overlap)) ? 0u : (rlen + 1) - (2 * min_overlap);
#pragma unroll
                for (uint32_t a = 0; a < SX_INDEL_MAX_ALLELES; ++a)
                {
                    const double ref_path_expect = static_cast<double>(base_expect + min(dl[a], base_expect));
                    const double indel_path_expect = static_cast<double>(base_expect + min(il[a], base_expect));
                    const double ref_path_term = d_mul(0.5, ref_path_expect);
                    const double indel_path_term = d_mul(0.5, indel_path_expect);
                    const double total = d_add(ref_path_term, indel_path_term);
                    lr[a] = loghalf;
                    li[a] = loghalf;
                    if (a < A && total > 0)
                    {
                        const double indel_prob = d_div(indel_path_term, total);
                        lr[a] = sx_log(d_sub(1.0, indel_prob));
                        li[a] = sx_log(indel_prob);
                    }
                }
                if (pl == 1)
                {
#pragma unroll
                    for (uint32_t a0 = 0; a0 <= SX_INDEL_MAX_ALLELES; ++a0)
                        if (a0 < nfull) s_term[warp][a0][lane] = get_log_sum(d_add(L[a0], correctMappingLogPrior), incorrect);
                }
                else
                {
#pragma unroll
                    for (uint32_t a1 = 0; a1 <= SX_INDEL_MAX_ALLELES; ++a1)
                    {
#pragma unroll
                        for (uint32_t a0 = 0; a0 <= a1; ++a0)
                        {
                            if (a1 >= nfull) continue;
                            const uint32_t g = a0 + (a1 * (a1 + 1)) / 2;
                            double raw;
                            if (a0 != a1)
                            {
                                double p0, p1;
                                if (a0 == 0)
                                {
                                    p0 = lr[a1 - 1];
                                    p1 = li[a1 - 1];
                                }
                                else
                                {
                                    p0 = li[a0 - 1];
                                    p1 = li[a1 - 1];
                                    const double nrm = get_log_sum(p0, p1);
                                    p0 = d_sub(p0, nrm);
                                    p1 = d_sub(p1, nrm);
                                }
                                raw = get_log_sum(d_add(L[a0], p0), d_add(L[a1], p1));
                            }
                            else raw = L[a0];
                            s_term[warp][g][lane] = get_log_sum(d_add(raw, correctMappingLogPrior), incorrect);
                        }
                    }
                }
                // updateSupportingReadStats: integrate mapping status per allele, normalise, first allele at or above the threshold
                double pm[SX_INDEL_MAX_ALLELES + 1];
                double mx = 0;
                uint32_t imax = 0;
#pragma unroll
                for (uint32_t a = 0; a <= SX_INDEL_MAX_ALLELES; ++a)
                {
                    if (a < nfull)
                    {
                        pm[a] = get_log_sum(d_add(L[a], correctMappingLogPrior), incorrect);
                        if (a == 0 || pm[a] > mx)
                        {
                            mx = pm[a];
                            imax = a;
                        }
                    }
                }
                (void)imax;
                double sum = 0;
#pragma unroll
                for (uint32_t a = 0; a <= SX_INDEL_MAX_ALLELES; ++a)
                    if (a < nfull)
                    {
                        pm[a] = sx_exp(d_sub(pm[a], mx));
                        sum = d_add(sum, pm[a]);
                    }
                sum = d_div(1.0, sum);
#pragma unroll
                for (uint32_t a = SX_INDEL_MAX_ALLELES + 1; a-- > 0;)
                    if (a < nfull && !(d_mul(pm[a], sum) < threshold)) choice = a; // lowest index wins
            }
            __syncwarp();
            // ordered accumulation: genotype `lane` adds the reads of this block in read order
            const uint32_t nvalid = min(32u, r1 - rb);
            if (lane < G)
                for (uint32_t k = 0; k < nvalid; ++k) gl = d_add(gl, s_term[warp][lane][k]);
#pragma unroll
            for (uint32_t s = 0; s < 2; ++s)
#pragma unroll
                for (uint32_t a = 0; a < SX_INDEL_MAX_ALLELES + 2; ++a) cnt[s][a] += __popc(__ballot_sync(FULL, valid && fwd == s && choice == a));
            __syncwarp();
        }
        if (lane < SX_INDEL_MAX_GT) res->gt_lhood[lane] = (lane < G) ? gl : 0.0;
        if (lane == 0)
        {
#pragma unroll
            for (int s = 0; s < 2; ++s)
#pragma unroll
                for (int a = 0; a < SX_INDEL_MAX_ALLELES + 2; ++a) res->support[s][a] = static_cast<uint16_t>(cnt[s][a]);
            res->n_gt = G;
            reinterpret_cast<uint32_t*>(res)[sizeof(sx_indel_result) / 4 - 1] = 0; // struct tail padding
        }
    }
}

} // namespace

int sx_k5_run(sx_ctx* ctx, const sx_indel_batch* d, sx_indel_result* out_dev, unsigned* launches)
{
    const int grid = static_cast<int>(std::min<uint32_t>((d->n_loci + K5_WARPS - 1) / K5_WARPS, (uint32_t)ctx->sm_count * 8));
    k5_indel_gl_kernel<<<grid, K5_WARPS * 32, 0, ctx->s_compute>>>(d->read_off, d->lnp_off, d->allele_off, d->ploidy, d->allele_del_len, d->allele_ins_len, d->allele_lnp,
                                                                  d->read_length, d->non_ambig, d->is_fwd, d->n_loci, ctx->d_tables, out_dev, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

extern "C" int sx_indel_gl_dev(sx_ctx* ctx, const sx_indel_batch* d, sx_indel_result* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!d || !out_dev) return sx_fail(ctx, SX_ERR_ARG, "sx_indel_gl_dev: NULL argument");
    if (d->n_loci == 0) return SX_OK;
    const int rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k5_run(ctx, d, out_dev, launches); });
    if (rc) return rc;
    return sx_check_status(ctx, "sx_indel_gl");
}

extern "C" int sx_indel_gl(sx_ctx* ctx, const sx_indel_batch* b, sx_indel_result* out_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    if (!b || !out_host || !b->read_off || !b->lnp_off || !b->allele_off || !b->ploidy) return sx_fail(ctx, SX_ERR_ARG, "sx_indel_gl: NULL argument");
    if (b->n_loci == 0) return SX_OK;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer t(ctx);
    sx_indel_batch d = *b;
    int rc;
    const size_t n_loci = b->n_loci, n_reads = b->read_off[b->n_loci], n_lnp = b->lnp_off[b->n_loci], n_al = b->allele_off[b->n_loci];
    if ((rc = sx_upload(ctx, sx_host_slot(0), b->read_off, n_loci + 1, d.read_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(1), b->lnp_off, n_loci + 1, d.lnp_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(2), b->allele_off, n_loci + 1, d.allele_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(3), b->ploidy, n_loci, d.ploidy, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(4), b->allele_del_len, n_al, d.allele_del_len, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(5), b->allele_ins_len, n_al, d.allele_ins_len, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(6), b->allele_lnp, n_lnp, d.allele_lnp, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(7), b->read_length, n_reads, d.read_length, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(8), b->non_ambig, n_reads, d.non_ambig, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(9), b->is_fwd, n_reads, d.is_fwd, 16))) return rc;
    sx_indel_result* d_out = nullptr;
    if ((rc = sx_take(ctx, sx_host_slot(10), n_loci, d_out, 0))) return rc;
    unsigned launches = 0;
    if ((rc = sx_k5_run(ctx, &d, d_out, &launches))) return rc;
    if ((rc = sx_download(ctx, out_host, d_out, n_loci))) return rc;
    if ((rc = t.finish(launches))) return rc;
    return sx_check_status(ctx, "sx_indel_gl");
}
