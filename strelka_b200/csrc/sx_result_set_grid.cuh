// sx_result_set_grid.cuh -- calculate_result_set_grid (applications/strelka/qscore_calculator.cpp:47-209), shared by K2b (somatic SNVs)
// and K5b (somatic indels).
//
// The double loop over (tumor freq, normal freq) is unrolled on the host into, per (normal gt, somatic state) combo, the ordered list of
// the terms it visits (sx_context.cu for K2b, k5b_somatic_indel.cu for K5b).  `Terms` gives them:
//   n_terms(combo)        the list's length (<= 44)
//   lprior(combo, i)      lprior_freq of term i, as the reference's double
//   nf(combo, i), tf(combo, i)   its normal and tumor grid indices
//   geno_prior(combo)     germlineGenotypeLogPrior[ngt] + (tgt == 0 ? lnmatch : lnmismatch), the reference's float sum
// so that each caller decides which of those values are per-call constants and which are per-locus ones.
//
// All lanes cooperate and all lanes return the same result; `scratch` holds 44 doubles of the warp's own.
#pragma once

#include "sx_device_util.cuh"

template <class Terms, class RS>
__device__ __forceinline__ void result_set_grid(const Terms& T, const float* nl, const float* tl, double* scratch, uint32_t lane, RS& rs)
{
    double log_post_prob[6];
    double max_log_prob = -INFINITY;
    rs.max_gt = 0;
#pragma unroll 1
    for (uint32_t combo = 0; combo < 6; ++combo)
    {
        const uint32_t nt = T.n_terms(combo);
        double max_log_sum = -INFINITY;
        // terms in the reference's loop order; two rounds of 32 lanes (nt <= 44)
        double l0 = -INFINITY, l1 = -INFINITY;
        if (lane < nt) l0 = d_add(d_add(T.lprior(combo, lane), static_cast<double>(nl[T.nf(combo, lane)])), static_cast<double>(tl[T.tf(combo, lane)]));
        if (lane + 32 < nt)
            l1 = d_add(d_add(T.lprior(combo, lane + 32), static_cast<double>(nl[T.nf(combo, lane + 32)])), static_cast<double>(tl[T.tf(combo, lane + 32)]));
        double m = fmax(l0, l1);
#pragma unroll
        for (int d = 16; d; d >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, d));
        max_log_sum = m;
        __syncwarp();
        if (lane < nt) scratch[lane] = sx_exp(d_sub(l0, max_log_sum));
        if (lane + 32 < nt) scratch[lane + 32] = sx_exp(d_sub(l1, max_log_sum));
        __syncwarp();
        double sum = 0.0;
        for (uint32_t i = 0; i < nt; ++i) sum = d_add(sum, scratch[i]);
        const double log_genotype_prior = static_cast<double>(T.geno_prior(combo));
        log_post_prob[combo] = d_add(d_add(log_genotype_prior, max_log_sum), sx_log(sum));
        if (log_post_prob[combo] > max_log_prob)
        {
            max_log_prob = log_post_prob[combo];
            rs.max_gt = combo; // DDIGT::get_state(ngt, tgt) = ngt*2 + tgt
        }
    }
    double sum_prob = 0.0;
#pragma unroll
    for (int c = 0; c < 6; ++c) sum_prob = d_add(sum_prob, sx_exp(d_sub(log_post_prob[c], max_log_prob)));
    const double log_sum_prob = sx_log(sum_prob);
    double min_not_somfrom_sum = INFINITY;
    double nonsom_prob = 0.0;
    rs.ntype = 0;
    rs.from_ntype_qphred = 0;
#pragma unroll
    for (uint32_t ngt = 0; ngt < 3; ++ngt)
    {
        double som_prob_given_ngt = 0;
#pragma unroll
        for (uint32_t tgt = 0; tgt < 2; ++tgt)
        {
            const double pp = sx_exp(d_sub(d_sub(log_post_prob[ngt * 2 + tgt], max_log_prob), log_sum_prob));
            if (tgt == 0) nonsom_prob = d_add(nonsom_prob, pp);
            else som_prob_given_ngt = d_add(som_prob_given_ngt, pp);
        }
        const double err_som_and_ngt = d_sub(1.0, som_prob_given_ngt);
        if (err_som_and_ngt < min_not_somfrom_sum)
        {
            min_not_somfrom_sum = err_som_and_ngt;
            rs.from_ntype_qphred = error_prob_to_qphred_d(err_som_and_ngt);
            rs.ntype = ngt;
        }
    }
    rs.qphred = error_prob_to_qphred_d(nonsom_prob);
}
