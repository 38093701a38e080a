// k2b_nonsomatic.cuh -- K2b's callable mode: the non-somatic quality (NQSS) of calculate_result_set_grid's isComputeNonSomatic branch
// (applications/strelka/position_somatic_snv_strand_grid.cpp:186-215).  Compiled __device__ by nvcc (k2b_somatic.cu spreads the terms over
// a warp) and as plain C++ by g++ (tests/cpp/k2b_nonsomatic_host.cpp), with the mirrored libm of sx_libm_mirror_d.h and unfused arithmetic
// (-fmad=false / -ffp-contract=off): the host and the device give the same bits.
//
// The reference's steps, on the tier1 likelihoods nl[0..20] (normal) and tl[0..20] (tumor):
//   pprob[fn + 21 ft] = nl[fn] + tl[ft] + gvcf_nonsomatic_gvcf_prior(fn, ft), two float adds, stored as a double   (441 prestrand states)
//   opt_normalize_ln_distro (blt_util/prob_util.hh:250-318) with DDIGT_GRID::is_nonsom as the predicate: true exactly on the diagonal
//     states fn == ft, index 22 f.
//     max     the first strict maximum: pprob[0] when that is NaN, else the largest non-NaN state (which of +0 / -0 it is changes no result)
//     opt_max the first predicate-true state's value, pprob[0]: the test `*p > max` follows the update of max for the same element
//     a state with max - p > 20 becomes +0 when its predicate is false or opt_max - p > 5; every other state becomes exp(-(max - p)),
//     summed in double in index order from +0; then every state is scaled by 1./sum.
//   nonsomatic_qphred = error_prob_to_qphred(1. - the sum of the 21 scaled diagonal states, f = 0..20)
// Skipped states are exact +0 and the sum starts at +0, so a sum over the non-zero terms alone, in index order, has the same bits.
#pragma once

#include <math.h>
#include <stdint.h>

#include "sx_libm_mirror_d.h"

#if defined(__CUDACC__)
#define K2BN_HD __device__ __forceinline__
#else
#define K2BN_HD static inline
#endif

constexpr uint32_t K2BN_GRID = 21;                      // DIGT_GRID::PRESTRAND_SIZE
constexpr uint32_t K2BN_STATES = K2BN_GRID * K2BN_GRID; // DDIGT_GRID::PRESTRAND_SIZE
constexpr uint32_t K2BN_DIAG_STRIDE = K2BN_GRID + 1;    // DDIGT_GRID::get_state(f, f) = 22 f

// isValidNonsomaticIndex (:90-113): the grid fraction (DIGT_GRID::get_fraction_from_index, strelka_digt_states.cpp:34-41) within the
// epsilon-padded [0.1, 0.9], all in float
K2BN_HD bool k2bn_valid_index(const uint32_t f)
{
    if (f == 0 || f == 1) return true; // SOMATIC_DIGT::REF, HOM
    const float ratio_increment = 0.5f / 10.f; // DIGT_GRID::RATIO_INCREMENT
    const float frac = (f == 2) ? 0.5f : ratio_increment * static_cast<float>(f < 12 ? (int)f - 2 : (int)f - 1);
    const float min_frac = 0.1f, min_frac_comp = static_cast<float>(1. - static_cast<double>(min_frac)), eps = 0.0001f;
    const float min_frac_eps = min_frac - eps, min_frac_comp_eps = min_frac_comp + eps;
    if (frac < min_frac_eps) return false;
    if (frac > min_frac_comp_eps) return false;
    return true;
}

// gvcf_nonsomatic_gvcf_prior (:129-155), float
K2BN_HD float k2bn_prior(const uint32_t fn, const uint32_t ft)
{
    if (!k2bn_valid_index(ft)) return -INFINITY;
    if (fn == ft) return 0.f;                        // std::log(1.f)
    if (fn == 0 || fn == 1) return -0.693147182f;    // std::log(0.5f), correctly rounded
    return -INFINITY;
}

// pprob[i], i = fn + 21 ft
K2BN_HD double k2bn_pprob(const float* nl, const float* tl, const uint32_t i)
{
    const uint32_t fn = i % K2BN_GRID, ft = i / K2BN_GRID;
    const float a = nl[fn] + tl[ft];
    return static_cast<double>(a + k2bn_prior(fn, ft));
}

// state i after opt_normalize_ln_distro's exp step, before the scaling
K2BN_HD double k2bn_term(const double p, const double max, const double opt_max, const uint32_t i)
{
    const double mdiff = max - p;
    if (mdiff > 20.0)
    {
        if (i % K2BN_DIAG_STRIDE != 0) return 0.0;
        if (opt_max - p > 5.0) return 0.0;
    }
    return sx_exp(-mdiff);
}

// error_prob_to_qphred<double> (blt_util/qscore.hh:40-66) of 1. - diag_sum
K2BN_HD int k2bn_qphred(const double diag_sum)
{
    const double l = sx_log10(1.0 - diag_sum);
    const double m = (-307.0 < l) ? l : -307.0; // std::max(minlog10, l)
    return static_cast<int>(floor(-10.0 * m + 0.5));
}

// the whole computation, one state after the other, as the reference loops (the host's form; the kernel spreads the same steps over a warp)
K2BN_HD int k2bn_nonsomatic_qphred(const float* nl, const float* tl)
{
    double max = k2bn_pprob(nl, tl, 0);
    for (uint32_t i = 1; i < K2BN_STATES; ++i)
    {
        const double p = k2bn_pprob(nl, tl, i);
        if (p > max) max = p;
    }
    const double opt_max = k2bn_pprob(nl, tl, 0);
    double sum = 0.0;
    for (uint32_t i = 0; i < K2BN_STATES; ++i)
    {
        const double t = k2bn_term(k2bn_pprob(nl, tl, i), max, opt_max, i);
        if (t != 0.0) sum += t;
    }
    const double inv = 1. / sum;
    double diag = 0.0;
    for (uint32_t f = 0; f < K2BN_GRID; ++f)
        diag += k2bn_term(k2bn_pprob(nl, tl, f * K2BN_DIAG_STRIDE), max, opt_max, f * K2BN_DIAG_STRIDE) * inv;
    return k2bn_qphred(diag);
}
