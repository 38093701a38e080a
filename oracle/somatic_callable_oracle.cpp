// oracle/somatic_callable_oracle.cpp -- TEST INFRASTRUCTURE.  The somatic SNV model in callable mode (position_somatic_snv_call with
// isComputeNonSomatic = true, applications/strelka/position_somatic_snv_strand_grid.cpp:228-363), restated on top of liboracle.so's K2b.
//
// With isComputeNonSomatic set, every test the flag takes part in reads `is_forced_output || isComputeNonSomatic` (:251, :309, and the
// wrapper's :183), so a callable-mode record is the forced record of the same position.  Its one new field, nonsomatic_qphred, comes from the
// tier1 view alone (:362): the forced tier1-only record carries those likelihoods, and the loop below restates :186-215 on them, with
// opt_normalize_ln_distro (blt_util/prob_util.hh:250-318) as the reference writes it.
#include "strelka_oracle.h"

#include "sx_libm_mirror_d.h"

#include <cmath>
#include <limits>
#include <vector>

namespace
{
const unsigned GRID = 21; // DIGT_GRID::PRESTRAND_SIZE

// isValidNonsomaticIndex, DIGT_GRID::get_fraction_from_index
bool is_valid_nonsomatic_index(const unsigned f)
{
    const float min_frac(0.1), min_frac_comp(1. - min_frac), eps(0.0001);
    const float min_frac_eps(min_frac - eps), min_frac_comp_eps(min_frac_comp + eps);
    if (f == 0 || f == 1) return true;
    const float ratio_increment(0.5f / static_cast<float>(9 + 1));
    float frac;
    if (f == 2) frac = 0.5f;
    else if (f < 3 + 9) frac = ratio_increment * (f - 3 + 1);
    else frac = ratio_increment * (f - 3 + 2);
    if (frac < min_frac_eps) return false;
    if (frac > min_frac_comp_eps) return false;
    return true;
}

// gvcf_nonsomatic_gvcf_prior
float nonsomatic_prior(const unsigned fn, const unsigned ft)
{
    const float lzero(-std::numeric_limits<float>::infinity());
    if (!is_valid_nonsomatic_index(ft)) return lzero;
    if (fn == ft) return std::log(1.f);
    if (fn == 0 || fn == 1) return std::log(0.5f);
    return lzero;
}

int nonsomatic_qphred(const float* normal_lhood, const float* tumor_lhood)
{
    std::vector<double> pprob(GRID * GRID);
    std::vector<bool> is_nonsom(GRID * GRID, false);
    for (unsigned fn = 0; fn < GRID; ++fn)
        for (unsigned ft = 0; ft < GRID; ++ft) pprob[fn + GRID * ft] = normal_lhood[fn] + tumor_lhood[ft] + nonsomatic_prior(fn, ft);
    for (unsigned f = 0; f < GRID; ++f) is_nonsom[f + GRID * f] = true;
    // opt_normalize_ln_distro
    bool is_max(false), is_opt_max(false);
    double max(0), opt_max(0);
    for (unsigned i = 0; i < pprob.size(); ++i)
    {
        const double p(pprob[i]);
        if ((!is_max) || (p > max))
        {
            max = p;
            is_max = true;
        }
        if (((!is_opt_max) || (p > max)) && is_nonsom[i])
        {
            opt_max = p;
            is_opt_max = true;
        }
    }
    double sum(0.);
    for (unsigned i = 0; i < pprob.size(); ++i)
    {
        const double mdiff(max - pprob[i]);
        if (mdiff > 20.)
        {
            if (!is_nonsom[i] || (opt_max - pprob[i]) > 5.)
            {
                pprob[i] = 0;
                continue;
            }
        }
        pprob[i] = sx_exp(-mdiff);
        sum += pprob[i];
    }
    sum = 1. / sum;
    for (double& p : pprob) p *= sum;
    double diag(0);
    for (unsigned f = 0; f < GRID; ++f) diag += pprob[f + GRID * f];
    // error_prob_to_qphred
    const double l(sx_log10(1. - diag));
    const double m((-307. < l) ? l : -307.);
    return static_cast<int>(std::floor(-10. * m + 0.5));
}
} // namespace

extern "C" int ox_site_gl_somatic_callable(const sx_params* p, const sx_pileup_batch* normal, const sx_pileup_batch* tumor, const uint8_t* /*is_forced_output*/,
                                           sx_ssnv_result* out)
{
    const uint32_t n(normal->n_sites);
    const std::vector<uint8_t> forced(n, 1);
    int rc(ox_site_gl_somatic(p, normal, tumor, forced.data(), out));
    if (rc) return rc;
    sx_pileup_batch n1(*normal), t1(*tumor);
    n1.t2_off = t1.t2_off = nullptr;
    n1.t2_calls = t1.t2_calls = nullptr;
    std::vector<sx_ssnv_result> tier1(n);
    if ((rc = ox_site_gl_somatic(p, &n1, &t1, forced.data(), tier1.data()))) return rc;
    for (uint32_t s = 0; s < n; ++s)
        out[s].nonsomatic_qphred = out[s].is_computed ? nonsomatic_qphred(tier1[s].normal_lhood, tier1[s].tumor_lhood) : 0;
    return 0;
}
