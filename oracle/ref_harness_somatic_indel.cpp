// ref_harness_somatic_indel.cpp -- TEST INFRASTRUCTURE ONLY (linked into oracle/_ref/libstrelka_ref_sindel.so by
// oracle/build_ref_somatic_indel.sh, next to oracle/_ref/libstrelka_ref.so).
//
// Drives the UNMODIFIED reference somatic_indel_caller_grid::get_somatic_indel (applications/strelka/somatic_indel_grid.cpp:181) on a
// flattened sx_sindel_batch: per locus an IndelData with two samples (normal 0, tumor 1) is rebuilt, its read_path_lnp maps filled from
// the batch with the alternates as real IndelKeys, isForcedOutput set and the tumor's indelToRefErrorProb injected through
// IndelSampleData's private _errorRates (explicit-instantiation idiom), then the function is called through dopt.sicaller_grid() as
// strelka_pos_processor.cpp:343-348 does.  get_somatic_indel keeps its per-tier values to itself, so each tier's float likelihoods
// are taken from the exported get_indel_digt_lhood / get_high_low_het_ratio_lhood (in get_indel_het_grid_lhood's order,
// somatic_indel_grid.cpp:80-89) and its result set from the exported calculate_result_set_grid, before any multi-indel rejection.
#include "../include/strelka_b200.h"

#include "applications/strelka/qscore_calculator.hh"
#include "applications/strelka/somatic_indel_grid.hh"
#include "applications/strelka/strelka_shared.hh"
#include "blt_util/blt_exception.hh"
#include "blt_util/math_util.hh"
#include "starling_common/IndelData.hh"
#include "starling_common/starling_indel_call_pprob_digt.hh"

#include <chrono>
#include <cmath>
#include <cstring>
#include <exception>
#include <string>

namespace
{
template <typename Tag, typename Tag::type M> struct MemberPtrOf3
{
    friend typename Tag::type memberPtr(Tag) { return M; }
};
struct SindelErrorRatesTag
{
    typedef IndelErrorRates IndelSampleData::*type;
    friend type memberPtr(SindelErrorRatesTag);
};
template struct MemberPtrOf3<SindelErrorRatesTag, &IndelSampleData::_errorRates>;

// equal table entries would be equal IndelKeys; the batch's tables hold distinct (pos, del_len, ins_len, ins_id), and the insert
// sequence spells ins_id in base 4 so that equal lengths with different ids stay distinct keys
IndelKey key_of(const sx_indel_key& k)
{
    std::string ins(k.ins_len, 'A');
    uint32_t id = k.ins_id;
    for (size_t i = 0; i < ins.size() && id; ++i, id >>= 2) ins[ins.size() - 1 - i] = "ACGT"[id & 3];
    return IndelKey(k.pos, (k.type == SX_INDEL_TYPE_MISMATCH) ? INDEL::MISMATCH : INDEL::INDEL, k.del_len, ins.c_str());
}
} // namespace

// out[l]: the final call of get_somatic_indel (is_output and the fields after it; status) and, for both tiers whatever the control flow,
// the 2x21 float likelihoods and calculate_result_set_grid's qphred / from_ntype_qphred / ntype / max_gt on them (evaluated = 1,
// multi_indel and is_overlap 0: they are internal to the reference function)
namespace
{
int run(const sx_sindel_opts* o, const sx_sindel_batch* b, const double* err_prob, uint32_t n_err, sx_sindel_result* out, const bool per_tier, double* secs,
        char* err, int errlen)
{
    try
    {
        strelka_options opt;
        opt.alignFileOpt.alignmentFilenames = {"normal.bam", "tumor.bam"}; // two samples for the options' per-sample models
        opt.alignFileOpt.isAlignmentTumor = {false, true};
        opt.somatic_indel_rate = o->somatic_indel_rate;
        opt.bindel_diploid_theta = o->bindel_diploid_theta;
        opt.indel_contam_tolerance = o->indel_contam_tolerance;
        opt.shared_indel_error_factor = o->shared_indel_error_factor;
        opt.randomBaseMatchProb = o->randomBaseMatchProb;
        opt.tier2.isRandomBaseMatchProb = true;
        opt.tier2.randomBaseMatchProb = o->tier2RandomBaseMatchProb;
        opt.useTier2Evidence = (o->useTier2Evidence != 0);
        opt.default_min_read_bp_flank = o->min_read_bp_flank[1];
        opt.normal_sample_min_read_bp_flank = o->min_read_bp_flank[0];
        const strelka_deriv_options dopt(opt);
        starling_sample_options normal_opt(opt), tumor_opt(opt);
        normal_opt.min_read_bp_flank = opt.normal_sample_min_read_bp_flank; // strelka_pos_processor.cpp:58
        blt_float_t germ[3];
        calculateGermlineGenotypeLogPrior(opt.bindel_diploid_theta, germ);
        const blt_float_t ln_som_match(log1p_switch(-opt.somatic_indel_rate)), ln_som_mismatch(std::log(opt.somatic_indel_rate));
        const auto errorRatesPtr(memberPtr(SindelErrorRatesTag()));
        for (uint32_t l = 0; l < b->n_loci; ++l)
        {
            sx_sindel_result& r(out[l]);
            std::memset(&r, 0, sizeof(r));
            if (b->err_idx[l] >= n_err) throw blt_exception("ref_somatic_indel: error-rate index past the table");
            const IndelKey indelKey(key_of(b->key[l]));
            IndelData indelData(2, indelKey);
            indelData.isForcedOutput = (b->is_forced_output[l] != 0);
            const sx_indel_key* alts(b->alts + b->alt_off[l]);
            for (unsigned s = 0; s < 2; ++s)
            {
                IndelSampleData& isd(indelData.getSampleData(s));
                for (uint32_t i = b->read_off[2 * l + s]; i < b->read_off[2 * l + s + 1]; ++i)
                {
                    const sx_sindel_read& rd(b->reads[i]);
                    ReadPathScores rps(rd.ref, rd.indel, rd.non_ambig, rd.read_length, rd.is_tier1 != 0, true, 0, 0);
                    for (unsigned k = 0; k < rd.n_alt; ++k) rps.alt_indel.push_back(std::make_pair(key_of(alts[rd.alt[k]]), rd.alt_lnp[k]));
                    isd.read_path_lnp[i - b->read_off[2 * l + s]] = rps;
                }
            }
            (indelData.getSampleData(1).*errorRatesPtr).indelToRefErrorProb.updateValue(err_prob[b->err_idx[l]]);

            somatic_indel_call sindel;
            sindel.sindel_tier = false;
            sindel.sindel_from_ntype_tier = false;
            sindel.rs.ntype = 0;
            sindel.rs.max_gt = 0;
            const auto t0(std::chrono::steady_clock::now());
            dopt.sicaller_grid().get_somatic_indel(opt, dopt, normal_opt, tumor_opt, indelKey, indelData, 0, 1, true, sindel);
            if (secs) *secs += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
            r.is_output = sindel.is_output() ? 1 : 0;
            if (r.is_output)
            {
                r.sindel_tier = sindel.sindel_tier;
                r.sindel_from_ntype_tier = sindel.sindel_from_ntype_tier;
                r.is_overlap = sindel.rs.is_overlap;
                r.ntype = sindel.rs.ntype;
                r.max_gt = sindel.rs.max_gt;
                r.qphred = sindel.rs.qphred;
                r.from_ntype_qphred = sindel.rs.from_ntype_qphred;
            }
            if (!per_tier) continue;

            const double sharedIndelErrorRate(std::pow(err_prob[b->err_idx[l]], opt.shared_indel_error_factor));
            const double lse(std::log(sharedIndelErrorRate)), lcse(log1p_switch(-sharedIndelErrorRate));
            for (unsigned t = 0; t < 2; ++t)
            {
                const bool is_tier2(t == 1);
                sx_sindel_tier& T(r.tier[t]);
                for (unsigned s = 0; s < 2; ++s)
                {
                    const starling_sample_options& sopt(s == 0 ? normal_opt : tumor_opt);
                    const IndelSampleData& isd(indelData.getSampleData(s));
                    double lhood[21];
                    get_indel_digt_lhood(opt, dopt, sopt, indelKey, isd, is_tier2, true, lhood);
                    for (unsigned i = 0; i < 9; ++i)
                    {
                        const double het_ratio((i + 1) * DIGT_GRID::RATIO_INCREMENT);
                        get_high_low_het_ratio_lhood(opt, dopt, sopt, indelKey, isd, het_ratio, is_tier2, true, lhood[3 + 18 - (i + 1)], lhood[3 + i]);
                    }
                    for (unsigned j = 0; j < 21; ++j) (s == 0 ? T.normal_lhood : T.tumor_lhood)[j] = (blt_float_t)lhood[j];
                }
                indel_result_set rs;
                calculate_result_set_grid((float)opt.indel_contam_tolerance, (float)lse, (float)lcse, T.normal_lhood, T.tumor_lhood, germ, ln_som_match,
                                          ln_som_mismatch, rs);
                T.qphred = rs.qphred;
                T.from_ntype_qphred = rs.from_ntype_qphred;
                T.ntype = rs.ntype;
                T.max_gt = rs.max_gt;
                T.evaluated = 1;
            }
        }
        return 0;
    }
    catch (const std::exception& e)
    {
        if (err && errlen > 0)
        {
            std::strncpy(err, e.what(), errlen - 1);
            err[errlen - 1] = 0;
        }
        return 1;
    }
}
} // namespace

extern "C" int ref_somatic_indel(const sx_sindel_opts* o, const sx_sindel_batch* b, const double* err_prob, uint32_t n_err, sx_sindel_result* out, char* err,
                                 int errlen)
{
    return run(o, b, err_prob, n_err, out, true, nullptr, err, errlen);
}

// the final call only; *secs accumulates the time inside get_somatic_indel itself (the IndelData objects around it are this harness's)
extern "C" int ref_somatic_indel_timed(const sx_sindel_opts* o, const sx_sindel_batch* b, const double* err_prob, uint32_t n_err, sx_sindel_result* out, double* secs,
                                       char* err, int errlen)
{
    *secs = 0;
    return run(o, b, err_prob, n_err, out, false, secs, err, errlen);
}
