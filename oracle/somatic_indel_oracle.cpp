// somatic_indel_oracle.cpp -- TEST INFRASTRUCTURE.  A scalar restatement of somatic_indel_caller_grid::get_somatic_indel
// (applications/strelka/somatic_indel_grid.cpp:181-361) on an sx_sindel_batch, written as the reference reads, one locus at a
// time.  It evaluates exp / log / log1p / log10 with the libm mirrors the K5b kernel uses (strelka_b200/csrc/sx_libm_mirror_d.h),
// and the option- and error-rate-derived values with the host libm, as the library does; the tests pin it to the reference's own
// function (oracle/ref_harness_somatic_indel.cpp) and the kernel to it.
#include "../include/strelka_b200.h"
#include "../strelka_b200/csrc/sx_libm_mirror_d.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <utility>
#include <vector>

namespace
{
typedef float blt_float_t;

double log1p_switch_host(const double x) // blt_util/math_util.hh:33-47 with the host libm
{
    if (std::abs(x) < 0.01) return ::log1p(x);
    return std::log(1 + x);
}
double log1p_switch(const double x) { return (std::fabs(x) < 0.01) ? sx_log1p(x) : sx_log(1.0 + x); }
double get_log_sum(double x1, double x2)
{
    if (x1 < x2) std::swap(x1, x2);
    return x1 + log1p_switch(sx_exp(x2 - x1));
}
int error_prob_to_qphred(const double prob) // blt_util/qscore.hh:40-66
{
    return static_cast<int>(std::floor(-10. * std::max(-307., sx_log10(prob)) + 0.5));
}
bool is_indel_conflict(const sx_indel_key& a, const sx_indel_key& b) // indel_util.cpp:29-45
{
    const bool mm = a.type == SX_INDEL_TYPE_MISMATCH || b.type == SX_INDEL_TYPE_MISMATCH;
    const int64_t e1 = (int64_t)a.pos + a.del_len + (mm ? 0 : 1), e2 = (int64_t)b.pos + b.del_len + (mm ? 0 : 1);
    return (e2 > a.pos) && (b.pos < e1);
}

const blt_float_t RATIO_INCREMENT = 0.5f / static_cast<blt_float_t>(9 + 1);

struct deriv
{
    double rbm[2], cmlp;
    blt_float_t germ[3], ln_som_match, ln_som_mismatch;
};

void het_observed(const unsigned read_length, const unsigned min_overlap, const sx_indel_key& k, const double r, double& lr, double& li)
{
    const unsigned base_expect((read_length + 1) < (2 * min_overlap) ? 0 : (read_length + 1) - (2 * min_overlap));
    const double ref_path_expect(base_expect + std::min((unsigned)k.del_len, base_expect));
    const double indel_path_expect(base_expect + std::min((unsigned)k.ins_len, base_expect));
    const double ref_path_term((1 - r) * ref_path_expect);
    const double indel_path_term(r * indel_path_expect);
    const double total_path_term(ref_path_term + indel_path_term);
    if (total_path_term > 0)
    {
        const double indel_prob(indel_path_term / total_path_term);
        lr = sx_log(1. - indel_prob);
        li = sx_log(indel_prob);
    }
}

double integrate(const deriv& D, const unsigned nonamb, const double lnp, const bool t2)
{
    return get_log_sum(lnp + D.cmlp, D.rbm[t2 ? 1 : 0] * nonamb);
}

// get_indel_digt_lhood + get_indel_het_grid_lhood of one sample
void sample_lhood(const deriv& D, const sx_sindel_read* r0, const sx_sindel_read* r1, const sx_indel_key& key, const unsigned flank, const bool t2, double* lhood)
{
    for (int i = 0; i < 21; ++i) lhood[i] = 0.;
    static const double loghalf(-std::log(2.));
    for (const sx_sindel_read* p = r0; p < r1; ++p)
    {
        if (!t2 && !p->is_tier1) continue;
        double alt_path_lnp(p->ref);
        for (unsigned k = 0; k < p->n_alt; ++k)
            if (p->alt_lnp[k] > alt_path_lnp) alt_path_lnp = p->alt_lnp[k];
        const double noindel_lnp(alt_path_lnp), hom_lnp(p->indel);
        double lr(loghalf), li(loghalf);
        het_observed(p->read_length, flank, key, 0.5, lr, li);
        const double het_lnp(get_log_sum(noindel_lnp + lr, hom_lnp + li));
        lhood[0] += integrate(D, p->non_ambig, noindel_lnp, t2);
        lhood[1] += integrate(D, p->non_ambig, hom_lnp, t2);
        lhood[2] += integrate(D, p->non_ambig, het_lnp, t2);
    }
    for (unsigned i = 0; i < 9; ++i)
    {
        const double het_ratio((i + 1) * RATIO_INCREMENT);
        const double chet_ratio(1. - het_ratio);
        const double log_het_ratio(std::log(het_ratio)), log_chet_ratio(std::log(chet_ratio));
        double high = 0, low = 0;
        for (const sx_sindel_read* p = r0; p < r1; ++p)
        {
            if (!t2 && !p->is_tier1) continue;
            double alt_path_lnp(p->ref);
            for (unsigned k = 0; k < p->n_alt; ++k)
                if (p->alt_lnp[k] > alt_path_lnp) alt_path_lnp = p->alt_lnp[k];
            const double noindel_lnp(alt_path_lnp), hom_lnp(p->indel);
            {
                double lr(log_chet_ratio), li(log_het_ratio);
                het_observed(p->read_length, flank, key, het_ratio, lr, li);
                low += integrate(D, p->non_ambig, get_log_sum(noindel_lnp + lr, hom_lnp + li), t2);
            }
            {
                double lr(log_het_ratio), li(log_chet_ratio);
                het_observed(p->read_length, flank, key, chet_ratio, lr, li);
                high += integrate(D, p->non_ambig, get_log_sum(noindel_lnp + lr, hom_lnp + li), t2);
            }
        }
        lhood[3 + 18 - (i + 1)] = high;
        lhood[3 + i] = low;
    }
}

// get_sum_path_pprob of one sample into (ref, indel, [(alt index, pprob)])
void sum_path_pprob(const deriv& D, const sx_sindel_read* r0, const sx_sindel_read* r1, const bool t2, float& tref, float& tindel,
                    std::vector<std::pair<unsigned, float>>& talt)
{
    int slot_of[256];
    for (int& s : slot_of) s = -1;
    for (const sx_sindel_read* p = r0; p < r1; ++p)
    {
        if (!t2 && !p->is_tier1) continue;
        const unsigned n_alleles = 2 + p->n_alt;
        const double allele_lnprior(std::log(1. / static_cast<double>(n_alleles)));
        float inc = D.rbm[t2 ? 1 : 0] * p->non_ambig;
        float ref = p->ref + D.cmlp + allele_lnprior;
        float indel = p->indel + D.cmlp + allele_lnprior;
        float alt[2];
        for (unsigned k = 0; k < p->n_alt; ++k) alt[k] = p->alt_lnp[k] + D.cmlp + allele_lnprior;
        double scale(std::max(inc, std::max(ref, indel)));
        for (unsigned k = 0; k < p->n_alt; ++k)
            if (scale < alt[k]) scale = alt[k];
        inc = sx_exp(inc - scale);
        ref = sx_exp(ref - scale);
        indel = sx_exp(indel - scale);
        for (unsigned k = 0; k < p->n_alt; ++k) alt[k] = sx_exp(alt[k] - scale);
        double sum(inc + ref + indel); // a float sum, widened
        for (unsigned k = 0; k < p->n_alt; ++k) sum += alt[k];
        ref /= sum;
        indel /= sum;
        for (unsigned k = 0; k < p->n_alt; ++k) alt[k] /= sum;
        tindel += indel;
        tref += ref;
        for (unsigned k = 0; k < p->n_alt; ++k)
        {
            const unsigned a = p->alt[k];
            if (slot_of[a] < 0)
            {
                slot_of[a] = (int)talt.size();
                talt.emplace_back(a, alt[k]);
            }
            else talt[slot_of[a]].second += alt[k];
        }
    }
}

bool is_multi_indel_allele(const deriv& D, const sx_indel_key* alts, const sx_sindel_read* rb[3], const bool t2, bool& is_overlap)
{
    float tref = 0, tindel = 0;
    std::vector<std::pair<unsigned, float>> talt;
    sum_path_pprob(D, rb[0], rb[1], t2, tref, tindel, talt);
    sum_path_pprob(D, rb[1], rb[2], t2, tref, tindel, talt);
    std::vector<std::pair<double, int>> scores;
    scores.push_back(std::make_pair(-tindel, -2));
    scores.push_back(std::make_pair(-tref, -1));
    for (int i = 0; i < (int)talt.size(); ++i) scores.push_back(std::make_pair(-talt[i].second, i));
    std::sort(scores.begin(), scores.end());
    while (scores[0].second >= 0 && scores[1].second >= 0)
    {
        if (is_indel_conflict(alts[talt[scores[0].second].first], alts[talt[scores[1].second].first])) break;
        scores.erase(scores.begin() + 1);
    }
    if ((scores[0].second != -2) && (scores[1].second != -2)) return true;
    if (scores.size() >= 3)
    {
        const double top_prob(scores[0].first + scores[1].first);
        const double top_frac(top_prob / (top_prob + scores[2].first));
        if (top_frac < .9) return true;
    }
    is_overlap = ((scores[0].second != -1) && (scores[1].second != -1));
    return false;
}

void result_set_grid(const blt_float_t contam_tolerance, const blt_float_t logSharedErrorRate, const blt_float_t logSharedErrorRateComplement,
                     const blt_float_t* normal_lhood, const blt_float_t* tumor_lhood, const deriv& D, sx_sindel_tier& rs)
{
    static const blt_float_t ln_one_half(std::log(1. / 2.));
    static const blt_float_t log_error_mod = -std::log(static_cast<double>(21 - 1));
    auto fraction_of = [](int index) -> blt_float_t {
        if (index == 0) return 0.f;
        if (index == 1) return 1.f;
        if (index == 2) return 0.5f;
        if (index < 3 + 9) return RATIO_INCREMENT * (index - 3 + 1);
        return RATIO_INCREMENT * (index - 3 + 2);
    };
    double log_post_prob[3][2];
    double max_log_prob = -std::numeric_limits<float>::infinity();
    rs.max_gt = 0;
    for (unsigned ngt = 0; ngt < 3; ++ngt)
        for (unsigned tgt = 0; tgt < 2; ++tgt)
        {
            double max_log_sum = -std::numeric_limits<float>::infinity();
            double log_sum[441];
            int index = 0;
            for (unsigned tf = 0; tf < 21; ++tf)
            {
                const blt_float_t tumor_freq = fraction_of(tf);
                const bool consider_norm_contam = contam_tolerance * tumor_freq >= RATIO_INCREMENT;
                for (unsigned nf = 0; nf < 21; ++nf)
                {
                    double lprior_freq;
                    if (tgt == 0)
                    {
                        if (nf != tf) continue;
                        lprior_freq = (nf == ngt) ? logSharedErrorRateComplement : logSharedErrorRate + log_error_mod;
                    }
                    else
                    {
                        if (nf == tf) continue;
                        if (ngt != 0)
                        {
                            if (nf != ngt) continue;
                            lprior_freq = log_error_mod;
                        }
                        else if (!consider_norm_contam)
                        {
                            if (nf != 0) continue;
                            lprior_freq = log_error_mod;
                        }
                        else
                        {
                            if ((nf != ngt) && (nf != 3)) continue;
                            lprior_freq = log_error_mod + ln_one_half;
                        }
                    }
                    const double lsum = lprior_freq + normal_lhood[nf] + tumor_lhood[tf];
                    log_sum[index++] = lsum;
                    if (lsum > max_log_sum) max_log_sum = lsum;
                }
            }
            double sum = 0.0;
            for (int i = 0; i < index; ++i) sum += sx_exp(log_sum[i] - max_log_sum);
            const double log_genotype_prior = D.germ[ngt] + ((tgt == 0) ? D.ln_som_match : D.ln_som_mismatch);
            log_post_prob[ngt][tgt] = log_genotype_prior + max_log_sum + sx_log(sum);
            if (log_post_prob[ngt][tgt] > max_log_prob)
            {
                max_log_prob = log_post_prob[ngt][tgt];
                rs.max_gt = ngt * 2 + tgt;
            }
        }
    double sum_prob = 0.0;
    for (unsigned ngt = 0; ngt < 3; ++ngt)
        for (unsigned tgt = 0; tgt < 2; ++tgt) sum_prob += sx_exp(log_post_prob[ngt][tgt] - max_log_prob);
    const double log_sum_prob = sx_log(sum_prob);
    double min_not_somfrom_sum(INFINITY), nonsom_prob = 0.0;
    for (unsigned ngt = 0; ngt < 3; ++ngt)
    {
        double som_prob_given_ngt(0);
        for (unsigned tgt = 0; tgt < 2; ++tgt)
        {
            const double pp = sx_exp(log_post_prob[ngt][tgt] - max_log_prob - log_sum_prob);
            if (tgt == 0) nonsom_prob += pp;
            else som_prob_given_ngt += pp;
        }
        const double err_som_and_ngt = 1.0 - som_prob_given_ngt;
        if (err_som_and_ngt < min_not_somfrom_sum)
        {
            min_not_somfrom_sum = err_som_and_ngt;
            rs.from_ntype_qphred = error_prob_to_qphred(err_som_and_ngt);
            rs.ntype = ngt;
        }
    }
    rs.qphred = error_prob_to_qphred(nonsom_prob);
}
} // namespace

// one record per locus, as sx_somatic_indel writes it (the caps give SX_SINDEL_ST_CAP; a bad candidate or error index: -1)
extern "C" int ox_somatic_indel(const sx_sindel_opts* o, const sx_sindel_batch* b, const double* err_prob, uint32_t n_err, sx_sindel_result* out)
{
    deriv D;
    D.rbm[0] = std::log(o->randomBaseMatchProb);
    D.rbm[1] = std::log(o->tier2RandomBaseMatchProb);
    D.cmlp = std::log(1.7e-10);
    const double theta = o->bindel_diploid_theta;
    D.germ[0] = (blt_float_t)log1p_switch_host(-(3. * theta) / 2.);
    D.germ[1] = (blt_float_t)std::log(theta / 2.);
    D.germ[2] = (blt_float_t)std::log(theta);
    D.ln_som_match = (blt_float_t)log1p_switch_host(-o->somatic_indel_rate);
    D.ln_som_mismatch = (blt_float_t)std::log(o->somatic_indel_rate);
    for (uint32_t l = 0; l < b->n_loci; ++l)
    {
        sx_sindel_result& res = out[l];
        std::memset(&res, 0, sizeof(res));
        const sx_indel_key& key = b->key[l];
        if (key.type != SX_INDEL_TYPE_INDEL || b->err_idx[l] >= n_err) return -1;
        const bool forced = b->is_forced_output[l] != 0;
        const sx_indel_key* alts = b->alts + b->alt_off[l];
        const uint32_t n_alts = b->alt_off[l + 1] - b->alt_off[l];
        const sx_sindel_read* rb[3] = {b->reads + b->read_off[2 * l], b->reads + b->read_off[2 * l + 1], b->reads + b->read_off[2 * l + 2]};
        bool over = n_alts > SX_SINDEL_MAX_ALTS;
        for (const sx_sindel_read* p = rb[0]; p < rb[2]; ++p)
            if (p->n_alt > 2 || (p->n_alt > 0 && p->alt[0] >= n_alts) || (p->n_alt > 1 && p->alt[1] >= n_alts)) over = true;
        if (over)
        {
            res.status = SX_SINDEL_ST_CAP;
            continue;
        }
        const double sharedIndelErrorRate(std::pow(err_prob[b->err_idx[l]], o->shared_indel_error_factor));
        const double logSharedIndelErrorRate(std::log(sharedIndelErrorRate));
        const double logSharedIndelErrorRateComplement(log1p_switch_host(-sharedIndelErrorRate));
        sx_sindel_tier* trs = res.tier;
        for (unsigned i = 0; i < 2; ++i)
        {
            const bool t2 = (i == 1);
            if (t2)
            {
                if (!o->useTier2Evidence) continue;
                if (trs[0].qphred == 0 && !forced)
                {
                    trs[1].qphred = 0;
                    continue;
                }
            }
            bool overlap = false;
            const bool filt = is_multi_indel_allele(D, alts, rb, t2, overlap);
            trs[i].is_overlap = overlap;
            trs[i].multi_indel = filt;
            if (filt && !forced)
            {
                trs[i].qphred = 0;
                continue;
            }
            double nl[21], tl[21];
            sample_lhood(D, rb[0], rb[1], key, (unsigned)o->min_read_bp_flank[0], t2, nl);
            sample_lhood(D, rb[1], rb[2], key, (unsigned)o->min_read_bp_flank[1], t2, tl);
            for (int j = 0; j < 21; ++j)
            {
                trs[i].normal_lhood[j] = (blt_float_t)nl[j];
                trs[i].tumor_lhood[j] = (blt_float_t)tl[j];
            }
            result_set_grid((blt_float_t)o->indel_contam_tolerance, (blt_float_t)logSharedIndelErrorRate, (blt_float_t)logSharedIndelErrorRateComplement,
                            trs[i].normal_lhood, trs[i].tumor_lhood, D, trs[i]);
            if (filt) trs[i].qphred = 0;
            trs[i].evaluated = 1;
        }
        if (!forced && (trs[0].qphred == 0 || trs[1].qphred == 0)) continue;
        unsigned sindel_tier = 0, from_tier = 0;
        if (o->useTier2Evidence)
        {
            if (trs[0].qphred > trs[1].qphred) sindel_tier = 1;
            if (trs[0].from_ntype_qphred > trs[1].from_ntype_qphred) from_tier = 1;
        }
        res.is_output = 1;
        res.sindel_tier = sindel_tier;
        res.sindel_from_ntype_tier = from_tier;
        res.is_overlap = trs[from_tier].is_overlap;
        res.max_gt = trs[from_tier].max_gt;
        res.from_ntype_qphred = trs[from_tier].from_ntype_qphred;
        if (trs[0].ntype != trs[1].ntype)
        {
            res.ntype = 3;
            res.from_ntype_qphred = 0;
        }
        else res.ntype = trs[from_tier].ntype == 0 ? 0 : trs[from_tier].ntype == 1 ? 1 : 2;
        res.qphred = trs[sindel_tier].qphred;
    }
    return 0;
}
