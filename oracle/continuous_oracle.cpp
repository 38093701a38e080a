// oracle/continuous_oracle.cpp -- TEST INFRASTRUCTURE, not product code.  A scalar restatement of the germline caller's continuous-frequency
// site model on the reference's containers' semantics: per position the skip test of process_pos_snp (starling_pos_processor.cpp:154-172),
// CleanPileupFilter (tier1) into a vector of calls, then process_pos_snp_continuous's addBase loop (:926-996) with
// updateContinuousSnvLocusWithSampleInfo (:751-881, allele-index table and per-call strand counts as written there) and
// updateContinuousSnvLocusInfo (:885-921).  The two Boost.Math functions are NOT restated here: they come from the kernels' own body
// (k2c_core.cuh: k2c_qscore, k2c_strand_bias), so comparing this oracle with the body checks the loci, counts, GT, reportability and order
// only.  GQ and strand bias are checked against the reference's own functions instead (tests/test_continuous.py: the exhaustive GQ grid and
// the strand-bias answers frozen in tests/golden/continuous_ref.npz).
#include "k2c_core.cuh"

#include <algorithm>
#include <vector>

namespace
{
struct call
{
    uint32_t base; // 0..3, 4 = ANY
    bool fwd;
};

struct sample_pileup
{
    std::vector<call> cleaned;
    uint32_t raw = 0;
};

struct locus
{
    sx_cont_locus rec;
    std::vector<sx_cont_sample> samples;
};
} // namespace

extern "C" uint32_t ocont_run(const sx_cont_opts* o, double err_rate, const sx_cont_batch* b, sx_cont_locus* loci_out, sx_cont_sample* samples_out,
                              uint32_t* site_rec_off, uint32_t cap_loci)
{
    const uint32_t S = b->n_samples;
    std::vector<locus> out;
    site_rec_off[0] = 0;
    for (uint32_t site = 0; site < b->n_sites; ++site)
    {
        const bool forced = b->forced_output && b->forced_output[site];
        std::vector<sample_pileup> sp(S);
        bool zero = true;
        for (uint32_t s = 0; s < S; ++s)
        {
            const sx_pileup_batch& p = b->sample[s];
            sp[s].raw = p.site_off[site + 1] - p.site_off[site];
            if (sp[s].raw) zero = false;
            for (uint32_t i = p.site_off[site]; i < p.site_off[site + 1]; ++i)
            {
                const uint32_t c = p.calls[i];
                if ((c >> 12) & 1u) continue; // is_call_filter
                const uint32_t id = (c >> 6) & 15u;
                sp[s].cleaned.push_back(call{id < 4 ? id : 4u, ((c >> 10) & 1u) != 0});
            }
        }
        if (!forced && zero)
        {
            site_rec_off[site + 1] = static_cast<uint32_t>(out.size());
            continue;
        }
        const char rb = b->sample[0].ref_base[site];
        const uint32_t ref = rb == 'A' ? 0 : rb == 'C' ? 1 : rb == 'G' ? 2 : rb == 'T' ? 3 : 4;
        bool any_output = false;
        auto add_base = [&](const uint32_t base, const bool forced_used) {
            const bool is_ref = base == ref;
            locus L;
            L.rec = sx_cont_locus{};
            L.rec.pos = b->pos_begin + static_cast<int32_t>(site);
            L.rec.alt = static_cast<uint8_t>(is_ref ? SX_CONT_REF_LOCUS : base);
            L.rec.ref = static_cast<uint8_t>(ref);
            L.rec.forced = forced ? 1 : 0;
            uint32_t sb[4] = {0, 0, 0, 0};
            for (uint32_t s = 0; s < S; ++s)
            {
                sx_cont_sample e = sx_cont_sample{};
                // AD: the allele-index table of the reference (its entry for an 'N' reference lies past the four bases; no call reads it)
                uint32_t idx[4] = {2, 2, 2, 2};
                const uint32_t full = is_ref ? 1u : 2u;
                for (uint32_t i = 0; i < 4; ++i) idx[i] = full;
                if (ref < 4) idx[ref] = 0;
                if (!is_ref) idx[base] = 1;
                uint32_t conf[2][2] = {{0, 0}, {0, 0}}, nonconf[2] = {0, 0};
                for (const call& c : sp[s].cleaned)
                {
                    if (c.base == 4) continue;
                    if (idx[c.base] == full)
                        ++nonconf[c.fwd];
                    else
                        ++conf[c.fwd][idx[c.base]];
                }
                e.ref_fwd = conf[1][0];
                e.ref_rev = conf[0][0];
                e.alt_fwd = is_ref ? 0 : conf[1][1];
                e.alt_rev = is_ref ? 0 : conf[0][1];
                e.non_confident_fwd = nonconf[1];
                e.non_confident_rev = nonconf[0];
                // strand bias over every cleaned call
                double strand_bias = 0.0;
                if (!is_ref)
                {
                    uint32_t fa = 0, ra = 0, fo = 0, ro = 0;
                    for (const call& c : sp[s].cleaned)
                    {
                        if (c.fwd)
                        {
                            if (c.base == base) ++fa;
                            else ++fo;
                        }
                        else if (c.base == base) ++ra;
                        else ++ro;
                    }
                    strand_bias = k2c_strand_bias(fa, ra, fo, ro);
                    sb[0] += fa;
                    sb[1] += ra;
                    sb[2] += fo;
                    sb[3] += ro;
                }
                e.strand_bias = std::min(o->max_abs_sample_strand_bias, std::max(-o->max_abs_sample_strand_bias, strand_bias));
                e.used = static_cast<uint32_t>(sp[s].cleaned.size());
                e.unused = sp[s].raw - e.used;
                // the cleaned pileup's spanningDeletionReadCount is 0
                e.total_depth = 0 + conf[1][0] + conf[1][1] + conf[0][0] + conf[0][1] + nonconf[1] + nonconf[0];
                e.allele_depth = is_ref ? conf[1][0] + conf[0][0] : conf[1][1] + conf[0][1];
                e.af = e.total_depth == 0 ? 0.0 : e.allele_depth / static_cast<double>(e.total_depth);
                if (is_ref) e.gt = SX_CONT_GT_HOMREF;
                else if (e.af >= (1. - o->min_het_vf)) e.gt = SX_CONT_GT_HOM;
                else if (e.af < o->min_het_vf) e.gt = SX_CONT_GT_HOMREF;
                else e.gt = SX_CONT_GT_HET;
                const k2c_q q = k2c_qscore(e.allele_depth, e.total_depth, err_rate, o->max_qscore);
                e.gq = q.gq;
                e.status = q.status;
                L.samples.push_back(e);
            }
            bool reportable = forced_used;
            if (!reportable && !is_ref)
                for (uint32_t s = 0; s < S; ++s)
                    if (L.samples[s].af > o->min_het_vf)
                    {
                        reportable = true;
                        break;
                    }
            if (!reportable) return;
            if (!is_ref)
            {
                L.rec.sb_fwd_alt = sb[0];
                L.rec.sb_rev_alt = sb[1];
                L.rec.sb_fwd_other = sb[2];
                L.rec.sb_rev_other = sb[3];
                L.rec.strand_bias = k2c_strand_bias(sb[0], sb[1], sb[2], sb[3]);
                for (uint32_t s = 0; s < S; ++s) L.rec.qual = std::max(L.rec.qual, L.samples[s].gq);
            }
            any_output = true;
            out.push_back(L);
        };
        for (uint32_t base = 0; base < 4; ++base)
        {
            if (base == ref) continue;
            add_base(base, forced);
        }
        if (!any_output) add_base(ref, true);
        site_rec_off[site + 1] = static_cast<uint32_t>(out.size());
    }
    const uint32_t total = static_cast<uint32_t>(out.size());
    if (total > cap_loci) return total;
    for (uint32_t r = 0; r < total; ++r)
    {
        loci_out[r] = out[r].rec;
        for (uint32_t s = 0; s < S; ++s) samples_out[(size_t)r * S + s] = out[r].samples[s];
    }
    return total;
}
