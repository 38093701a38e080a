// integration/sx_shim.hh -- the C++ shim a reference maintainer adds at the reference's own call sites to route the hot path through
// libstrelka_b200.so (include/strelka_b200.h).  Included ONLY by the patched copies of the reference's translation units that
// integration/build_patched.py makes (the reference tree itself is never modified, nor copied into this repository).
//
// One sx_ctx per process: the reference runs one single-threaded process per genome segment.  ABI errors become blt_exception, the
// reference's own convention (e.g. starling_pos_processor_base.cpp:755-760).  Setting SX_SHIM_OFF=1 in the environment keeps the
// reference's CPU functions (A/B runs of the same binary).
#pragma once

#include "strelka_b200.h"
#include "strelka_b200.hh"

#include "alignment/GlobalAligner.hh"
#include "blt_common/blt_shared.hh"
#include "blt_common/position_snp_call_pprob_digt.hh"
#include "blt_common/snp_pos_info.hh"
#include "blt_util/blt_exception.hh"

#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

namespace sx_shim
{
static_assert(sizeof(base_call) == 2, "base_call must be the 16-bit word the ABI carries (blt_common/snp_pos_info.hh:109-118)");

inline bool enabled()
{
    static const bool on(std::getenv("SX_SHIM_OFF") == nullptr);
    return on;
}

struct Counters
{
    unsigned long long site_gl_germline = 0, site_gl_somatic = 0, global_align = 0, somatic_indel = 0, germline_indel = 0, continuous_site = 0;
    bool germline_indel_route = false; // set by the translation unit that routes germline indel genotyping (SX_SHIM_GERMLINE)
    bool continuous_route = false;     // ... and continuous-frequency sites (SX_SHIM_CONTINUOUS)
    ~Counters()
    {
        // (fields are read by position: a new counter goes at the end, and only binaries with its route print it)
        if (std::getenv("SX_SHIM_REPORT"))
            std::fprintf(stderr, "sx_shim: %llu germline site calls, %llu somatic site calls, %llu haplotype alignments through libstrelka_b200.so, %llu somatic indel calls%s",
                         site_gl_germline, site_gl_somatic, global_align, somatic_indel, germline_indel_route ? ", " : "\n");
        // the continuous-site counter is appended only when that route ran, so the line of a diploid run is the one it has always been
        const bool cont(continuous_route && continuous_site > 0);
        if (std::getenv("SX_SHIM_REPORT") && germline_indel_route) std::fprintf(stderr, "%llu germline indel calls%s", germline_indel, cont ? ", " : "\n");
        if (std::getenv("SX_SHIM_REPORT") && cont) std::fprintf(stderr, "%llu continuous site calls\n", continuous_site);
    }
};
inline Counters& counters()
{
    static Counters c;
    return c;
}

inline sx_ctx* context(const sx_params& p)
{
    struct Holder
    {
        sx_ctx* ctx = nullptr;
        explicit Holder(const sx_params& q)
        {
            const char* dev(std::getenv("SX_SHIM_DEVICE"));
            if (sx_create(dev ? std::atoi(dev) : 0, &q, &ctx) != SX_OK) throw blt_exception(sx_last_error(nullptr));
        }
        ~Holder() { sx_destroy(ctx); }
    };
    static Holder h(p);
    return h.ctx;
}

inline void check(sx_ctx* ctx, const int rc)
{
    if (rc != SX_OK) throw blt_exception(sx_last_error(ctx));
}

inline sx_params params_of(const blt_options& opt)
{
    sx_params p;
    sx_default_params(&p);
    p.bsnp_diploid_theta = opt.bsnp_diploid_theta;
    p.bsnp_ssd_no_mismatch = opt.bsnp_ssd_no_mismatch;
    p.bsnp_ssd_one_mismatch = opt.bsnp_ssd_one_mismatch;
    p.is_min_vexp = opt.is_min_vexp;
    p.min_vexp = opt.min_vexp;
    p.is_bsnp_diploid = opt.is_bsnp_diploid();
    p.hetVariantFrequencyExtension = opt.hetVariantFrequencyExtension;
    return p;
}

inline const uint16_t* words(const std::vector<base_call>& v) { return reinterpret_cast<const uint16_t*>(v.data()); }

/// computeSampleDiploidSiteGenotype (applications/starling/starling_pos_processor.cpp:254-267): CleanPileupFilter + CleanPileupErrorProb +
/// position_snp_call_pprob_digt of one sample's position, from the RAW pile-up column
inline void site_gl_germline(const blt_options& opt, const snp_pos_info& raw, const bool is_always_test, diploid_genotype& dgt)
{
    sx_ctx* ctx(context(params_of(opt)));
    const uint32_t off[2] = {0u, static_cast<uint32_t>(raw.calls.size())};
    const uint16_t none(0);
    const char ref_base(raw.get_ref_base());
    const uint8_t ploidy(static_cast<uint8_t>(dgt.ploidy));
    sx_pileup_batch b;
    std::memset(&b, 0, sizeof(b));
    b.n_sites = 1;
    b.site_off = off;
    b.calls = raw.calls.empty() ? &none : words(raw.calls);
    b.ref_base = &ref_base;
    b.ploidy = &ploidy;
    sx_digt_result r;
    check(ctx, sx_site_gl_germline(ctx, &b, is_always_test ? 1 : 0, &r));
    ++counters().site_gl_germline;
    const int keep_ploidy(dgt.ploidy);
    dgt.reset();
    dgt.ploidy = keep_ploidy;
    dgt.ref_gt = r.ref_gt;
    if (!r.is_computed) return; // the reference returned before touching the rest (position_snp_call_pprob_digt.cpp:484-492)
    dgt.strand_bias = r.strand_bias;
    const sx_digt_result_set* in[2] = {&r.genome, &r.poly};
    diploid_genotype::result_set* out[2] = {&dgt.genome, &dgt.poly};
    for (int k = 0; k < 2; ++k)
    {
        out[k]->max_gt = in[k]->max_gt;
        out[k]->ref_pprob = in[k]->ref_pprob;
        out[k]->snp_qphred = in[k]->snp_qphred;
        out[k]->max_gt_qphred = in[k]->max_gt_qphred;
    }
    for (unsigned gt = 0; gt < 10; ++gt) dgt.phredLoghood[gt] = r.phredLoghood[gt];
}

/// _aligner.align(hap.begin, hap.end, ref.begin, ref.end, result) (starling_common/ActiveRegionProcessor.cpp:591)
inline void global_align(const AlignmentScores<int>& sc, const std::string& query, const std::string& ref, AlignmentResult<int>& result)
{
    sx_params p;
    sx_default_params(&p);
    sx_ctx* ctx(context(p));
    sx_ga_scores s = {sc.match, sc.mismatch, sc.open, sc.extend, sc.offEdge, sc.insertDelete, sc.isAllowEdgeInsertion ? 1 : 0, sc.isRequireEdgeDeletion ? 1 : 0};
    std::string q(query), r(ref);
    const uint32_t qo[2] = {0u, static_cast<uint32_t>(q.size())}, ro[2] = {0u, static_cast<uint32_t>(r.size())};
    const uint32_t maxOps(static_cast<uint32_t>(q.size() + r.size() + 2));
    q.resize(q.size() + 16);
    r.resize(r.size() + 16);
    sx_ga_batch b = {1u, q.data(), r.data(), qo, ro, maxOps};
    sx_ga_result res;
    std::vector<uint32_t> cig(maxOps);
    check(ctx, sx_global_align(ctx, &s, &b, &res, cig.data()));
    ++counters().global_align;
    if (res.status != 0) throw blt_exception("sx_global_align: problem too large for the kernel");
    result.score = res.score;
    result.align.beginPos = res.beginPos;
    result.align.apath.clear();
    static const ALIGNPATH::align_t kind[9] = {ALIGNPATH::MATCH, ALIGNPATH::INSERT, ALIGNPATH::DELETE, ALIGNPATH::SKIP, ALIGNPATH::SOFT_CLIP, ALIGNPATH::HARD_CLIP,
                                               ALIGNPATH::PAD, ALIGNPATH::SEQ_MATCH, ALIGNPATH::SEQ_MISMATCH};
    for (uint32_t k = 0; k < res.n_ops; ++k) result.align.apath.push_back(ALIGNPATH::path_segment(kind[cig[k] & 15u], cig[k] >> 4));
}

#ifdef SX_SHIM_SOMATIC
/// sscaller_strand_grid().position_somatic_snv_call(nepi, tepi, nepi_t2, tepi_t2, isComputeNonSomatic, sgtg)
/// (applications/strelka/strelka_pos_processor.cpp:213-219), from the RAW tumor / normal columns (tier1 + tier2 calls).  With
/// isComputeNonSomatic (--somatic-callable-regions-file) the call is K2b's callable mode, which also gives sgtg.rs.nonsomatic_qphred for the
/// reference's own SomaticCallableProcessor; those calls count as somatic site calls.
inline sx_params somatic_params_of(const strelka_options& opt)
{
    sx_params p(params_of(opt));
    p.somatic_snv_rate = opt.somatic_snv_rate;
    p.shared_site_error_rate = opt.shared_site_error_rate;
    p.shared_site_error_strand_bias_fraction = opt.shared_site_error_strand_bias_fraction;
    p.ssnv_contam_tolerance = opt.ssnv_contam_tolerance;
    return p;
}

inline void site_gl_somatic(const strelka_options& opt, const snp_pos_info& normal, const snp_pos_info& tumor, const bool isComputeNonSomatic,
                            somatic_snv_genotype_grid& sgtg)
{
    sx_ctx* ctx(context(somatic_params_of(opt)));
    const uint16_t none(0);
    const char ref_base(normal.get_ref_base());
    const snp_pos_info* pi[2] = {&normal, &tumor};
    uint32_t off[2][2], t2off[2][2];
    sx_pileup_batch b[2];
    for (int s = 0; s < 2; ++s)
    {
        off[s][0] = t2off[s][0] = 0;
        off[s][1] = static_cast<uint32_t>(pi[s]->calls.size());
        t2off[s][1] = static_cast<uint32_t>(pi[s]->tier2_calls.size());
        std::memset(&b[s], 0, sizeof(b[s]));
        b[s].n_sites = 1;
        b[s].site_off = off[s];
        b[s].calls = pi[s]->calls.empty() ? &none : words(pi[s]->calls);
        if (opt.useTier2Evidence)
        {
            b[s].t2_off = t2off[s];
            b[s].t2_calls = pi[s]->tier2_calls.empty() ? &none : words(pi[s]->tier2_calls);
        }
        b[s].ref_base = &ref_base;
    }
    const uint8_t forced(sgtg.is_forced_output ? 1 : 0);
    sx_ssnv_result r;
    check(ctx, isComputeNonSomatic ? sx_site_gl_somatic_callable(ctx, &b[0], &b[1], &forced, &r) : sx_site_gl_somatic(ctx, &b[0], &b[1], &forced, &r));
    ++counters().site_gl_somatic;
    sgtg.ref_gt = r.ref_gt;
    if (!r.is_computed) return;
    sgtg.snv_tier = r.snv_tier != 0;
    sgtg.snv_from_ntype_tier = r.snv_from_ntype_tier != 0;
    sgtg.rs.ntype = r.ntype;
    sgtg.rs.max_gt = r.max_gt;
    sgtg.rs.qphred = r.qphred;
    sgtg.rs.from_ntype_qphred = r.from_ntype_qphred;
    sgtg.rs.normal_alt_id = r.normal_alt_id;
    sgtg.rs.tumor_alt_id = r.tumor_alt_id;
    sgtg.rs.strandBias = r.strandBias;
    sgtg.rs.nonsomatic_qphred = r.nonsomatic_qphred;
}

/// _dopt.sicaller_grid().get_somatic_indel(_opt, _dopt, normal_opt, tumor_opt, indelKey, indelData, NORMAL, TUMOR, is_use_alt_indel = true, sindel)
/// (applications/strelka/strelka_pos_processor.cpp:343-348) as a one-locus sx_somatic_indel batch built from the two samples' read_path_lnp.
/// A locus the library does not take -- more distinct alternates than SX_SINDEL_MAX_ALTS, a read with more than two, or an alternate that is
/// neither an indel nor a mismatch -- runs through the reference's own function instead.
inline void somatic_indel(const strelka_options& opt, const strelka_deriv_options& dopt, const starling_sample_options& normal_opt,
                          const starling_sample_options& tumor_opt, const IndelKey& indelKey, const IndelData& indelData, const unsigned normalSampleIndex,
                          const unsigned tumorSampleIndex, somatic_indel_call& sindel)
{
    auto cpu = [&]() {
        dopt.sicaller_grid().get_somatic_indel(opt, dopt, normal_opt, tumor_opt, indelKey, indelData, normalSampleIndex, tumorSampleIndex, true, sindel);
    };
    const IndelSampleData* sd[2] = {&indelData.getSampleData(normalSampleIndex), &indelData.getSampleData(tumorSampleIndex)};
    auto key_of = [](const IndelKey& k, sx_indel_key& o) {
        std::memset(&o, 0, sizeof(o));
        o.pos = static_cast<int32_t>(k.pos);
        o.del_len = static_cast<uint16_t>(k.delete_length());
        o.ins_len = static_cast<uint16_t>(k.insert_length());
        o.type = k.isMismatch() ? SX_INDEL_TYPE_MISMATCH : SX_INDEL_TYPE_INDEL;
    };
    // the distinct alternates the reads name (get_sum_path_pprob keys them by IndelKey) and the reads in map order
    std::vector<IndelKey> alt_keys;
    std::vector<sx_sindel_read> reads;
    uint32_t read_off[3] = {0u, 0u, 0u};
    for (unsigned s = 0; s < 2; ++s)
    {
        for (const auto& e : sd[s]->read_path_lnp)
        {
            const ReadPathScores& rp(e.second);
            if (rp.alt_indel.size() > 2) return cpu();
            sx_sindel_read r;
            std::memset(&r, 0, sizeof(r));
            r.ref = rp.ref;
            r.indel = rp.indel;
            r.read_length = rp.read_length;
            r.non_ambig = rp.nonAmbiguousBasesInRead;
            r.is_tier1 = rp.is_tier1_read ? 1 : 0;
            r.n_alt = static_cast<uint8_t>(rp.alt_indel.size());
            for (unsigned k = 0; k < rp.alt_indel.size(); ++k)
            {
                const IndelKey& ak(rp.alt_indel[k].first);
                if (ak.type != INDEL::INDEL && ak.type != INDEL::MISMATCH) return cpu();
                unsigned idx(0);
                while (idx < alt_keys.size() && !(alt_keys[idx] == ak)) ++idx;
                if (idx == alt_keys.size())
                {
                    if (alt_keys.size() == SX_SINDEL_MAX_ALTS) return cpu();
                    alt_keys.push_back(ak);
                }
                r.alt[k] = static_cast<uint8_t>(idx);
                r.alt_lnp[k] = rp.alt_indel[k].second;
            }
            reads.push_back(r);
        }
        read_off[s + 1] = static_cast<uint32_t>(reads.size());
    }
    sx_ctx* ctx(context(somatic_params_of(opt)));
    sx_sindel_opts o;
    sx_default_sindel_opts(&o);
    o.somatic_indel_rate = opt.somatic_indel_rate;
    o.bindel_diploid_theta = opt.bindel_diploid_theta;
    o.indel_contam_tolerance = opt.indel_contam_tolerance;
    o.shared_indel_error_factor = opt.shared_indel_error_factor;
    o.randomBaseMatchProb = opt.randomBaseMatchProb;
    o.tier2RandomBaseMatchProb = opt.tier2.isRandomBaseMatchProb ? opt.tier2.randomBaseMatchProb : opt.randomBaseMatchProb; // starling_base_shared.cpp:44-52
    o.useTier2Evidence = opt.useTier2Evidence ? 1 : 0;
    o.min_read_bp_flank[0] = normal_opt.min_read_bp_flank;
    o.min_read_bp_flank[1] = tumor_opt.min_read_bp_flank;
    sx_indel_key key;
    key_of(indelKey, key);
    std::vector<sx_indel_key> alts(alt_keys.size() + 1);
    for (unsigned a = 0; a < alt_keys.size(); ++a) key_of(alt_keys[a], alts[a]);
    if (reads.empty()) reads.resize(1); // (a valid pointer; read_off says there are none)
    const uint8_t forced(indelData.isForcedOutput ? 1 : 0);
    const uint32_t err_idx(0), alt_off[2] = {0u, static_cast<uint32_t>(alt_keys.size())};
    const double err_prob(sd[1]->getErrorRates().indelToRefErrorProb.getValue());
    sx_sindel_batch b;
    std::memset(&b, 0, sizeof(b));
    b.n_loci = 1;
    b.key = &key;
    b.is_forced_output = &forced;
    b.err_idx = &err_idx;
    b.alt_off = alt_off;
    b.alts = alts.data();
    b.read_off = read_off;
    b.reads = reads.data();
    sx_sindel_result r;
    check(ctx, sx_somatic_indel(ctx, &o, &b, &err_prob, 1, &r));
    if (r.status != 0) return cpu(); // (SX_SINDEL_ST_CAP; not reached after the checks above)
    ++counters().somatic_indel;
    sindel.is_forced_output = indelData.isForcedOutput;
    if (!r.is_output) return; // the reference returned before the tier choice (somatic_indel_grid.cpp:296-300)
    sindel.sindel_tier = r.sindel_tier != 0;
    sindel.sindel_from_ntype_tier = r.sindel_from_ntype_tier != 0;
    sindel.rs.ntype = r.ntype;
    sindel.rs.max_gt = r.max_gt;
    sindel.rs.qphred = r.qphred;
    sindel.rs.from_ntype_qphred = r.from_ntype_qphred;
    sindel.rs.is_overlap = r.is_overlap != 0;
}
#endif

#ifdef SX_SHIM_GERMLINE
inline bool register_germline_indel_route()
{
    counters().germline_indel_route = true;
    return true;
}
static const bool germline_indel_route_registered = register_germline_indel_route();

/// getVariantAlleleGroupGenotypeLhoodsForSample(opt, dopt, sample_opt, callerPloidy, sampleIndex, alleleGroup, contrastGroup, genotypeLogLhood,
/// supportCounts) of updateIndelLocusWithSampleInfo (applications/starling/starling_pos_processor.cpp:1384) as a one-group sx_indel_gl batch.
/// The batch is filled with the reference's own getAlleleGroupSupportingReadIds / getAlleleLogLhoodFromRead and the contrast fold of
/// AlleleGroupGenotype.cpp:225-238.  K5's context is made for the run's randomBaseMatchProb, readConfidentSupportThreshold and the sample's
/// min_read_bp_flank; a group outside K5's domain (no or more than SX_INDEL_MAX_ALLELES alleles, a ploidy other than 1 or 2), or a call with
/// other values of those options than the context was made for, keeps the reference function.
inline void germline_indel(const starling_base_options& opt, const starling_base_deriv_options& dopt, const starling_sample_options& sample_opt,
                           const unsigned callerPloidy, const unsigned sampleIndex, const OrthogonalVariantAlleleCandidateGroup& alleleGroup,
                           const OrthogonalVariantAlleleCandidateGroup& contrastGroup, std::vector<double>& genotypeLogLhood, LocusSupportingReadStats& stats)
{
    sx_params p(params_of(opt));
    p.randomBaseMatchProb = opt.randomBaseMatchProb;
    p.readConfidentSupportThreshold = opt.readConfidentSupportThreshold.numval();
    p.min_read_bp_flank = sample_opt.min_read_bp_flank;
    struct Holder // K5's context: its tables are made from these options at sx_create
    {
        sx_ctx* ctx = nullptr;
        sx_params p;
        explicit Holder(const sx_params& q) : p(q)
        {
            const char* dev(std::getenv("SX_SHIM_DEVICE"));
            if (sx_create(dev ? std::atoi(dev) : 0, &q, &ctx) != SX_OK) throw blt_exception(sx_last_error(nullptr));
        }
        ~Holder() { sx_destroy(ctx); }
    };
    static Holder h(p);
    const unsigned A(alleleGroup.size());
    if (A < 1 || A > SX_INDEL_MAX_ALLELES || (callerPloidy != 1 && callerPloidy != 2) || h.p.randomBaseMatchProb != p.randomBaseMatchProb ||
        h.p.readConfidentSupportThreshold != p.readConfidentSupportThreshold || h.p.min_read_bp_flank != p.min_read_bp_flank)
    {
        getVariantAlleleGroupGenotypeLhoodsForSample(opt, dopt, sample_opt, callerPloidy, sampleIndex, alleleGroup, contrastGroup, genotypeLogLhood, stats);
        return;
    }
    std::set<unsigned> readIds;
    getAlleleGroupSupportingReadIds(sampleIndex, alleleGroup, readIds, true);
    OrthogonalVariantAlleleCandidateGroup extended(alleleGroup);
    for (const auto& it : contrastGroup.alleles) extended.alleles.push_back(it);
    std::vector<float> lnp;
    std::vector<uint16_t> read_length, non_ambig, del_len, ins_len;
    std::vector<uint8_t> is_fwd;
    for (const unsigned readId : readIds)
    {
        std::vector<double> v(extended.size() + 1);
        getAlleleLogLhoodFromRead(sampleIndex, extended, readId, v);
        for (unsigned i = A + 1; i < v.size(); ++i)
            if (v[i] > v[0]) v[0] = v[i];
        for (unsigned i = 0; i <= A; ++i) lnp.push_back(static_cast<float>(v[i])); // (ReadPathScores floats: exact)
        const ReadPathScores* ex(nullptr); // getExemplarReadScore
        for (unsigned a = 0; a < A && !ex; ++a)
        {
            const auto& m(alleleGroup.data(a).getSampleData(sampleIndex).read_path_lnp);
            const auto f(m.find(readId));
            if (f != m.end()) ex = &f->second;
        }
        read_length.push_back(ex->read_length);
        non_ambig.push_back(ex->nonAmbiguousBasesInRead);
        is_fwd.push_back(ex->is_fwd_strand ? 1 : 0);
    }
    for (unsigned a = 0; a < A; ++a)
    {
        del_len.push_back(static_cast<uint16_t>(alleleGroup.key(a).delete_length()));
        ins_len.push_back(static_cast<uint16_t>(alleleGroup.key(a).insert_length()));
    }
    const uint32_t n(readIds.size()), read_off[2] = {0, n}, lnp_off[2] = {0, n * (A + 1)}, allele_off[2] = {0, A};
    const uint8_t ploidy(static_cast<uint8_t>(callerPloidy));
    const float f0(0.f);
    const uint16_t u0(0);
    const uint8_t b0(0);
    sx_indel_batch b;
    b.n_loci = 1;
    b.read_off = read_off;
    b.lnp_off = lnp_off;
    b.allele_off = allele_off;
    b.ploidy = &ploidy;
    b.allele_del_len = del_len.data();
    b.allele_ins_len = ins_len.data();
    b.allele_lnp = n ? lnp.data() : &f0;
    b.read_length = n ? read_length.data() : &u0;
    b.non_ambig = n ? non_ambig.data() : &u0;
    b.is_fwd = n ? is_fwd.data() : &b0;
    sx_indel_result r;
    check(h.ctx, sx_indel_gl(h.ctx, &b, &r));
    ++counters().germline_indel;
    genotypeLogLhood.assign(r.gt_lhood, r.gt_lhood + r.n_gt);
    stats.setAltCount(A);
    for (int s = 0; s < 2; ++s)
    {
        SupportingReadCountGroup& c(stats.getCounts(s == 1));
        for (unsigned a = 0; a <= A; ++a)
            if (r.support[s][a]) c.incrementAlleleCount(a, r.support[s][a]);
        c.nonConfidentCount += r.support[s][SX_INDEL_MAX_ALLELES + 1];
    }
}
#endif

#ifdef SX_SHIM_CONTINUOUS
inline bool register_continuous_route()
{
    counters().continuous_route = true;
    return true;
}
static const bool continuous_route_registered = register_continuous_route();

inline sx_cont_opts cont_opts_of(const starling_options& opt)
{
    sx_cont_opts o;
    sx_default_cont_opts(&o);
    o.min_het_vf = opt.min_het_vf;
    o.max_abs_sample_strand_bias = opt.maxAbsSampleVariantStrandBias;
    o.expected_qscore = opt.continuousFrequencyCallerExpectedObservationQuality;
    o.max_qscore = opt.continuousFrequencyCallerMaxQscore;
    return o;
}

/// K2c's records of one position (process_pos_snp_continuous, applications/starling/starling_pos_processor.cpp:926-996) from every sample's RAW
/// column; the caller builds the loci from them with the reference's own updateSiteSampleInfo / updateContinuousSiteSampleInfo / add_site.
struct ContinuousSite
{
    std::vector<sx_cont_locus> loci;
    std::vector<sx_cont_sample> samples; // record r's sample s at r * n_samples + s
};

inline void continuous_site(const starling_options& opt, const std::vector<const snp_pos_info*>& raw, const char ref_base, const bool forced, const pos_t pos,
                            ContinuousSite& out)
{
    sx_ctx* ctx(context(params_of(opt)));
    const sx_cont_opts o(cont_opts_of(opt));
    const uint32_t S(static_cast<uint32_t>(raw.size()));
    const uint16_t none(0);
    const uint8_t f(forced ? 1 : 0);
    uint32_t off[SX_CONT_MAX_SAMPLES][2];
    sx_cont_batch b;
    std::memset(&b, 0, sizeof(b));
    b.n_sites = 1;
    b.n_samples = S;
    b.pos_begin = static_cast<int32_t>(pos);
    b.forced_output = &f;
    for (uint32_t s = 0; s < S; ++s)
    {
        off[s][0] = 0;
        off[s][1] = static_cast<uint32_t>(raw[s]->calls.size());
        b.sample[s].n_sites = 1;
        b.sample[s].site_off = off[s];
        b.sample[s].calls = raw[s]->calls.empty() ? &none : words(raw[s]->calls);
        b.sample[s].ref_base = &ref_base;
    }
    out.loci.resize(4);
    out.samples.resize(4 * S);
    uint32_t rec_off[2], total(0);
    sx_cont_out co;
    std::memset(&co, 0, sizeof(co));
    co.loci = out.loci.data();
    co.samples = out.samples.data();
    co.site_rec_off = rec_off;
    co.cap_loci = 4;
    check(ctx, sx_site_continuous(ctx, &o, &b, &co, &total));
    out.loci.resize(total);
    out.samples.resize((size_t)total * S);
    ++counters().continuous_site;
}

/// The K2c strand bias is within 1e-9 of the reference's (DESIGN.md section 3).  Within that of a multiple of 0.05 -- a boundary of the
/// one-decimal SB / SNVSB print or of the HighSNVSB threshold -- the reference's own strandBias decides.
inline bool near_strand_bias_boundary(const double sb)
{
    if (!std::isfinite(sb)) return false;
    const double k(std::floor(sb / 0.05 + 0.5));
    return std::fabs(sb - k * 0.05) < 1e-9;
}

/// the sample strand bias of updateContinuousSnvLocusWithSampleInfo (:789-824) from the cleaned calls, by the reference's function
inline double reference_sample_strand_bias(const snp_pos_info& cleaned, const unsigned alt)
{
    unsigned fa(0), ra(0), fo(0), ro(0);
    for (const base_call& bc : cleaned.calls)
    {
        if (bc.is_fwd_strand) (bc.base_id == alt ? fa : fo)++;
        else (bc.base_id == alt ? ra : ro)++;
    }
    return starling_continuous_variant_caller::strandBias(fa, ra, fo, ro);
}

/// getAlleleSequencingErrorQscore(a, n, ...) of the continuous indel genotype (starling_pos_processor.cpp:2026-2030) through sx_cont_qscore; a
/// tie-flagged answer is the reference function's
inline int cont_qscore(const starling_base_options& opt, const unsigned a, const unsigned n)
{
    sx_ctx* ctx(context(params_of(opt)));
    sx_cont_opts o;
    sx_default_cont_opts(&o);
    o.expected_qscore = opt.continuousFrequencyCallerExpectedObservationQuality;
    o.max_qscore = opt.continuousFrequencyCallerMaxQscore;
    int32_t gq(0);
    uint32_t st(0);
    check(ctx, sx_cont_qscore(ctx, &o, 1, &a, &n, &gq, &st));
    if (st & SX_CONT_ST_QSCORE_TIE)
        return starling_continuous_variant_caller::getAlleleSequencingErrorQscore(a, n, opt.continuousFrequencyCallerExpectedObservationQuality,
                                                                                  opt.continuousFrequencyCallerMaxQscore);
    return gq;
}
#endif
} // namespace sx_shim
