// ref_harness_indel_reads.cpp -- TEST INFRASTRUCTURE ONLY (oracle/_ref/libstrelka_ref_indel_reads.so, built by
// oracle/build_ref_indel_reads.sh next to the other reference-backed checkers).
//
// Pins the chain K6 -> K6b -> K5b against the reference's own containers, with no hand-made transpose in between: ONE two-sample
// IndelBuffer is rebuilt from the IndelKeys of two flattened sx_score_indels_batch (normal = sample 0, tumor = sample 1), the UNMODIFIED
// score_indels (starling_common/starling_read_align_score_indels.cpp:454) runs for every read of both samples with its sampleIndex and
// its rseg.getReadIndex(), and then, for every candidate, the UNMODIFIED somatic_indel_caller_grid::get_somatic_indel
// (applications/strelka/somatic_indel_grid.cpp:181) runs on the buffer's own IndelData, as strelka_pos_processor.cpp:343-348 does.  On
// request the buffer's read_path_lnp maps are also flattened, in the maps' own iteration order, so a test can lay them beside the link.
// The harness never sees a window index -> id table: a window entry is known to it only as an IndelKey.
//
// As in ref_harness_score_indels.cpp, this unit includes starling_read_align.cpp to reach the file-static tie-break
// isFirstCandidateAlignmentPreferred (nothing is copied or modified), and injects error rates through IndelSampleData's private
// _errorRates with the explicit-instantiation idiom.
#include "../include/strelka_b200.h"

#include "starling_common/starling_read_align.cpp" // NOLINT: see above

#include "applications/strelka/qscore_calculator.hh"
#include "applications/strelka/somatic_indel_grid.hh"
#include "applications/strelka/strelka_shared.hh"
#include "blt_util/math_util.hh"
#include "htsapi/align_path_bam_util.hh"
#include "htsapi/bam_record.hh"
#include "starling_common/starling_indel_call_pprob_digt.hh"
#include "starling_common/starling_read.hh"
#include "starling_common/starling_read_align_score_indels.hh"

#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

namespace
{
template <typename Tag, typename Tag::type M> struct MemberPtrOf4
{
    friend typename Tag::type memberPtr(Tag) { return M; }
};
struct LinkErrorRatesTag
{
    typedef IndelErrorRates IndelSampleData::*type;
    friend type memberPtr(LinkErrorRatesTag);
};
template struct MemberPtrOf4<LinkErrorRatesTag, &IndelSampleData::_errorRates>;

IndelKey key_of(const sx_indel_key& k, const char* pool, const uint32_t* off, const uint32_t i)
{
    const std::string ins(pool + off[i], pool + off[i + 1]);
    if (ins.size() != k.ins_len) throw blt_exception("ref_indel_reads: insert sequence length does not match ins_len");
    return IndelKey(k.pos, (k.type == SX_INDEL_TYPE_MISMATCH) ? INDEL::MISMATCH : INDEL::INDEL, k.del_len, ins.c_str());
}

void cal_of(const sx_score_indels_batch* b, const uint32_t a, const bool fwd, const std::vector<IndelKey>& winKeys, CandidateAlignment& cal)
{
    cal.al.pos = b->aln_pos[a];
    cal.al.is_fwd_strand = fwd;
    for (uint32_t s = b->aln_seg_off[a]; s < b->aln_seg_off[a + 1]; ++s)
    {
        const sx_aln_seg& sg(b->segs[s]);
        ALIGNPATH::align_t t(ALIGNPATH::NONE);
        switch (sg.kind)
        {
        case SX_SEG_MATCH: t = ALIGNPATH::MATCH; break;
        case SX_SEG_INSERT: t = ALIGNPATH::INSERT; break;
        case SX_SEG_DELETE: t = ALIGNPATH::DELETE; break;
        case SX_SEG_SOFTCLIP: t = ALIGNPATH::SOFT_CLIP; break;
        case SX_SEG_HARDCLIP: t = ALIGNPATH::HARD_CLIP; break;
        default: throw blt_exception("ref_indel_reads: segment kind outside score_indels' domain");
        }
        cal.al.path.push_back(ALIGNPATH::path_segment(t, sg.len));
    }
    indel_set_t iset;
    for (uint32_t i = b->aln_key_off[a]; i < b->aln_key_off[a + 1]; ++i) iset.insert(winKeys.at(b->aln_keys[i]));
    cal.setIndels(iset);
}
} // namespace

struct ref_indel_reads_sample // one sample: its K6 batch, K1's scores, the insert sequences behind its window entries, its read ids
{
    const sx_score_indels_batch* b;
    const double* lnp;
    const char* ins_pool;
    const uint32_t* ins_off;
    const uint32_t* read_id;
};

struct ref_indel_reads_maps // optional: the buffer's read_path_lnp maps of the candidates, flattened in iteration order
{
    uint32_t* read_off;     // [2 * n_loci + 1]
    sx_sindel_read* reads;  // alt[] as indices into the locus's table
    uint32_t* entry_id;     // the map key (read id) of each entry
    uint32_t* alt_off;      // [n_loci + 1]
    uint32_t* alt_gid;      // the locus's table: the distinct ids its entries name, ascending
    uint32_t cap_reads, cap_alts;
};

// gid_key / gid_ins_*: every IndelKey of the batch by id (the buffer is filled from these).  out[l]: as ref_somatic_indel writes it.
extern "C" int ref_indel_reads_chain(const sx_sindel_opts* o, const ref_indel_reads_sample* samples /*[2]*/, const sx_indel_key* gid_key, const char* gid_ins_pool,
                                     const uint32_t* gid_ins_off, uint32_t n_gid, const sx_indel_loci* loci, const double* err_prob, uint32_t n_err,
                                     sx_sindel_result* out, ref_indel_reads_maps* maps, char* err, int errlen)
{
    try
    {
        strelka_options opt;
        opt.alignFileOpt.alignmentFilenames = {"normal.bam", "tumor.bam"};
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
        const sx_score_indels_opts& so(samples[0].b->opts);
        opt.is_candidate_indel_signal_test = false;
        opt.maxIndelSize = so.max_indel_size;
        opt.upstream_oligo_size = so.upstream_oligo_size;
        opt.is_smoothed_alignments = (so.is_smoothed_alignments != 0);
        opt.smoothed_lnp_range = so.smoothed_lnp_range;
        const strelka_deriv_options dopt(opt);
        starling_sample_options sample_opt[2] = {starling_sample_options(opt), starling_sample_options(opt)};
        sample_opt[0].min_read_bp_flank = opt.normal_sample_min_read_bp_flank; // strelka_pos_processor.cpp:58
        for (unsigned s = 0; s < 2; ++s)
            if (samples[s].b->opts.min_read_bp_flank != sample_opt[s].min_read_bp_flank || samples[s].b->opts.max_indel_size != so.max_indel_size)
                throw blt_exception("ref_indel_reads: the K6 batches' options differ from the caller's sample options");
        const auto errorRatesPtr(memberPtr(LinkErrorRatesTag()));

        // ---- one buffer over every key
        std::vector<IndelKey> keyOfGid;
        std::map<IndelKey, uint32_t> gidOfKey;
        int32_t lo(n_gid ? gid_key[0].pos : 0), hi(lo + 1);
        for (uint32_t g = 0; g < n_gid; ++g)
        {
            keyOfGid.push_back(key_of(gid_key[g], gid_ins_pool, gid_ins_off, g));
            if (!gidOfKey.insert(std::make_pair(keyOfGid.back(), g)).second) throw blt_exception("ref_indel_reads: two ids for one IndelKey");
            lo = std::min(lo, gid_key[g].pos);
            hi = std::max(hi, gid_key[g].pos + (int32_t)gid_key[g].del_len);
        }
        reference_contig_segment ref;
        {
            std::string seq;
            static const char cyc[4] = {'A', 'C', 'G', 'T'};
            for (int32_t p = lo - 512; p < hi + 512; ++p) seq.push_back(cyc[(p & 0x7fffffff) % 4]);
            ref.seq() = seq;
            ref.set_offset(lo - 512);
        }
        IndelBuffer indelBuffer(opt, dopt, ref);
        depth_buffer db[2], db2[2];
        indelBuffer.registerSample(db[0], db2[0], false);
        indelBuffer.registerSample(db[1], db2[1], false);
        indelBuffer.finalizeSamples();
        for (uint32_t g = 0; g < n_gid; ++g)
            for (unsigned s = 0; s < 2; ++s)
            {
                IndelObservation obs;
                obs.key = keyOfGid[g];
                obs.data.id = 1000000 + 2 * g + s;
                obs.data.iat = INDEL_ALIGN_TYPE::GENOME_TIER1_READ;
                indelBuffer.addIndelObservation(s, obs);
            }
        // the per-sample facts score_indels reads, from each sample's window entries
        for (unsigned s = 0; s < 2; ++s)
        {
            const sx_score_indels_batch* b(samples[s].b);
            for (uint32_t k = 0; k < b->n_keys; ++k)
            {
                IndelData* idp(indelBuffer.getIndelDataPtr(key_of(b->keys[k], samples[s].ins_pool, samples[s].ins_off, k)));
                if (idp == nullptr) throw blt_exception("ref_indel_reads: a window entry is no key of the batch");
                const bool cand((b->keys[k].flags & SX_IKF_CANDIDATE) != 0);
                if (idp->status.is_candidate_indel_cached && idp->status.is_candidate_indel != cand) throw blt_exception("ref_indel_reads: candidacy differs between windows");
                idp->status.is_candidate_indel = cand;
                idp->status.is_candidate_indel_cached = true;
                IndelErrorRates& rates(idp->getSampleData(s).*errorRatesPtr);
                rates.refToIndelErrorProb.updateLogValue(b->keys[k].ref_to_indel_lnp);
                rates.indelToRefErrorProb.updateLogValue(b->keys[k].indel_to_ref_lnp);
            }
        }
        for (uint32_t g = 0; g < n_gid; ++g) // (an id in no window: no read can evaluate it)
        {
            IndelData* idp(indelBuffer.getIndelDataPtr(keyOfGid[g]));
            if (idp->status.is_candidate_indel_cached) continue;
            idp->status.is_candidate_indel = false;
            idp->status.is_candidate_indel_cached = true;
        }

        // ---- score_indels for every read of both samples
        std::vector<std::unique_ptr<bam_record>> bams;
        std::vector<std::unique_ptr<starling_read>> sreads;
        for (unsigned s = 0; s < 2; ++s)
        {
            const sx_score_indels_batch* b(samples[s].b);
            const double* lnp(samples[s].lnp);
            if (b->full_len || b->full_off) throw blt_exception("ref_indel_reads: only full read segments are rebuilt");
            for (uint32_t region = 0; region < b->n_regions; ++region)
            {
                std::vector<IndelKey> winKeys;
                for (uint32_t k = b->region_key_off[region]; k < b->region_key_off[region + 1]; ++k) winKeys.push_back(key_of(b->keys[k], samples[s].ins_pool, samples[s].ins_off, k));
                for (uint32_t r = b->region_read_off[region]; r < b->region_read_off[region + 1]; ++r)
                {
                    const uint32_t a0(b->aln_off[r]), a1(b->aln_off[r + 1]);
                    if (a0 == a1) continue;
                    const bool fwd((b->read_flags[r] & SX_SIF_FWD) != 0);
                    const int len(b->read_len[r]);
                    std::unique_ptr<bam_record> br(new bam_record);
                    br->set_qname("R");
                    std::string seq(len, 'A');
                    for (int i = 0; i < len - (int)b->non_ambig[r]; ++i) seq[i] = 'N';
                    const std::vector<uint8_t> qual(len, 30);
                    br->set_readqual(seq.c_str(), qual.data());
                    alignment al;
                    al.pos = b->aln_pos[a0];
                    al.is_fwd_strand = fwd;
                    al.path.push_back(ALIGNPATH::path_segment(ALIGNPATH::MATCH, len));
                    br->get_data()->core.pos = al.pos;
                    edit_bam_cigar(al.path, *(br->get_data()));
                    if (!fwd) br->get_data()->core.flag |= 0x10;
                    sreads.emplace_back(new starling_read(*br, al, (b->read_flags[r] & SX_SIF_TIER1) ? MAPLEVEL::TIER1_MAPPED : MAPLEVEL::TIER2_MAPPED, samples[s].read_id[r]));
                    bams.push_back(std::move(br));
                    const read_segment& rseg(sreads.back()->get_full_segment());
                    std::set<CandidateAlignment> cals;
                    std::vector<double> scores;
                    for (uint32_t a = a0; a < a1; ++a)
                    {
                        CandidateAlignment cal;
                        cal_of(b, a, fwd, winKeys, cal);
                        const auto ins(cals.insert(cal));
                        if (!ins.second || std::next(ins.first) != cals.end()) throw blt_exception("ref_indel_reads: alignments are not in std::set<CandidateAlignment> order");
                        scores.push_back(lnp[a]);
                    }
                    // starling_read_align.cpp:1573-1593 with the reference's own tie-break
                    double maxScore(0);
                    const CandidateAlignment* maxPtr(nullptr);
                    uint32_t index(0);
                    for (const CandidateAlignment& ical : cals)
                    {
                        const double path_lnp(scores[index++]);
                        if (nullptr != maxPtr)
                        {
                            if (path_lnp < maxScore) continue;
                            if ((path_lnp <= maxScore) && isFirstCandidateAlignmentPreferred(indelBuffer, *maxPtr, ical)) continue;
                        }
                        maxScore = path_lnp;
                        maxPtr = &ical;
                    }
                    score_indels(opt, dopt, sample_opt[s], rseg, indelBuffer, s, cals, (b->read_flags[r] & SX_SIF_INCOMPLETE) != 0, scores, maxScore, maxPtr);
                }
            }
        }

        // ---- get_somatic_indel on the buffer's own IndelData, and the maps as they stand
        blt_float_t germ[3];
        calculateGermlineGenotypeLogPrior(opt.bindel_diploid_theta, germ);
        const blt_float_t ln_som_match(log1p_switch(-opt.somatic_indel_rate)), ln_som_mismatch(std::log(opt.somatic_indel_rate));
        uint32_t n_entries(0), n_alts(0);
        for (uint32_t l = 0; l < loci->n_loci; ++l)
        {
            sx_sindel_result& r(out[l]);
            std::memset(&r, 0, sizeof(r));
            if (loci->gid[l] >= n_gid || loci->err_idx[l] >= n_err) throw blt_exception("ref_indel_reads: locus id or error-rate index out of range");
            const IndelKey& indelKey(keyOfGid[loci->gid[l]]);
            IndelData& indelData(*indelBuffer.getIndelDataPtr(indelKey));
            if (maps)
            {
                std::set<uint32_t> named;
                for (unsigned s = 0; s < 2; ++s)
                    for (const auto& val : indelData.getSampleData(s).read_path_lnp)
                        for (const auto& alt : val.second.alt_indel) named.insert(gidOfKey.at(alt.first));
                const std::vector<uint32_t> table(named.begin(), named.end());
                maps->alt_off[l] = n_alts;
                if (n_alts + table.size() > maps->cap_alts) throw blt_exception("ref_indel_reads: alternate capacity");
                for (const uint32_t g : table) maps->alt_gid[n_alts++] = g;
                for (unsigned s = 0; s < 2; ++s)
                {
                    maps->read_off[2 * l + s] = n_entries;
                    for (const auto& val : indelData.getSampleData(s).read_path_lnp)
                    {
                        if (n_entries >= maps->cap_reads) throw blt_exception("ref_indel_reads: entry capacity");
                        const ReadPathScores& rps(val.second);
                        sx_sindel_read& e(maps->reads[n_entries]);
                        std::memset(&e, 0, sizeof(e));
                        e.ref = rps.ref;
                        e.indel = rps.indel;
                        e.read_length = rps.read_length;
                        e.non_ambig = rps.nonAmbiguousBasesInRead;
                        e.is_tier1 = rps.is_tier1_read;
                        e.n_alt = rps.alt_indel.size();
                        for (unsigned a = 0; a < rps.alt_indel.size() && a < 2; ++a)
                        {
                            const uint32_t g(gidOfKey.at(rps.alt_indel[a].first));
                            e.alt[a] = std::lower_bound(table.begin(), table.end(), g) - table.begin();
                            e.alt_lnp[a] = rps.alt_indel[a].second;
                        }
                        maps->entry_id[n_entries++] = val.first;
                    }
                }
            }
            indelData.isForcedOutput = (loci->is_forced_output[l] != 0);
            (indelData.getSampleData(1).*errorRatesPtr).indelToRefErrorProb.updateValue(err_prob[loci->err_idx[l]]);
            somatic_indel_call sindel;
            sindel.sindel_tier = false;
            sindel.sindel_from_ntype_tier = false;
            sindel.rs.ntype = 0;
            sindel.rs.max_gt = 0;
            dopt.sicaller_grid().get_somatic_indel(opt, dopt, sample_opt[0], sample_opt[1], indelKey, indelData, 0, 1, true, sindel);
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
            // per tier, as ref_harness_somatic_indel.cpp reports it: the exported likelihood functions and calculate_result_set_grid
            const double sharedIndelErrorRate(std::pow(err_prob[loci->err_idx[l]], opt.shared_indel_error_factor));
            const double lse(std::log(sharedIndelErrorRate)), lcse(log1p_switch(-sharedIndelErrorRate));
            for (unsigned t = 0; t < 2; ++t)
            {
                sx_sindel_tier& T(r.tier[t]);
                for (unsigned s = 0; s < 2; ++s)
                {
                    const IndelSampleData& isd(indelData.getSampleData(s));
                    double lhood[21];
                    get_indel_digt_lhood(opt, dopt, sample_opt[s], indelKey, isd, t == 1, true, lhood);
                    for (unsigned i = 0; i < 9; ++i)
                    {
                        const double het_ratio((i + 1) * DIGT_GRID::RATIO_INCREMENT);
                        get_high_low_het_ratio_lhood(opt, dopt, sample_opt[s], indelKey, isd, het_ratio, t == 1, true, lhood[3 + 18 - (i + 1)], lhood[3 + i]);
                    }
                    for (unsigned j = 0; j < 21; ++j) (s == 0 ? T.normal_lhood : T.tumor_lhood)[j] = (blt_float_t)lhood[j];
                }
                indel_result_set rs;
                calculate_result_set_grid((float)opt.indel_contam_tolerance, (float)lse, (float)lcse, T.normal_lhood, T.tumor_lhood, germ, ln_som_match, ln_som_mismatch, rs);
                T.qphred = rs.qphred;
                T.from_ntype_qphred = rs.from_ntype_qphred;
                T.ntype = rs.ntype;
                T.max_gt = rs.max_gt;
                T.evaluated = 1;
            }
        }
        if (maps)
        {
            maps->read_off[2 * loci->n_loci] = n_entries;
            maps->alt_off[loci->n_loci] = n_alts;
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
