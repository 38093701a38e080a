// ref_harness_germline_indel.cpp -- TEST INFRASTRUCTURE ONLY (oracle/_ref/libstrelka_ref_germline_indel.so, built by
// oracle/build_ref_germline_indel.sh next to the other reference-backed checkers).
//
// Pins the chain K6 -> K6g -> K5 against the reference's own containers and functions, with no restatement in between: ONE one-sample
// IndelBuffer is rebuilt from the IndelKeys of a flattened sx_score_indels_batch, the UNMODIFIED score_indels
// (starling_common/starling_read_align_score_indels.cpp:454) runs for every read with its rseg.getReadIndex(), and then, for every allele
// group given by ids, OrthogonalVariantAlleleCandidateGroups of the buffer's own iterators go to the UNMODIFIED
//   getAlleleGroupSupportingReadIds     starling_common/OrthogonalVariantAlleleCandidateGroupUtil.cpp:113-128 (the supporting read ids)
//   getAlleleLogLhoodFromRead           :132-196, on the extended group (alleles, then contrasts), before the contrast fold
//   getVariantAlleleGroupGenotypeLhoodsForSample   starling_common/AlleleGroupGenotype.cpp:185-258 (genotype likelihoods, read stats)
// as updateIndelLocusWithSampleInfo (applications/starling/starling_pos_processor.cpp:1337-1400) does.  The harness never sees a window
// index -> id table: a window entry is known to it only as an IndelKey.
//
// As in ref_harness_indel_reads.cpp (which is left as it is; the few helpers below are restated here), this unit includes
// starling_read_align.cpp to reach the file-static tie-break isFirstCandidateAlignmentPreferred, and injects error rates through
// IndelSampleData's private _errorRates with the explicit-instantiation idiom.
#include "../include/strelka_b200.h"

#include "starling_common/starling_read_align.cpp" // NOLINT: see above

#include "blt_util/math_util.hh"
#include "htsapi/align_path_bam_util.hh"
#include "htsapi/bam_record.hh"
#include "starling_common/AlleleGroupGenotype.hh"
#include "starling_common/OrthogonalVariantAlleleCandidateGroupUtil.hh"
#include "starling_common/starling_read.hh"
#include "starling_common/starling_read_align_score_indels.hh"

#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

namespace
{
template <typename Tag, typename Tag::type M> struct MemberPtrOfG
{
    friend typename Tag::type memberPtr(Tag) { return M; }
};
struct GermlineErrorRatesTag
{
    typedef IndelErrorRates IndelSampleData::*type;
    friend type memberPtr(GermlineErrorRatesTag);
};
template struct MemberPtrOfG<GermlineErrorRatesTag, &IndelSampleData::_errorRates>;

/// starling_base_options of one germline sample
struct germline_options final : public starling_base_options
{
    const AlignmentFileOptions& getAlignmentFileOptions() const override
    {
        static AlignmentFileOptions alignFileOpt;
        if (alignFileOpt.alignmentFilenames.empty()) alignFileOpt.alignmentFilenames.push_back("sample.bam");
        return alignFileOpt;
    }
};

IndelKey gkey_of(const sx_indel_key& k, const char* pool, const uint32_t* off, const uint32_t i)
{
    const std::string ins(pool + off[i], pool + off[i + 1]);
    if (ins.size() != k.ins_len) throw blt_exception("ref_germline_indel: insert sequence length does not match ins_len");
    return IndelKey(k.pos, (k.type == SX_INDEL_TYPE_MISMATCH) ? INDEL::MISMATCH : INDEL::INDEL, k.del_len, ins.c_str());
}

void gcal_of(const sx_score_indels_batch* b, const uint32_t a, const bool fwd, const std::vector<IndelKey>& winKeys, CandidateAlignment& cal)
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
        default: throw blt_exception("ref_germline_indel: segment kind outside score_indels' domain");
        }
        cal.al.path.push_back(ALIGNPATH::path_segment(t, sg.len));
    }
    indel_set_t iset;
    for (uint32_t i = b->aln_key_off[a]; i < b->aln_key_off[a + 1]; ++i) iset.insert(winKeys.at(b->aln_keys[i]));
    cal.setIndels(iset);
}
} // namespace

struct ref_germline_sample // the sample: its K6 batch, K1's scores, the insert sequences behind its window entries, its read ids
{
    const sx_score_indels_batch* b;
    const double* lnp;
    const char* ins_pool;
    const uint32_t* ins_off;
    const uint32_t* read_id;
};

struct ref_germline_reads // per group: the supporting read ids and getAlleleLogLhoodFromRead of each on the extended group
{
    uint32_t* read_off;  // [n_groups + 1]
    uint32_t* read_id;   // ascending within a group (std::set order)
    uint32_t* lnp_off;   // [n_groups + 1] a read holds 1 + A + C doubles
    double* ext_lnp;
    uint16_t* read_length; // the exemplar ReadPathScores' fields
    uint16_t* non_ambig;
    uint8_t* is_fwd;
    uint32_t cap_reads, cap_lnp;
};

// gid_key / gid_ins_*: every IndelKey of the batch by id (the buffer is filled from these).  out[g]: the genotype likelihoods and read stats.
extern "C" int ref_germline_indel_chain(const sx_params* p, const ref_germline_sample* sample, const sx_indel_key* gid_key, const char* gid_ins_pool,
                                        const uint32_t* gid_ins_off, uint32_t n_gid, const sx_allele_groups* groups, sx_indel_result* out, ref_germline_reads* rd,
                                        char* err, int errlen)
{
    try
    {
        germline_options opt;
        opt.is_candidate_indel_signal_test = false;
        opt.randomBaseMatchProb = p->randomBaseMatchProb;
        {
            char buf[64];
            snprintf(buf, sizeof(buf), "%.17g", p->readConfidentSupportThreshold);
            opt.readConfidentSupportThreshold.update(buf);
        }
        const sx_score_indels_batch* b(sample->b);
        const sx_score_indels_opts& so(b->opts);
        opt.default_min_read_bp_flank = so.min_read_bp_flank;
        if (p->min_read_bp_flank != so.min_read_bp_flank) throw blt_exception("ref_germline_indel: the K6 batch's flank differs from the caller's sample options");
        opt.maxIndelSize = so.max_indel_size;
        opt.upstream_oligo_size = so.upstream_oligo_size;
        opt.is_smoothed_alignments = (so.is_smoothed_alignments != 0);
        opt.smoothed_lnp_range = so.smoothed_lnp_range;
        const starling_base_deriv_options dopt(opt);
        const starling_sample_options sample_opt(opt);
        const auto errorRatesPtr(memberPtr(GermlineErrorRatesTag()));

        // ---- one buffer over every key
        std::vector<IndelKey> keyOfGid;
        std::map<IndelKey, uint32_t> gidOfKey;
        int32_t lo(n_gid ? gid_key[0].pos : 0), hi(lo + 1);
        for (uint32_t g = 0; g < n_gid; ++g)
        {
            keyOfGid.push_back(gkey_of(gid_key[g], gid_ins_pool, gid_ins_off, g));
            if (!gidOfKey.insert(std::make_pair(keyOfGid.back(), g)).second) throw blt_exception("ref_germline_indel: two ids for one IndelKey");
            lo = std::min(lo, gid_key[g].pos);
            hi = std::max(hi, gid_key[g].pos + (int32_t)gid_key[g].del_len);
        }
        reference_contig_segment ref;
        {
            std::string seq;
            static const char cyc[4] = {'A', 'C', 'G', 'T'};
            for (int32_t q = lo - 512; q < hi + 512; ++q) seq.push_back(cyc[(q & 0x7fffffff) % 4]);
            ref.seq() = seq;
            ref.set_offset(lo - 512);
        }
        IndelBuffer indelBuffer(opt, dopt, ref);
        depth_buffer db, db2;
        indelBuffer.registerSample(db, db2, false);
        indelBuffer.finalizeSamples();
        for (uint32_t g = 0; g < n_gid; ++g)
        {
            IndelObservation obs;
            obs.key = keyOfGid[g];
            obs.data.id = 1000000 + g;
            obs.data.iat = INDEL_ALIGN_TYPE::GENOME_TIER1_READ;
            indelBuffer.addIndelObservation(0, obs);
        }
        for (uint32_t k = 0; k < b->n_keys; ++k)
        {
            IndelData* idp(indelBuffer.getIndelDataPtr(gkey_of(b->keys[k], sample->ins_pool, sample->ins_off, k)));
            if (idp == nullptr) throw blt_exception("ref_germline_indel: a window entry is no key of the batch");
            const bool cand((b->keys[k].flags & SX_IKF_CANDIDATE) != 0);
            if (idp->status.is_candidate_indel_cached && idp->status.is_candidate_indel != cand) throw blt_exception("ref_germline_indel: candidacy differs between windows");
            idp->status.is_candidate_indel = cand;
            idp->status.is_candidate_indel_cached = true;
            IndelErrorRates& rates(idp->getSampleData(0).*errorRatesPtr);
            rates.refToIndelErrorProb.updateLogValue(b->keys[k].ref_to_indel_lnp);
            rates.indelToRefErrorProb.updateLogValue(b->keys[k].indel_to_ref_lnp);
        }
        for (uint32_t g = 0; g < n_gid; ++g)
        {
            IndelData* idp(indelBuffer.getIndelDataPtr(keyOfGid[g]));
            if (idp->status.is_candidate_indel_cached) continue;
            idp->status.is_candidate_indel = false;
            idp->status.is_candidate_indel_cached = true;
        }

        // ---- score_indels for every read
        std::vector<std::unique_ptr<bam_record>> bams;
        std::vector<std::unique_ptr<starling_read>> sreads;
        if (b->full_len || b->full_off) throw blt_exception("ref_germline_indel: only full read segments are rebuilt");
        for (uint32_t region = 0; region < b->n_regions; ++region)
        {
            std::vector<IndelKey> winKeys;
            for (uint32_t k = b->region_key_off[region]; k < b->region_key_off[region + 1]; ++k) winKeys.push_back(gkey_of(b->keys[k], sample->ins_pool, sample->ins_off, k));
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
                sreads.emplace_back(new starling_read(*br, al, (b->read_flags[r] & SX_SIF_TIER1) ? MAPLEVEL::TIER1_MAPPED : MAPLEVEL::TIER2_MAPPED, sample->read_id[r]));
                bams.push_back(std::move(br));
                const read_segment& rseg(sreads.back()->get_full_segment());
                std::set<CandidateAlignment> cals;
                std::vector<double> scores;
                for (uint32_t a = a0; a < a1; ++a)
                {
                    CandidateAlignment cal;
                    gcal_of(b, a, fwd, winKeys, cal);
                    const auto ins(cals.insert(cal));
                    if (!ins.second || std::next(ins.first) != cals.end()) throw blt_exception("ref_germline_indel: alignments are not in std::set<CandidateAlignment> order");
                    scores.push_back(sample->lnp[a]);
                }
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
                score_indels(opt, dopt, sample_opt, rseg, indelBuffer, 0, cals, (b->read_flags[r] & SX_SIF_INCOMPLETE) != 0, scores, maxScore, maxPtr);
            }
        }

        // ---- per group, the reference's functions on the buffer's own iterators
        uint32_t n_reads(0), n_lnp(0);
        for (uint32_t g = 0; g < groups->n_groups; ++g)
        {
            OrthogonalVariantAlleleCandidateGroup group, contrast;
            for (uint32_t i = groups->allele_off[g]; i < groups->allele_off[g + 1]; ++i)
                group.addVariantAllele(indelBuffer.getIndelIter(keyOfGid.at(groups->allele_gid[i])));
            for (uint32_t i = groups->contrast_off[g]; i < groups->contrast_off[g + 1]; ++i)
                contrast.addVariantAllele(indelBuffer.getIndelIter(keyOfGid.at(groups->contrast_gid[i])));
            OrthogonalVariantAlleleCandidateGroup extended(group);
            for (const auto& it : contrast.alleles) extended.alleles.push_back(it);
            std::set<unsigned> readIds;
            getAlleleGroupSupportingReadIds(0, group, readIds, true);
            rd->read_off[g] = n_reads;
            rd->lnp_off[g] = n_lnp;
            for (const unsigned readId : readIds)
            {
                std::vector<double> lhood(extended.size() + 1);
                getAlleleLogLhoodFromRead(0, extended, readId, lhood);
                if (n_reads >= rd->cap_reads || n_lnp + lhood.size() > rd->cap_lnp) throw blt_exception("ref_germline_indel: read capacity");
                const ReadPathScores* ex(nullptr);
                for (unsigned a = 0; a < group.size() && !ex; ++a)
                {
                    const auto& m(group.data(a).getSampleData(0).read_path_lnp);
                    const auto f(m.find(readId));
                    if (f != m.end()) ex = &f->second;
                }
                rd->read_id[n_reads] = readId;
                rd->read_length[n_reads] = ex->read_length;
                rd->non_ambig[n_reads] = ex->nonAmbiguousBasesInRead;
                rd->is_fwd[n_reads] = ex->is_fwd_strand ? 1 : 0;
                ++n_reads;
                for (const double x : lhood) rd->ext_lnp[n_lnp++] = x;
            }
            std::vector<double> gl;
            LocusSupportingReadStats stats;
            getVariantAlleleGroupGenotypeLhoodsForSample(opt, dopt, sample_opt, groups->ploidy[g], 0, group, contrast, gl, stats);
            sx_indel_result& o(out[g]);
            std::memset(&o, 0, sizeof(o));
            o.n_gt = gl.size();
            for (size_t k = 0; k < gl.size() && k < SX_INDEL_MAX_GT; ++k) o.gt_lhood[k] = gl[k];
            for (int s = 0; s < 2; ++s)
            {
                const SupportingReadCountGroup& c(stats.getCounts(s == 1));
                for (unsigned a = 0; a <= group.size(); ++a) o.support[s][a] = c.confidentAlleleCount(a);
                o.support[s][SX_INDEL_MAX_ALLELES + 1] = c.nonConfidentCount;
            }
        }
        rd->read_off[groups->n_groups] = n_reads;
        rd->lnp_off[groups->n_groups] = n_lnp;
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
