// ref_harness_pileup_metrics.cpp -- TEST INFRASTRUCTURE ONLY.
//
// Drives the UNMODIFIED reference's starling_pos_processor_base::pileup_read_segment (starling_pos_processor_base.cpp:1127-1421) for every
// read of a flattened sx_pileup_reads_batch with the scoring metrics switched on, and reads each position's snp_pos_info back through the
// reference's own accessors -- the K4m answers (include/strelka_b200.h) as the reference computes them:
//   SX_PM_MAPQ      no metrics option: only insert_mapq_count runs ("always"), sample 0
//   SX_PM_GERMLINE  an options subclass whose is_compute_germline_scoring_metrics() is true (as starling_options), sample 0
//   SX_PM_SOMATIC   is_compute_somatic_scoring_metrics = true (as strelka_options) on a two-sample processor, the reads piled into sample 1
// and then MapqTracker, fastRanksum::get_z_stat / getExpectedCategory2Value, MeanTracker::mean and the medians of
// position_somatic_snv_strand_grid_vcf.cpp:159-189 (math_util.hh median).  pileup_read_segment is private: it is reached through the
// explicit-instantiation idiom, as in ref_harness.cpp.  Linked into oracle/_ref/libstrelka_ref_pileup_metrics.so by
// build_ref_pileup_metrics.sh.
#include "../include/strelka_b200.h"

#include "appstats/RunStatsManager.hh"
#include "blt_util/align_path.hh"
#include "blt_util/blt_exception.hh"
#include "blt_util/math_util.hh"
#include "htsapi/align_path_bam_util.hh"
#include "htsapi/bam_record.hh"
#include "starling_common/starling_pos_processor_base.hh"
#include "starling_common/starling_read.hh"
#include "starling_common/starling_streams_base.hh"

#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

namespace
{
struct metrics_options final : public starling_base_options
{
    const AlignmentFileOptions& getAlignmentFileOptions() const override
    {
        static AlignmentFileOptions alignFileOpt;
        if (alignFileOpt.alignmentFilenames.size() < 2)
        {
            alignFileOpt.alignmentFilenames.clear();
            alignFileOpt.alignmentFilenames.push_back("normal.bam");
            alignFileOpt.alignmentFilenames.push_back("tumor.bam");
        }
        return alignFileOpt;
    }
    bool is_compute_germline_scoring_metrics() const override { return germline; }
    bool germline = false;
};

struct MetricsPosProcessor : public starling_pos_processor_base
{
    using starling_pos_processor_base::starling_pos_processor_base;
    void process_pos_variants_impl(const pos_t, const bool) override {}
    void resetRegionForTest(const std::string& chrom, const known_pos_range2& range) { resetRegionBase(chrom, range); }
    CandidateSnvBuffer& snvBuffer() { return getCandidateSnvBuffer(); }
};

template <typename Tag, typename Tag::type M> struct MemberPtrOf
{
    friend typename Tag::type memberPtr(Tag) { return M; }
};
struct PileupTag
{
    typedef void (starling_pos_processor_base::*type)(const read_segment&, const unsigned);
    friend type memberPtr(PileupTag);
};
template struct MemberPtrOf<PileupTag, &starling_pos_processor_base::pileup_read_segment>;

void set_err(char* err, int errlen, const char* msg)
{
    if (err && errlen > 0)
    {
        std::strncpy(err, msg, errlen - 1);
        err[errlen - 1] = 0;
    }
}
} // namespace

extern "C" int ref_pileup_metrics(const sx_pileup_reads_batch* b, uint32_t mode, sx_pileup_metrics_rec* out, char* err, int errlen)
{
    try
    {
        if (mode != SX_PM_MAPQ && mode != SX_PM_GERMLINE && mode != SX_PM_SOMATIC) throw blt_exception("ref_pileup_metrics: mode");
        metrics_options opt;
        opt.is_candidate_indel_signal_test = false;
        opt.isBasecallQualAdjustedForMapq = (b->opts.isBasecallQualAdjustedForMapq != 0);
        opt.minBasecallErrorPhredProb = b->opts.minBasecallErrorPhredProb;
        opt.mismatchDensityFilterFlankSize = b->opts.mismatchDensityFilterFlankSize;
        opt.mismatchDensityFilterMaxMismatchCount = b->opts.mismatchDensityFilterMaxMismatchCount;
        opt.useTier2Evidence = (b->opts.useTier2Evidence != 0);
        opt.tier2.mismatchDensityFilterMaxMismatchCount = b->opts.tier2MismatchDensityFilterMaxMismatchCount;
        opt.minDistanceFromReadEdge = b->opts.minDistanceFromReadEdge;
        opt.germline = mode == SX_PM_GERMLINE;
        opt.is_compute_somatic_scoring_metrics = mode == SX_PM_SOMATIC;
        const unsigned sample(mode == SX_PM_SOMATIC ? 1u : 0u);
        starling_base_deriv_options dopt(opt);
        reference_contig_segment ref;
        ref.seq() = std::string(b->ref, b->ref_len);
        ref.set_offset(b->ref_begin);
        starling_streams_base streams(2);
        RunStatsManager stats("");
        MetricsPosProcessor proc(opt, dopt, ref, streams, 2, stats);
        proc.resetRegionForTest("chrT", known_pos_range2(b->report_begin, b->report_end));
        for (uint32_t i = 0; i < b->n_cand_snv; ++i)
        {
            static const char BASE[4] = {'A', 'C', 'G', 'T'};
            proc.snvBuffer().addCandidateSnv(sample, b->report_begin + static_cast<pos_t>(b->cand_snv[i] >> 2), BASE[b->cand_snv[i] & 3], 1, 0.5f);
        }
        const auto pileup(memberPtr(PileupTag()));
        std::vector<std::unique_ptr<bam_record>> bams;
        std::vector<std::unique_ptr<starling_read>> sreads;
        for (uint32_t r = 0; r < b->n_reads; ++r)
        {
            const sx_pileup_read& rd(b->reads[r]);
            if (rd.flags & SX_PRF_SKIP) continue;
            const int len(rd.len);
            std::unique_ptr<bam_record> br(new bam_record);
            br->set_qname("R");
            const std::string dummy(len, 'A');
            std::vector<uint8_t> q(len);
            for (int i = 0; i < len; ++i) q[i] = b->qual_bits == 4 ? b->qual_dict[(b->qual[rd.qual_off + (i >> 1)] >> ((~i & 1) << 2)) & 15] : b->qual[rd.qual_off + i];
            br->set_readqual(dummy.c_str(), q.data());
            std::memcpy(bam_get_seq(br->get_data()), b->seq4 + rd.seq_off, (len + 1) / 2);
            alignment al;
            al.pos = rd.pos;
            al.is_fwd_strand = (rd.flags & SX_PRF_FWD) != 0;
            for (uint32_t s = rd.seg_off; s < b->reads[r + 1].seg_off; ++s)
            {
                const sx_aln_seg& sg(b->segs[s]);
                if (sg.len == 0 && sg.kind == SX_SEG_HARDCLIP) continue; // a pad of the window pass's slot layout
                ALIGNPATH::align_t t(ALIGNPATH::NONE);
                switch (sg.kind)
                {
                case SX_SEG_MATCH: t = ALIGNPATH::MATCH; break;
                case SX_SEG_INSERT: t = ALIGNPATH::INSERT; break;
                case SX_SEG_DELETE: t = ALIGNPATH::DELETE; break;
                case SX_SEG_SKIP: t = ALIGNPATH::SKIP; break;
                case SX_SEG_SOFTCLIP: t = ALIGNPATH::SOFT_CLIP; break;
                case SX_SEG_HARDCLIP: t = ALIGNPATH::HARD_CLIP; break;
                default: throw blt_exception("ref_pileup_metrics: unknown segment kind");
                }
                al.path.push_back(ALIGNPATH::path_segment(t, sg.len));
            }
            br->get_data()->core.pos = al.pos;
            br->get_data()->core.qual = rd.mapq;
            edit_bam_cigar(al.path, *(br->get_data()));
            const MAPLEVEL::index_t lev((rd.flags & SX_PRF_TIER1) ? MAPLEVEL::TIER1_MAPPED : (rd.flags & SX_PRF_TIER1OR2) ? MAPLEVEL::TIER2_MAPPED : MAPLEVEL::SUB_MAPPED);
            sreads.emplace_back(new starling_read(*br, al, lev, r));
            bams.push_back(std::move(br));
            (proc.*pileup)(sreads.back()->get_full_segment(), sample);
        }
        const pos_basecall_buffer& buf(proc.sample(sample).basecallBuffer);
        const uint32_t n_sites(static_cast<uint32_t>(b->report_end - b->report_begin));
        for (uint32_t i = 0; i < n_sites; ++i)
        {
            const snp_pos_info& pi(buf.get_pos(b->report_begin + static_cast<pos_t>(i)));
            sx_pileup_metrics_rec& o(out[i]);
            std::memset(&o, 0, sizeof(o));
            o.mapq_count = pi.mapqTracker.count;
            o.mapq_zero = pi.mapqTracker.zeroCount;
            o.mapq_sum_sq = pi.mapqTracker.sumSquare;
            if (mode == SX_PM_GERMLINE) // starling_pos_processor.cpp:237-244
            {
                o.read_pos_ranksum = pi.get_read_pos_ranksum();
                o.mq_ranksum = pi.get_mq_ranksum();
                o.baseq_ranksum = pi.get_baseq_ranksum();
                o.mean_edge_distance = pi.distanceFromReadEdge.mean();
                o.raw_pos = pi.get_raw_pos();
                o.raw_baseq = pi.get_raw_baseQ();
            }
            else if (mode == SX_PM_SOMATIC) // position_somatic_snv_strand_grid_vcf.cpp:159-189, 208
            {
                o.read_pos_ranksum = pi.readPositionRankSum.get_z_stat();
                const auto& apos(pi.altAlleleReadPositionInfo);
                o.n_alt_read_pos = static_cast<uint32_t>(apos.size());
                if (!apos.empty())
                {
                    std::vector<uint16_t> readpos, readposcomp;
                    for (const auto& x : apos) readpos.push_back(x.readPos);
                    for (const auto& x : apos) readposcomp.push_back(x.readLength - x.readPos);
                    const auto pmedian(median(readpos.begin(), readpos.end()));
                    const auto lmedian(median(readposcomp.begin(), readposcomp.end()));
                    o.median_read_pos = std::min(pmedian, lmedian);
                    if (readpos.size() >= 3)
                    {
                        for (auto& p : readpos) p = std::abs(p - pmedian);
                        o.median_read_pos_var = median(readpos.begin(), readpos.end());
                    }
                }
            }
        }
        return 0;
    }
    catch (const std::exception& e)
    {
        set_err(err, errlen, e.what());
        return 1;
    }
}
