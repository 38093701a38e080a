// allele_groups_oracle.cpp -- TEST INFRASTRUCTURE.  Scalar restatement of K6g allele_groups (include/strelka_b200.h) in the reference's shape:
// one IndelBuffer-like std::map<id, std::map<read id, ReadPathScores-like>> for the sample, filled record by record the way score_indels writes
// read_path_lnp[readId] (starling_read_align_score_indels.cpp:1071), then per group the reference's own steps: the supporting reads by a
// std::map<unsigned,unsigned> count into a std::set (getAlleleGroupIntersectionReadIds, OrthogonalVariantAlleleCandidateGroupUtil.cpp:60-107),
// getAlleleLogLhoodFromRead on the extended group in doubles (:132-196), the contrast fold and the exemplar entry (AlleleGroupGenotype.cpp:
// 160-180, 216-242).  Shares no code with strelka_b200/csrc/k6g_core.cuh.
#include "../include/strelka_b200.h"

#include <algorithm>
#include <map>
#include <set>
#include <vector>

namespace
{
struct PathScores // ReadPathScores (IndelData.hh:64-125) as the genotyper sees it
{
    float ref, indel;
    uint16_t nonAmbiguousBasesInRead, read_length;
    bool is_tier1_read, is_fwd_strand;
};
struct SampleData
{
    std::map<unsigned, PathScores> read_path_lnp;
    bool overwritten = false;
};
} // namespace

extern "C" int ox_link_allele_groups(const sx_indel_reads_sample* s, const sx_allele_groups* G, sx_allele_group_reads_out* out)
{
    const uint32_t n_groups(G->n_groups);
    std::map<uint32_t, SampleData> buffer;
    for (uint32_t g = 0; g < n_groups; ++g)
    {
        if (G->allele_off[0] != 0 || G->contrast_off[0] != 0 || G->allele_off[g + 1] < G->allele_off[g] || G->contrast_off[g + 1] < G->contrast_off[g])
            return SX_ERR_ARG;
        const uint32_t A(G->allele_off[g + 1] - G->allele_off[g]);
        if (A < 1 || A > SX_INDEL_MAX_ALLELES || (G->ploidy[g] != 1 && G->ploidy[g] != 2)) return SX_ERR_ARG;
        for (uint32_t i = G->allele_off[g]; i < G->allele_off[g + 1]; ++i)
        {
            if (G->allele_gid[i] >= G->n_gid) return SX_ERR_ARG;
            buffer[G->allele_gid[i]];
        }
        for (uint32_t i = G->contrast_off[g]; i < G->contrast_off[g + 1]; ++i)
        {
            if (G->contrast_gid[i] >= G->n_gid) return SX_ERR_ARG;
            buffer[G->contrast_gid[i]];
        }
    }
    if (n_groups == 0)
    {
        out->totals[0] = out->totals[1] = out->read_off[0] = out->lnp_off[0] = out->allele_off[0] = 0;
        return SX_OK;
    }
    for (uint32_t g = 0; g < s->n_regions; ++g)
    {
        const uint32_t k0(s->region_key_off[g]), n_win(s->region_key_off[g + 1] - k0);
        for (uint32_t r = s->region_read_off[g]; r < s->region_read_off[g + 1]; ++r)
        {
            const unsigned readId(s->read_id ? s->read_id[r] : r);
            for (uint32_t i = s->rec_off[r]; i < s->rec_off[r] + s->n_rec[r]; ++i)
            {
                const sx_read_indel_score& rec(s->recs[i]);
                if (!(rec.flags & SX_RIS_SCORED)) continue;
                if (rec.key >= n_win || s->key_gid[k0 + rec.key] >= G->n_gid) return SX_ERR_ARG;
                const auto it(buffer.find(s->key_gid[k0 + rec.key]));
                if (it == buffer.end()) continue;
                SampleData& sd(it->second);
                if (sd.read_path_lnp.count(readId)) sd.overwritten = true;
                sd.read_path_lnp[readId] = PathScores{rec.ref_lnp, rec.indel_lnp, s->non_ambig[r], s->read_len[r], (s->read_flags[r] & SX_SIF_TIER1) != 0,
                                                      (s->read_flags[r] & SX_SIF_FWD) != 0};
            }
        }
    }
    // per group: the supporting reads in std::set order, each with its A+1 values and exemplar entry
    struct Supporting
    {
        std::vector<float> lnp;
        const PathScores* exemplar;
    };
    std::vector<std::vector<Supporting>> reads(n_groups);
    uint32_t n_reads(0), n_lnp(0);
    for (uint32_t g = 0; g < n_groups; ++g)
    {
        std::vector<const SampleData*> group, extended;
        for (uint32_t i = G->allele_off[g]; i < G->allele_off[g + 1]; ++i) group.push_back(&buffer[G->allele_gid[i]]);
        extended = group;
        for (uint32_t i = G->contrast_off[g]; i < G->contrast_off[g + 1]; ++i) extended.push_back(&buffer[G->contrast_gid[i]]);
        bool overwritten(false);
        for (const SampleData* sd : extended) overwritten |= sd->overwritten;
        out->status[g] = overwritten ? SX_INDEL_READS_ST_DUP_READ : 0u;
        out->read_off[g] = n_reads;
        out->lnp_off[g] = n_lnp;
        out->allele_off[g] = G->allele_off[g];
        if (overwritten) continue;
        const unsigned nonrefAlleleCount(group.size());
        std::map<unsigned, unsigned> countReadIds;
        for (const SampleData* sd : group)
            for (const auto& score : sd->read_path_lnp)
            {
                if (!score.second.is_tier1_read) continue;
                ++countReadIds[score.first];
            }
        std::set<unsigned> readIds;
        for (const auto& value : countReadIds)
            if (value.second >= nonrefAlleleCount) readIds.insert(value.first);
        for (const unsigned readId : readIds)
        {
            // getAlleleLogLhoodFromRead on the extended group
            std::vector<double> alleleLogLhood(extended.size() + 1);
            bool isZeroAlleleCoverage(true), isPartialAlleleCoverage(false);
            for (unsigned a = 0; a < extended.size(); ++a)
            {
                const auto it(extended[a]->read_path_lnp.find(readId));
                if (it == extended[a]->read_path_lnp.end())
                {
                    isPartialAlleleCoverage = true;
                    continue;
                }
                alleleLogLhood[0] = isZeroAlleleCoverage ? static_cast<double>(it->second.ref) : std::max(alleleLogLhood[0], static_cast<double>(it->second.ref));
                alleleLogLhood[a + 1] = it->second.indel;
                isZeroAlleleCoverage = false;
            }
            if (isPartialAlleleCoverage)
                for (unsigned a = 0; a < extended.size(); ++a)
                    if (!extended[a]->read_path_lnp.count(readId)) alleleLogLhood[a + 1] = alleleLogLhood[0];
            // the contrast fold
            for (unsigned a = nonrefAlleleCount + 1; a < extended.size() + 1; ++a)
                if (alleleLogLhood[a] > alleleLogLhood[0]) alleleLogLhood[0] = alleleLogLhood[a];
            alleleLogLhood.resize(nonrefAlleleCount + 1);
            const PathScores* exemplar(nullptr);
            for (const SampleData* sd : group)
            {
                const auto it(sd->read_path_lnp.find(readId));
                if (it != sd->read_path_lnp.end())
                {
                    exemplar = &it->second;
                    break;
                }
            }
            Supporting sup{std::vector<float>(alleleLogLhood.begin(), alleleLogLhood.end()), exemplar};
            reads[g].push_back(sup);
        }
        n_reads += reads[g].size();
        n_lnp += reads[g].size() * (nonrefAlleleCount + 1);
    }
    out->read_off[n_groups] = out->totals[0] = n_reads;
    out->lnp_off[n_groups] = out->totals[1] = n_lnp;
    out->allele_off[n_groups] = G->allele_off[n_groups];
    if (n_reads > out->cap_reads || n_lnp > out->cap_lnp) return SX_ERR_CAPACITY;
    for (uint32_t g = 0; g < n_groups; ++g)
    {
        out->ploidy[g] = G->ploidy[g];
        for (uint32_t i = G->allele_off[g]; i < G->allele_off[g + 1]; ++i)
        {
            out->allele_del_len[i] = G->gid_key[G->allele_gid[i]].del_len;
            out->allele_ins_len[i] = G->gid_key[G->allele_gid[i]].ins_len;
        }
        float* lnp(out->allele_lnp + out->lnp_off[g]);
        uint32_t at(out->read_off[g]);
        for (const Supporting& sup : reads[g])
        {
            for (const float x : sup.lnp) *lnp++ = x;
            out->read_length[at] = sup.exemplar->read_length;
            out->non_ambig[at] = sup.exemplar->nonAmbiguousBasesInRead;
            out->is_fwd[at] = sup.exemplar->is_fwd_strand ? 1 : 0;
            ++at;
        }
    }
    return SX_OK;
}
