// indel_reads_oracle.cpp -- TEST INFRASTRUCTURE.  Scalar restatement of K6b indel_reads (include/strelka_b200.h) in the reference's shape:
// one IndelBuffer-like std::map<id, IndelData-like>, each entry holding two std::map<read id, ReadPathScores-like>, filled record by
// record the way score_indels writes read_path_lnp[readId] (starling_read_align_score_indels.cpp:1071) and then walked in key order the
// way process_pos_indel_somatic does (strelka_pos_processor.cpp:297-348).  Shares no code with strelka_b200/csrc/k6b_core.cuh.
#include "../include/strelka_b200.h"

#include <cstring>
#include <map>
#include <set>
#include <utility>
#include <vector>

namespace
{
struct PathScores // ReadPathScores (IndelData.hh:64-125) as the link sees it
{
    float ref, indel;
    uint16_t nonAmbiguousBasesInRead, read_length;
    bool is_tier1_read;
    std::vector<std::pair<uint32_t, float>> alt_indel; // (id, lnp) in insertAlt's order
};
struct SampleData
{
    std::map<uint32_t, PathScores> read_path_lnp;
    bool overwritten = false;
};
struct Data
{
    SampleData sample[2];
};
} // namespace

extern "C" int ox_link_indel_reads(const sx_indel_reads_sample* normal, const sx_indel_reads_sample* tumor, const sx_indel_loci* loci, sx_indel_reads_out* out)
{
    std::map<uint32_t, Data> buffer;
    for (uint32_t l = 0; l < loci->n_loci; ++l)
    {
        if (loci->gid[l] >= loci->n_gid || (l && loci->gid[l] <= loci->gid[l - 1])) return SX_ERR_ARG;
        buffer[loci->gid[l]];
    }
    const sx_indel_reads_sample* samples[2] = {normal, tumor};
    for (unsigned sampleIndex = 0; sampleIndex < 2; ++sampleIndex)
    {
        const sx_indel_reads_sample& s(*samples[sampleIndex]);
        for (uint32_t g = 0; g < s.n_regions; ++g)
        {
            const uint32_t k0(s.region_key_off[g]), n_win(s.region_key_off[g + 1] - k0);
            for (uint32_t r = s.region_read_off[g]; r < s.region_read_off[g + 1]; ++r)
            {
                const uint32_t readId(s.read_id ? s.read_id[r] : r);
                for (uint32_t i = s.rec_off[r]; i < s.rec_off[r] + s.n_rec[r]; ++i)
                {
                    const sx_read_indel_score& rec(s.recs[i]);
                    if (!(rec.flags & SX_RIS_SCORED)) continue;
                    if (rec.key >= n_win || s.key_gid[k0 + rec.key] >= loci->n_gid) return SX_ERR_ARG;
                    const auto it(buffer.find(s.key_gid[k0 + rec.key]));
                    if (it == buffer.end()) continue;
                    PathScores ps = {rec.ref_lnp, rec.indel_lnp, s.non_ambig[r], s.read_len[r], (s.read_flags[r] & SX_SIF_TIER1) != 0, {}};
                    for (unsigned a = 0; a < rec.n_alt && a < 2; ++a)
                    {
                        if (rec.alt_key[a] >= n_win || s.key_gid[k0 + rec.alt_key[a]] >= loci->n_gid) return SX_ERR_ARG;
                        ps.alt_indel.push_back(std::make_pair(s.key_gid[k0 + rec.alt_key[a]], rec.alt_lnp[a]));
                    }
                    SampleData& sd(it->second.sample[sampleIndex]);
                    if (sd.read_path_lnp.count(readId)) sd.overwritten = true;
                    sd.read_path_lnp[readId] = ps;
                }
            }
        }
    }
    // sizes first: a capacity that is too small leaves everything but the entries and the table rows written
    uint32_t n_entries(0), n_alts(0), l(0);
    std::vector<std::vector<uint32_t>> tables(loci->n_loci);
    for (const auto& val : buffer)
    {
        const Data& d(val.second);
        std::set<uint32_t> named;
        for (const SampleData& sd : d.sample)
            for (const auto& rv : sd.read_path_lnp)
                for (const auto& alt : rv.second.alt_indel) named.insert(alt.first);
        uint32_t st(0);
        if (d.sample[0].overwritten || d.sample[1].overwritten) st |= SX_INDEL_READS_ST_DUP_READ;
        if (named.size() > SX_SINDEL_MAX_ALTS) st |= SX_SINDEL_ST_CAP;
        out->status[l] = st;
        out->alt_off[l] = n_alts;
        for (unsigned sampleIndex = 0; sampleIndex < 2; ++sampleIndex)
        {
            out->read_off[2 * l + sampleIndex] = n_entries;
            if (!st) n_entries += d.sample[sampleIndex].read_path_lnp.size();
        }
        if (!st)
        {
            tables[l].assign(named.begin(), named.end());
            n_alts += named.size();
        }
        ++l;
    }
    out->alt_off[loci->n_loci] = out->totals[1] = n_alts;
    out->read_off[2 * loci->n_loci] = out->totals[0] = n_entries;
    if (n_entries > out->cap_reads || n_alts > out->cap_alts) return SX_ERR_CAPACITY;
    l = 0;
    for (const auto& val : buffer)
    {
        if (!out->status[l])
        {
            const std::vector<uint32_t>& table(tables[l]);
            for (size_t a = 0; a < table.size(); ++a) out->alts[out->alt_off[l] + a] = loci->gid_key[table[a]];
            for (unsigned sampleIndex = 0; sampleIndex < 2; ++sampleIndex)
            {
                sx_sindel_read* e(out->reads + out->read_off[2 * l + sampleIndex]);
                for (const auto& rv : val.second.sample[sampleIndex].read_path_lnp)
                {
                    const PathScores& ps(rv.second);
                    std::memset(e, 0, sizeof(*e));
                    e->ref = ps.ref;
                    e->indel = ps.indel;
                    e->read_length = ps.read_length;
                    e->non_ambig = ps.nonAmbiguousBasesInRead;
                    e->is_tier1 = ps.is_tier1_read;
                    e->n_alt = ps.alt_indel.size();
                    for (size_t a = 0; a < ps.alt_indel.size(); ++a)
                    {
                        size_t at(0);
                        while (table[at] != ps.alt_indel[a].first) ++at;
                        e->alt[a] = at;
                        e->alt_lnp[a] = ps.alt_indel[a].second;
                    }
                    ++e;
                }
            }
        }
        ++l;
    }
    return SX_OK;
}
