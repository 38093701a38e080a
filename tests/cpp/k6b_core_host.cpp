// tests/cpp/k6b_core_host.cpp -- TEST ONLY.  Compiles the body of K6b (strelka_b200/csrc/k6b_core.cuh, __host__ __device__) with g++ and
// runs it the way the kernels of k6b_indel_reads.cu do: table, the list builder (k6_lists_host.h: count, scan, backwards scatter, sort at
// depth `smem_sort`), the alternate sets, scan, write.
#include "k6_lists_host.h"

extern "C" int k6bcore_run(const sx_indel_reads_sample* normal, const sx_indel_reads_sample* tumor, const sx_indel_loci* loci, sx_indel_reads_out* o, uint32_t smem_sort)
{
    const uint32_t n_loci(loci->n_loci);
    std::vector<uint32_t> locus_of(loci->n_gid, K6B_NONE);
    for (uint32_t l = 0; l < n_loci; ++l)
    {
        if (loci->gid[l] >= loci->n_gid) return SX_ERR_ARG;
        locus_of[loci->gid[l]] = l;
    }
    k6b_view v;
    v.s[0] = *normal;
    v.s[1] = *tumor;
    v.loci = *loci;
    v.locus_of = locus_of.data();
    k6l_host_lists L;
    uint32_t bad(k6l_host_build(v, 2, n_loci, smem_sort, L));
    std::vector<uint32_t> alt_ids((size_t)SX_SINDEL_MAX_ALTS * n_loci, 0x7B7B7B7Bu);
    uint32_t n_entries(0), n_alts_total(0);
    for (uint32_t l = 0; l < n_loci; ++l)
    {
        uint32_t* set(alt_ids.data() + (size_t)SX_SINDEL_MAX_ALTS * l);
        uint32_t n_set(0);
        bool over(false);
        for (uint32_t sample = 0; sample < 2; ++sample)
        {
            const sx_indel_reads_sample& s(v.s[sample]);
            const uint32_t base(L.off[2 * l + sample]), n(L.off[2 * l + sample + 1] - base);
            for (uint32_t i = 0; i < n; ++i)
            {
                const sx_read_indel_score& rc(s.recs[L.rec[base + i]]);
                uint32_t ids[2];
                const uint32_t na(rc.n_alt ? k6b_alt_ids(s, loci->n_gid, k6b_region_of(s, L.read[base + i]), rc, ids, bad) : 0u);
                for (uint32_t a = 0; a < na; ++a)
                    if (ids[a] != K6B_NONE && !k6b_set_insert(set, n_set, ids[a])) over = true;
            }
        }
        const uint32_t st((L.dup[l] ? SX_INDEL_READS_ST_DUP_READ : 0u) | (over ? SX_SINDEL_ST_CAP : 0u));
        o->status[l] = st;
        o->alt_off[l] = n_alts_total;
        for (uint32_t sample = 0; sample < 2; ++sample)
        {
            o->read_off[2 * l + sample] = n_entries;
            if (!st) n_entries += L.off[2 * l + sample + 1] - L.off[2 * l + sample];
        }
        if (!st) n_alts_total += n_set;
    }
    if (bad) return SX_ERR_ARG;
    o->read_off[2 * n_loci] = o->totals[0] = n_entries;
    o->alt_off[n_loci] = o->totals[1] = n_alts_total;
    if (n_entries > o->cap_reads || n_alts_total > o->cap_alts) return SX_ERR_CAPACITY;
    for (uint32_t l = 0; l < n_loci; ++l)
    {
        if (o->status[l]) continue;
        const uint32_t* ids(alt_ids.data() + (size_t)SX_SINDEL_MAX_ALTS * l);
        const uint32_t a0(o->alt_off[l]), n_alts(o->alt_off[l + 1] - a0);
        for (uint32_t a = 0; a < n_alts; ++a) o->alts[a0 + a] = loci->gid_key[ids[a]];
        for (uint32_t sample = 0; sample < 2; ++sample)
        {
            const sx_indel_reads_sample& s(v.s[sample]);
            const uint32_t base(L.off[2 * l + sample]), n(L.off[2 * l + sample + 1] - base), out0(o->read_off[2 * l + sample]);
            for (uint32_t i = 0; i < n; ++i)
            {
                const uint32_t j(base + L.order[base + i]);
                o->reads[out0 + i] = k6b_entry(s, loci->n_gid, L.read[j], s.recs[L.rec[j]], ids, n_alts);
            }
        }
    }
    return SX_OK;
}
