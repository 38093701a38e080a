// tests/cpp/k6g_core_host.cpp -- TEST ONLY.  Compiles the body of K6g (strelka_b200/csrc/k6g_core.cuh, __host__ __device__) with g++ and
// runs it the way the kernels of k6g_allele_groups.cu do: mark, the list builder (k6_lists_host.h: count, scan, backwards scatter, sort at
// depth `smem_sort`), group count, scan, write.
#include "k6_lists_host.h"
#include "k6g_core.cuh"

extern "C" int k6gcore_run(const sx_indel_reads_sample* sample, const sx_allele_groups* G, sx_allele_group_reads_out* o, uint32_t smem_sort)
{
    const uint32_t n_gid(G->n_gid), n_groups(G->n_groups);
    std::vector<uint32_t> list_of(n_gid, K6B_NONE);
    for (uint32_t g = 0; g < n_groups; ++g)
    {
        if (!k6g_group_ok(*G, g)) return SX_ERR_ARG;
        for (uint32_t i = G->allele_off[g]; i < G->allele_off[g + 1]; ++i) list_of[G->allele_gid[i]] = G->allele_gid[i];
        for (uint32_t i = G->contrast_off[g]; i < G->contrast_off[g + 1]; ++i) list_of[G->contrast_gid[i]] = G->contrast_gid[i];
    }
    if (n_groups == 0)
    {
        o->totals[0] = o->totals[1] = o->read_off[0] = o->lnp_off[0] = o->allele_off[0] = 0;
        return SX_OK;
    }
    const k6b_view v(k6g_view(*sample, n_gid, list_of.data()));
    k6l_host_lists lists;
    if (k6l_host_build(v, 1, n_gid, smem_sort, lists)) return SX_ERR_ARG;
    const k6g_lists L{lists.off.data(), lists.id.data(), lists.order.data(), lists.rec.data(), lists.read.data()};
    uint32_t n_reads(0), n_lnp(0);
    for (uint32_t g = 0; g < n_groups; ++g)
    {
        const uint32_t a0(G->allele_off[g]), A(G->allele_off[g + 1] - a0);
        const uint32_t* agid(G->allele_gid + a0);
        bool d(false);
        for (uint32_t i = a0; i < a0 + A; ++i) d |= lists.dup[G->allele_gid[i]] != 0;
        for (uint32_t i = G->contrast_off[g]; i < G->contrast_off[g + 1]; ++i) d |= lists.dup[G->contrast_gid[i]] != 0;
        uint32_t n(0);
        if (!d)
            for (uint32_t p = L.off[agid[0]]; p < L.off[agid[0] + 1]; ++p) n += k6g_supports(*sample, L, agid, A, p) ? 1u : 0u;
        o->status[g] = d ? SX_INDEL_READS_ST_DUP_READ : 0u;
        o->read_off[g] = n_reads;
        o->lnp_off[g] = n_lnp;
        o->allele_off[g] = a0;
        n_reads += n;
        n_lnp += n * (A + 1);
    }
    o->read_off[n_groups] = o->totals[0] = n_reads;
    o->lnp_off[n_groups] = o->totals[1] = n_lnp;
    o->allele_off[n_groups] = G->allele_off[n_groups];
    if (n_reads > o->cap_reads || n_lnp > o->cap_lnp) return SX_ERR_CAPACITY;
    for (uint32_t g = 0; g < n_groups; ++g)
    {
        const uint32_t a0(G->allele_off[g]), A(G->allele_off[g + 1] - a0);
        const uint32_t *agid(G->allele_gid + a0), *cgid(G->contrast_gid + G->contrast_off[g]), C(G->contrast_off[g + 1] - G->contrast_off[g]);
        o->ploidy[g] = G->ploidy[g];
        for (uint32_t a = 0; a < A; ++a)
        {
            o->allele_del_len[a0 + a] = G->gid_key[agid[a]].del_len;
            o->allele_ins_len[a0 + a] = G->gid_key[agid[a]].ins_len;
        }
        if (o->status[g]) continue;
        uint32_t at(o->read_off[g]);
        for (uint32_t p = L.off[agid[0]]; p < L.off[agid[0] + 1]; ++p)
        {
            if (!k6g_supports(*sample, L, agid, A, p)) continue;
            float lnp[SX_INDEL_MAX_ALLELES + 1];
            k6g_allele_lnp(*sample, L, agid, A, cgid, C, L.id[p], lnp);
            for (uint32_t a = 0; a <= A; ++a) o->allele_lnp[o->lnp_off[g] + (at - o->read_off[g]) * (A + 1) + a] = lnp[a];
            const uint32_t r(L.read[k6g_slot(L, agid[0], p)]);
            o->read_length[at] = sample->read_len[r];
            o->non_ambig[at] = sample->non_ambig[r];
            o->is_fwd[at] = (sample->read_flags[r] & SX_SIF_FWD) ? 1 : 0;
            ++at;
        }
    }
    return SX_OK;
}
