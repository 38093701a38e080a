// tests/cpp/k6g_core_host.cpp -- TEST ONLY.  Compiles the body of K6g (strelka_b200/csrc/k6g_core.cuh, __host__ __device__) with g++ and
// runs it the way the kernels of k6g_allele_groups.cu do: mark, count, scan, scatter, sort, group count, scan, write.  The scatter visits the
// reads BACKWARDS, so the lists reach the sort in an order the device never produces: the output must not depend on it.  `smem_sort` is the
// depth up to which a list is sorted in a side buffer (the kernel's shared memory), beyond it in the scratch itself.
#include "k6g_core.cuh"

#include <vector>

extern "C" int k6gcore_run(const sx_indel_reads_sample* sample, const sx_allele_groups* G, sx_allele_group_reads_out* o, uint32_t smem_sort)
{
    const uint32_t n_gid(G->n_gid), n_groups(G->n_groups);
    std::vector<uint32_t> list_of(n_gid, K6B_NONE), list_off(n_gid + 1, 0), dup(n_gid, 0);
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
    uint32_t bad(0);
    for (uint32_t r = 0; r < sample->n_reads; ++r) bad |= k6b_for_each_entry(v, 0u, r, [&](uint32_t x, uint32_t) { ++list_off[x + 1]; });
    if (bad) return SX_ERR_ARG;
    for (uint32_t i = 0; i < n_gid; ++i) list_off[i + 1] += list_off[i];
    const uint32_t n_pairs(list_off[n_gid]);
    std::vector<uint32_t> cursor(list_off.begin(), list_off.end() - 1), id(n_pairs), rec(n_pairs), read(n_pairs), order(n_pairs), key, val;
    for (uint32_t r = sample->n_reads; r-- > 0;)
        k6b_for_each_entry(v, 0u, r, [&](uint32_t x, uint32_t i) {
            const uint32_t at(cursor[x]++);
            id[at] = k6b_read_id(*sample, r);
            rec[at] = i;
            read[at] = r;
        });
    for (uint32_t x = 0; x < n_gid; ++x)
    {
        const uint32_t base(list_off[x]), n(list_off[x + 1] - base);
        if (n <= smem_sort)
        {
            key.assign(id.begin() + base, id.begin() + base + n);
            val.resize(n);
            for (uint32_t i = 0; i < n; ++i) val[i] = i;
            k6b_sort_by_key(key.data(), val.data(), n, 0u, 1u, [] {});
            for (uint32_t i = 0; i < n; ++i)
            {
                id[base + i] = key[i];
                order[base + i] = val[i];
            }
        }
        else
        {
            for (uint32_t i = 0; i < n; ++i) order[base + i] = i;
            k6b_sort_by_key(id.data() + base, order.data() + base, n, 0u, 1u, [] {});
        }
        for (uint32_t i = 0; i + 1 < n; ++i) dup[x] |= id[base + i] == id[base + i + 1];
    }
    const k6g_lists L{list_off.data(), id.data(), order.data(), rec.data(), read.data()};
    uint32_t n_reads(0), n_lnp(0);
    for (uint32_t g = 0; g < n_groups; ++g)
    {
        const uint32_t a0(G->allele_off[g]), A(G->allele_off[g + 1] - a0);
        const uint32_t* agid(G->allele_gid + a0);
        bool d(false);
        for (uint32_t i = a0; i < a0 + A; ++i) d |= dup[G->allele_gid[i]] != 0;
        for (uint32_t i = G->contrast_off[g]; i < G->contrast_off[g + 1]; ++i) d |= dup[G->contrast_gid[i]] != 0;
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
