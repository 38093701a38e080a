// k6g_core.cuh -- the body of K6g allele_groups (include/strelka_b200.h, "K6g allele_groups"): one sample's K6 sx_read_indel_score records
// regrouped into K5's per-group supporting-read lists and allele log-likelihoods.
//
// The reference reads the IndelBuffer's read_path_lnp maps per group (getAlleleGroupSupportingReadIds, getAlleleLogLhoodFromRead,
// OrthogonalVariantAlleleCandidateGroupUtil.cpp:64-196, and the contrast fold of AlleleGroupGenotype.cpp:216-242).  Here those maps are
// per-id lists sorted by read id -- built with K6b's record walk, key -> id translation and sort (k6b_core.cuh) -- and a group's lookups
// are binary searches in them.  Everything that decides a byte of the output is in this header, __host__ __device__, so that
// tests/cpp/k6g_core_host.cpp runs exactly this code on the CPU; k6g_allele_groups.cu adds only the kernels' index arithmetic.
#pragma once

#include "k6b_core.cuh"

// The view of K6b's record walk for one sample: the "loci" are the ids some group names (list_of[id] = id, K6B_NONE elsewhere).
K6B_HD k6b_view k6g_view(const sx_indel_reads_sample& s, const uint32_t n_gid, const uint32_t* list_of)
{
    k6b_view v;
    v.s[0] = s;
    v.s[1] = sx_indel_reads_sample{};
    v.loci = sx_indel_loci{};
    v.loci.n_gid = n_gid;
    v.locus_of = list_of;
    return v;
}

// Group g is in K5's domain and names only ids below n_gid, and its offsets ascend from 0.
K6B_HD bool k6g_group_ok(const sx_allele_groups& G, const uint32_t g)
{
    if (g == 0 && (G.allele_off[0] != 0 || G.contrast_off[0] != 0)) return false;
    const uint32_t a0(G.allele_off[g]), a1(G.allele_off[g + 1]), c0(G.contrast_off[g]), c1(G.contrast_off[g + 1]);
    if (a1 < a0 || a1 - a0 < 1 || a1 - a0 > SX_INDEL_MAX_ALLELES || c1 < c0) return false;
    if (G.ploidy[g] != 1 && G.ploidy[g] != 2) return false;
    for (uint32_t i = a0; i < a1; ++i)
        if (G.allele_gid[i] >= G.n_gid) return false;
    for (uint32_t i = c0; i < c1; ++i)
        if (G.contrast_gid[i] >= G.n_gid) return false;
    return true;
}

// The per-id lists: id x's entries are positions off[x] .. off[x+1) of `id` (read ids, ascending); the entry at position p came from scatter
// slot off[x] + order[p], whose record and read are rec[] and read[] there.
struct k6g_lists
{
    const uint32_t* off;   // [n_gid + 1]
    const uint32_t* id;    // sorted read ids
    const uint32_t* order; // position -> scatter slot, relative to the list's start
    const uint32_t* rec;   // scatter slot -> record index in the sample's recs
    const uint32_t* read;  // scatter slot -> read index in the sample
};

// position of read id q in id x's list, K6B_NONE when it has no entry there
K6B_HD uint32_t k6g_find(const k6g_lists& L, const uint32_t x, const uint32_t q)
{
    uint32_t lo(L.off[x]), hi(L.off[x + 1]);
    while (lo < hi)
    {
        const uint32_t mid(lo + (hi - lo) / 2);
        if (L.id[mid] < q) lo = mid + 1;
        else hi = mid;
    }
    return (lo < L.off[x + 1] && L.id[lo] == q) ? lo : K6B_NONE;
}

K6B_HD uint32_t k6g_slot(const k6g_lists& L, const uint32_t x, const uint32_t p) { return L.off[x] + L.order[p]; }

// The entry at position p of the group's first allele's list (x0) supports the group: a tier-1 read with an entry in every allele.
K6B_HD bool k6g_supports(const sx_indel_reads_sample& s, const k6g_lists& L, const uint32_t* agid, const uint32_t A, const uint32_t p)
{
    if (!(s.read_flags[L.read[k6g_slot(L, agid[0], p)]] & SX_SIF_TIER1)) return false;
    for (uint32_t a = 1; a < A; ++a)
        if (k6g_find(L, agid[a], L.id[p]) == K6B_NONE) return false;
    return true;
}

// std::max(a, b) of the reference: b only when a < b
K6B_HD float k6g_max(const float a, const float b) { return (a < b) ? b : a; }

// getAlleleLogLhoodFromRead on the extended group (alleles, then contrasts) and the contrast fold, for supporting read id q: lnp[0 .. A]
K6B_HD void k6g_allele_lnp(const sx_indel_reads_sample& s, const k6g_lists& L, const uint32_t* agid, const uint32_t A, const uint32_t* cgid, const uint32_t C,
                           const uint32_t q, float* lnp)
{
    float l0(0.f);
    for (uint32_t a = 0; a < A; ++a) // (every one holds the read: it supports the group)
    {
        const sx_read_indel_score& rec(s.recs[L.rec[k6g_slot(L, agid[a], k6g_find(L, agid[a], q))]]);
        l0 = a == 0 ? rec.ref_lnp : k6g_max(l0, rec.ref_lnp);
        lnp[1 + a] = rec.indel_lnp;
    }
    for (uint32_t c = 0; c < C; ++c)
    {
        const uint32_t p(k6g_find(L, cgid[c], q));
        if (p != K6B_NONE) l0 = k6g_max(l0, s.recs[L.rec[k6g_slot(L, cgid[c], p)]].ref_lnp);
    }
    const float uncovered(l0); // a contrast allele without an entry takes L[0] as the first step left it
    for (uint32_t c = 0; c < C; ++c)
    {
        const uint32_t p(k6g_find(L, cgid[c], q));
        const float v(p != K6B_NONE ? s.recs[L.rec[k6g_slot(L, cgid[c], p)]].indel_lnp : uncovered);
        if (v > l0) l0 = v;
    }
    lnp[0] = l0;
}
