// k6b_core.cuh -- the body of K6b indel_reads (include/strelka_b200.h, "K6b indel_reads"): K6's read-major sx_read_indel_score records
// regrouped into K5b's locus-major read_path_lnp lists.
//
// What the reference does implicitly -- score_indels writes read_path_lnp[readId] into the shared IndelBuffer
// (starling_read_align_score_indels.cpp:1071) and get_somatic_indel walks that std::map (somatic_indel_grid.cpp:181-361) -- is a
// count / scan / scatter / sort-by-read-id here.  Everything that decides a byte of the output is in this header, __host__ __device__,
// so that tests/cpp/k6b_core_host.cpp runs exactly this code on the CPU; k6b_indel_reads.cu adds only the kernels' index arithmetic.
#pragma once

#include "strelka_b200.h"

#include <stdint.h>

#ifdef __CUDACC__
#define K6B_HD __host__ __device__ __forceinline__
#else
#define K6B_HD inline
#endif

constexpr uint32_t K6B_NONE = 0xffffffffu;
constexpr uint32_t K6B_ST_BAD_ID = 1u; // a window index past its region's window, or an id >= n_gid

struct k6b_view
{
    sx_indel_reads_sample s[2]; // normal, tumor
    sx_indel_loci loci;
    const uint32_t* locus_of;   // [n_gid] id -> locus, K6B_NONE where the id is no listed locus
};

// the region of read r: the last g with region_read_off[g] <= r
K6B_HD uint32_t k6b_region_of(const sx_indel_reads_sample& s, const uint32_t r)
{
    uint32_t lo(0), hi(s.n_regions);
    while (hi - lo > 1)
    {
        const uint32_t mid((lo + hi) / 2);
        if (s.region_read_off[mid] <= r) lo = mid;
        else hi = mid;
    }
    return lo;
}

// window index `key` of region g as a batch-wide id; K6B_NONE (and K6B_ST_BAD_ID) when the index or the id is out of range
K6B_HD uint32_t k6b_gid_of(const sx_indel_reads_sample& s, const uint32_t n_gid, const uint32_t g, const uint32_t key, uint32_t& st)
{
    const uint32_t k0(s.region_key_off[g]), k1(s.region_key_off[g + 1]);
    if (key >= k1 - k0)
    {
        st |= K6B_ST_BAD_ID;
        return K6B_NONE;
    }
    const uint32_t id(s.key_gid[k0 + key]);
    if (id >= n_gid)
    {
        st |= K6B_ST_BAD_ID;
        return K6B_NONE;
    }
    return id;
}

K6B_HD uint32_t k6b_read_id(const sx_indel_reads_sample& s, const uint32_t r) { return s.read_id ? s.read_id[r] : r; }

// Visits the records of read r of sample `sample` that become read_path_lnp entries of a listed locus: f(locus, record index).
template <typename F> K6B_HD uint32_t k6b_for_each_entry(const k6b_view& v, const uint32_t sample, const uint32_t r, F f)
{
    const sx_indel_reads_sample& s(v.s[sample]);
    const uint32_t n(s.n_rec[r]);
    uint32_t st(0);
    if (n == 0) return st;
    const uint32_t g(k6b_region_of(s, r)), i0(s.rec_off[r]);
    for (uint32_t i = i0; i < i0 + n; ++i)
    {
        const sx_read_indel_score& rec(s.recs[i]);
        if (!(rec.flags & SX_RIS_SCORED)) continue; // suboverlap marks are not in read_path_lnp
        const uint32_t id(k6b_gid_of(s, v.loci.n_gid, g, rec.key, st));
        if (id == K6B_NONE) continue;
        const uint32_t l(v.locus_of[id]);
        if (l != K6B_NONE) f(l, i);
    }
    return st;
}

// Sorts key[0..n) ascending, val[] following, with lanes `lane` of `n_lanes` working together: the bitonic network in its one-direction
// form (each merge starts with the mirrored comparators i <-> i ^ (k - 1), then the half-cleaners i <-> i ^ j), every comparator putting
// the smaller key at the lower index.  Elements past n would be +inf and never move, so their comparators are skipped and n need not be
// a power of two.  `sync` separates the steps (__syncwarp on the device).  key/val may be shared or global memory.
template <typename Sync> K6B_HD void k6b_sort_by_key(uint32_t* key, uint32_t* val, const uint32_t n, const uint32_t lane, const uint32_t n_lanes, Sync sync)
{
    for (uint32_t k = 2; (k >> 1) < n; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1)
        {
            const uint32_t mask((j == (k >> 1)) ? k - 1 : j);
            for (uint32_t i = lane; i < n; i += n_lanes)
            {
                const uint32_t p(i ^ mask);
                if (p > i && p < n)
                {
                    const uint32_t a(key[i]), b(key[p]);
                    if (b < a)
                    {
                        key[i] = b;
                        key[p] = a;
                        const uint32_t t(val[i]);
                        val[i] = val[p];
                        val[p] = t;
                    }
                }
            }
            sync();
        }
}

// A locus's alternate ids: at most SX_SINDEL_MAX_ALTS distinct values, kept ascending.  false: the id is new and the set is full.
K6B_HD bool k6b_set_insert(uint32_t* set, uint32_t& n, const uint32_t id)
{
    uint32_t at(0);
    while (at < n && set[at] < id) ++at;
    if (at < n && set[at] == id) return true;
    if (n == SX_SINDEL_MAX_ALTS) return false;
    for (uint32_t i = n; i > at; --i) set[i] = set[i - 1];
    set[at] = id;
    ++n;
    return true;
}

// The ids record `rec` of a read of region g names as alternates: ids[0..return), in alt_indel order.
K6B_HD uint32_t k6b_alt_ids(const sx_indel_reads_sample& s, const uint32_t n_gid, const uint32_t g, const sx_read_indel_score& rec, uint32_t* ids, uint32_t& st)
{
    const uint32_t n(rec.n_alt < 2 ? rec.n_alt : 2);
    for (uint32_t a = 0; a < n; ++a) ids[a] = k6b_gid_of(s, n_gid, g, rec.alt_key[a], st);
    return n;
}

// The read_path_lnp entry of record `rec` of read r, its alternates as indices into the locus's table alt_ids[0..n_alts): every byte.
K6B_HD sx_sindel_read k6b_entry(const sx_indel_reads_sample& s, const uint32_t n_gid, const uint32_t r, const sx_read_indel_score& rec, const uint32_t* alt_ids,
                                const uint32_t n_alts)
{
    sx_sindel_read e;
    e.ref = rec.ref_lnp;
    e.indel = rec.indel_lnp;
    e.read_length = s.read_len[r];
    e.non_ambig = s.non_ambig[r];
    e.is_tier1 = (s.read_flags[r] & SX_SIF_TIER1) ? 1 : 0;
    uint32_t ids[2], st(0);
    const uint32_t n(rec.n_alt ? k6b_alt_ids(s, n_gid, k6b_region_of(s, r), rec, ids, st) : 0u);
    e.n_alt = (uint8_t)n;
    for (uint32_t a = 0; a < 2; ++a)
    {
        uint32_t at(0);
        if (a < n)
            while (at + 1 < n_alts && alt_ids[at] != ids[a]) ++at;
        e.alt[a] = (uint8_t)at;
        e.alt_lnp[a] = a < n ? rec.alt_lnp[a] : 0.f;
    }
    return e;
}
