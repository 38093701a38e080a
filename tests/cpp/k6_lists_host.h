// tests/cpp/k6_lists_host.h -- TEST ONLY.  The list builder of K6b and K6g (strelka_b200/csrc/k6_lists.cuh) on the CPU, with the body's
// record walk and sort (k6b_core.cuh): count, scan, scatter, sort.  The scatter visits the reads BACKWARDS, so the segments reach the sort in
// an order the device never produces: the output must not depend on it.  `smem_sort` is the depth up to which a segment is sorted in a side
// buffer (the kernel's shared memory), beyond it in the scratch itself.
#pragma once

#include "k6b_core.cuh"

#include <vector>

struct k6l_host_lists
{
    std::vector<uint32_t> off, id, rec, read, order; // as the device's k6l_lists: segment n_samples * owner + sample at off[]
    std::vector<uint8_t> dup;                        // per owner: a read id twice in one of its segments
};

// The lists of the records `v` walks for the n_owners owners of v.locus_of; returns the walk's status bits (K6B_ST_BAD_ID).
inline uint32_t k6l_host_build(const k6b_view& v, const uint32_t n_samples, const uint32_t n_owners, const uint32_t smem_sort, k6l_host_lists& L)
{
    const uint32_t n_seg(n_samples * n_owners);
    uint32_t bad(0);
    L.off.assign(n_seg + 1, 0);
    for (uint32_t sample = 0; sample < n_samples; ++sample)
        for (uint32_t r = 0; r < v.s[sample].n_reads; ++r)
            bad |= k6b_for_each_entry(v, sample, r, [&](uint32_t o, uint32_t) { ++L.off[n_samples * o + sample + 1]; });
    for (uint32_t i = 0; i < n_seg; ++i) L.off[i + 1] += L.off[i];
    const uint32_t n_pairs(L.off[n_seg]);
    std::vector<uint32_t> cursor(L.off.begin(), L.off.end() - 1), key, val;
    L.id.assign(n_pairs, 0);
    L.rec.assign(n_pairs, 0);
    L.read.assign(n_pairs, 0);
    L.order.assign(n_pairs, 0);
    for (uint32_t sample = 0; sample < n_samples; ++sample)
        for (uint32_t r = v.s[sample].n_reads; r-- > 0;)
            k6b_for_each_entry(v, sample, r, [&](uint32_t o, uint32_t i) {
                const uint32_t at(cursor[n_samples * o + sample]++);
                L.id[at] = k6b_read_id(v.s[sample], r);
                L.rec[at] = i;
                L.read[at] = r;
            });
    L.dup.assign(n_owners, 0);
    for (uint32_t seg = 0; seg < n_seg; ++seg)
    {
        const uint32_t base(L.off[seg]), n(L.off[seg + 1] - base);
        if (n <= smem_sort)
        {
            key.assign(L.id.begin() + base, L.id.begin() + base + n);
            val.resize(n);
            for (uint32_t i = 0; i < n; ++i) val[i] = i;
            k6b_sort_by_key(key.data(), val.data(), n, 0u, 1u, [] {});
            for (uint32_t i = 0; i < n; ++i)
            {
                L.id[base + i] = key[i];
                L.order[base + i] = val[i];
            }
        }
        else
        {
            for (uint32_t i = 0; i < n; ++i) L.order[base + i] = i;
            k6b_sort_by_key(L.id.data() + base, L.order.data() + base, n, 0u, 1u, [] {});
        }
        for (uint32_t i = 0; i + 1 < n; ++i) L.dup[seg / n_samples] |= L.id[base + i] == L.id[base + i + 1];
    }
    return bad;
}
