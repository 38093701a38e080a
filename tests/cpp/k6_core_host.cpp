// tests/cpp/k6_core_host.cpp -- TEST ONLY.  Compiles the device body of K6 (strelka_b200/csrc/k6_core.cuh, __host__ __device__)
// with g++ and runs it read by read on the CPU, so that the container without a GPU can check the kernel's logic against the
// oracle.  Not part of the product: libstrelka_b200.so has no host execution path.
#include "k6_core.cuh"

#include <algorithm>
#include <vector>

// list_walk == 0: the plain body, region by region, read by read.
// list_walk != 0: what sx_k6_run and k6_score_list_kernel do -- the host memsets of n_rec / max_aln / eval_aln for every read, then
// the body on the dense list of reads that have alignments, walked backwards (the kernel's regrouping makes the order arbitrary), each
// read with its region from k6_region_of and the scratch k6_score_read_tiered picks.  counts[0] = reads skipped (no alignment),
// counts[1 + tier] = listed reads per k6_scratch_tier.
extern "C" int k6core_run(const sx_score_indels_batch* b, const double* lnp, sx_read_indel_score* recs, uint32_t* n_rec, uint32_t* max_aln, uint32_t* eval_aln,
                          uint32_t* status_out, uint32_t list_walk, uint32_t* counts)
{
    std::fill(counts, counts + 4, 0u);
    uint32_t maxA(1), maxE(1);
    for (uint32_t r = 0; r < b->n_reads; ++r)
    {
        maxA = std::max(maxA, b->aln_off[r + 1] - b->aln_off[r]);
        maxE = std::max(maxE, std::min<uint32_t>(K6_MAX_EVAL, b->rec_off[r + 1] - b->rec_off[r]));
    }
    std::vector<uint32_t> ord(maxA);
    std::vector<double> smooth(maxA);
    std::vector<float> present(maxE), absent(maxE), alt((size_t)maxE * maxE);
    std::vector<uint16_t> slot(maxE);
    std::vector<uint8_t> filt(maxA), has(maxE), pair((size_t)maxE * maxE);
    std::vector<uint16_t> ev(maxE);
    k6_scratch S;
    S.ord = {ord.data(), 1};
    S.smooth = {smooth.data(), 1};
    S.filt = {filt.data(), 1};
    S.ev = {ev.data(), 1};
    S.slot = {slot.data(), 1};
    S.present = {present.data(), 1};
    S.absent = {absent.data(), 1};
    S.has = {has.data(), 1};
    S.alt = {alt.data(), 1};
    S.pair = {pair.data(), 1};
    S.maxA = maxA;
    S.maxE = maxE;
    k6_view v;
    v.b = *b;
    v.lnp = lnp;
    v.recs = recs;
    v.n_rec = n_rec;
    v.max_aln = max_aln;
    v.eval_aln = eval_aln;
    uint32_t status(0);
    if (list_walk == 0)
    {
        for (uint32_t region = 0; region < b->n_regions; ++region)
            for (uint32_t r = b->region_read_off[region]; r < b->region_read_off[region + 1]; ++r) status |= k6_score_read(v, region, r, S);
    }
    else
    {
        std::fill(n_rec, n_rec + b->n_reads, 0u); // sx_k6_run's memsets
        std::fill(max_aln, max_aln + b->n_reads, 0xFFFFFFFFu);
        std::fill(eval_aln, eval_aln + b->n_reads, 0xFFFFFFFFu);
        std::vector<uint32_t> list; // k6_max_kernel's list
        for (uint32_t r = 0; r < b->n_reads; ++r)
        {
            if (b->aln_off[r + 1] > b->aln_off[r]) list.push_back(r);
            else ++counts[0];
        }
        for (auto it = list.rbegin(); it != list.rend(); ++it)
        {
            const uint32_t r(*it);
            ++counts[1 + k6_scratch_tier(v.b, r)];
            status |= k6_score_read_tiered(v, k6_region_of(b->region_read_off, b->n_regions, r), r, S);
        }
    }
    *status_out = status;
    return 0;
}
