// tests/cpp/k2c_core_host.cpp -- TEST ONLY.  Compiles the body of K2c (strelka_b200/csrc/k2c_core.cuh) with g++ and runs it the way the
// kernels of k2c_continuous.cu do: count each column, size each site's records, scan, write.  The sites are written in DESCENDING order,
// so the output must not depend on the order in which sites are visited.
#include "k2c_core.cuh"

#include <vector>

extern "C" void k2ccore_qscore(const uint32_t* a, const uint32_t* n, uint64_t count, double err_rate, int32_t max_q, int32_t* gq, uint32_t* status)
{
    for (uint64_t i = 0; i < count; ++i)
    {
        const k2c_q q = k2c_qscore(a[i], n[i], err_rate, max_q);
        gq[i] = q.gq;
        status[i] = q.status;
    }
}

extern "C" void k2ccore_strand_bias(const uint32_t* c, uint64_t count, double* out)
{
    for (uint64_t i = 0; i < count; ++i) out[i] = k2c_strand_bias(c[4 * i], c[4 * i + 1], c[4 * i + 2], c[4 * i + 3]);
}

// returns the record count; records are written only when it fits cap_loci
extern "C" uint32_t k2ccore_run(const sx_cont_opts* o, double err_rate, const sx_cont_batch* b, sx_cont_locus* loci_out, sx_cont_sample* samples_out,
                                uint32_t* site_rec_off, uint32_t cap_loci)
{
    const uint32_t n = b->n_sites, S = b->n_samples;
    std::vector<k2c_counts> cnt((size_t)n * S);
    for (uint32_t site = 0; site < n; ++site)
        for (uint32_t s = 0; s < S; ++s)
        {
            k2c_counts& c = cnt[(size_t)site * S + s];
            c = k2c_counts{};
            const sx_pileup_batch& p = b->sample[s];
            for (uint32_t i = p.site_off[site]; i < p.site_off[site + 1]; ++i)
                if (!k2c_is_filtered(p.calls[i])) ++c.n[k2c_is_fwd(p.calls[i])][k2c_base_of(p.calls[i])];
            c.raw = p.site_off[site + 1] - p.site_off[site];
        }
    uint8_t loci[5];
    site_rec_off[0] = 0;
    for (uint32_t site = 0; site < n; ++site)
    {
        const bool forced = b->forced_output && b->forced_output[site];
        site_rec_off[site + 1] = site_rec_off[site] + k2c_site_loci(&cnt[(size_t)site * S], S, k2c_ref_id(b->sample[0].ref_base[site]), forced, o->min_het_vf, loci);
    }
    const uint32_t total = site_rec_off[n];
    if (total > cap_loci) return total;
    for (uint32_t site = n; site-- > 0;)
    {
        const k2c_counts* c = &cnt[(size_t)site * S];
        const uint32_t ref = k2c_ref_id(b->sample[0].ref_base[site]);
        const bool forced = b->forced_output && b->forced_output[site];
        const uint32_t m = k2c_site_loci(c, S, ref, forced, o->min_het_vf, loci), r0 = site_rec_off[site];
        for (uint32_t li = 0; li < m; ++li)
        {
            int32_t qual = 0;
            for (uint32_t s = 0; s < S; ++s)
            {
                const sx_cont_sample e = k2c_entry(c[s], ref, loci[li], *o, err_rate);
                samples_out[(size_t)(r0 + li) * S + s] = e;
                if (e.gq > qual) qual = e.gq;
            }
            loci_out[r0 + li] = k2c_locus(c, S, b->pos_begin + static_cast<int32_t>(site), ref, loci[li], forced, qual);
        }
    }
    return total;
}
