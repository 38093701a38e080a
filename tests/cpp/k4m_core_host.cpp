// tests/cpp/k4m_core_host.cpp -- TEST ONLY.  Compiles K4m's per-site statistics (strelka_b200/csrc/k4m_core.cuh) with g++ and runs them on
// CSR observation words, one site after another.
#include "k4m_core.cuh"

extern "C" void k4m_host_sites(const uint64_t* words, const uint32_t* off, uint32_t n_sites, uint32_t mode, sx_pileup_metrics_rec* out)
{
    for (uint32_t s = 0; s < n_sites; ++s) k4m_site_scalar(words + off[s], off[s + 1] - off[s], mode, &out[s]);
}

// the packing of one observation, as the kernel writes it
extern "C" uint64_t k4m_host_pack(uint32_t mapq, uint32_t qscore, uint32_t is_ref, uint32_t submapped, uint32_t somatic, uint32_t edge, uint32_t cycle,
                                  uint32_t read_pos, uint32_t read_size)
{
    const k4m_obs o = {mapq, qscore, is_ref, submapped, somatic, edge, cycle, read_pos, read_size};
    return k4m_pack(o);
}

extern "C" uint32_t k4m_host_edge_distance(uint32_t p, uint32_t full_off, uint32_t full_size) { return k4m_edge_distance(p, full_off, full_size); }
