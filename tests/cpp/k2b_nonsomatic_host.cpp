// tests/cpp/k2b_nonsomatic_host.cpp -- TEST ONLY.  Compiles the body of K2b's callable mode (strelka_b200/csrc/k2b_nonsomatic.cuh) with g++
// and runs it on the tier1 likelihoods of each record, as the kernel does: the whole computation, and the predicate of each state.
#include "k2b_nonsomatic.cuh"

#include "strelka_b200.h"

extern "C" void k2bn_host_qphred(const sx_ssnv_result* r, uint64_t count, int32_t* out)
{
    for (uint64_t i = 0; i < count; ++i) out[i] = k2bn_nonsomatic_qphred(r[i].normal_lhood, r[i].tumor_lhood);
}

// per record, which of opt_normalize_ln_distro's outcomes its states reach: bit 0 a state kept (exp), bit 1 a state dropped as off the
// diagonal, bit 2 a diagonal state dropped by the opt_max test, bit 3 a diagonal state kept although max - p > 20
extern "C" void k2bn_host_outcomes(const sx_ssnv_result* r, uint64_t count, uint32_t* out)
{
    for (uint64_t k = 0; k < count; ++k)
    {
        const float *nl = r[k].normal_lhood, *tl = r[k].tumor_lhood;
        double max = k2bn_pprob(nl, tl, 0);
        for (uint32_t i = 1; i < K2BN_STATES; ++i)
        {
            const double p = k2bn_pprob(nl, tl, i);
            if (p > max) max = p;
        }
        const double opt_max = k2bn_pprob(nl, tl, 0);
        uint32_t m = 0;
        for (uint32_t i = 0; i < K2BN_STATES; ++i)
        {
            const double p = k2bn_pprob(nl, tl, i);
            if (!(max - p > 20.0)) m |= 1u;
            else if (i % K2BN_DIAG_STRIDE != 0) m |= 2u;
            else if (opt_max - p > 5.0) m |= 4u;
            else m |= 8u;
        }
        out[k] = m;
    }
}
