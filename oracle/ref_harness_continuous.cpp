// oracle/ref_harness_continuous.cpp -- TEST INFRASTRUCTURE, not product code.  A C-ABI shim over the reference's own
// starling_continuous_variant_caller::getAlleleSequencingErrorQscore and ::strandBias (applications/starling/
// starling_continuous_variant_caller.cpp, compiled unmodified by oracle/build_ref.sh), batched for the goldens and the `ref` tests.
#include "applications/starling/starling_continuous_variant_caller.hh"

#include <cstdint>

extern "C" void refc_qscore(const uint32_t* a, const uint32_t* n, uint64_t count, int expected_qscore, int max_qscore, int32_t* out)
{
    for (uint64_t i = 0; i < count; ++i) out[i] = starling_continuous_variant_caller::getAlleleSequencingErrorQscore(a[i], n[i], expected_qscore, max_qscore);
}

// counts[4 * i ..] = fwdAlt, revAlt, fwdOther, revOther
extern "C" void refc_strand_bias(const uint32_t* counts, uint64_t count, double* out)
{
    for (uint64_t i = 0; i < count; ++i)
        out[i] = starling_continuous_variant_caller::strandBias(counts[4 * i], counts[4 * i + 1], counts[4 * i + 2], counts[4 * i + 3]);
}
