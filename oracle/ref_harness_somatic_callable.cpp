// oracle/ref_harness_somatic_callable.cpp -- TEST INFRASTRUCTURE, not product code.  A C-ABI shim that drives the reference's own
// somatic_snv_caller_strand_grid::position_somatic_snv_call with isComputeNonSomatic = true (applications/strelka/
// position_somatic_snv_strand_grid.cpp:228-363, compiled unmodified by oracle/build_ref.sh) on flattened pile-up batches, the way
// strelka_pos_processor::process_pos_snp_somatic does when it writes the callable regions (strelka_pos_processor.cpp:181-224): each
// position's result goes to the reference's SomaticCallableProcessor, whose BED text is returned with the records.
#include "../include/strelka_b200.h"

#include "applications/strelka/SomaticCallableProcessor.hh"
#include "applications/strelka/position_somatic_snv_strand_grid.hh"
#include "applications/strelka/strelka_shared.hh"
#include "blt_common/snp_pos_info.hh"
#include "starling_common/PileupCleaner.hh"

#include <cstring>
#include <exception>
#include <sstream>
#include <string>

namespace
{
void set_err(char* err, int errlen, const char* msg)
{
    if (err && errlen > 0)
    {
        std::strncpy(err, msg, errlen - 1);
        err[errlen - 1] = 0;
    }
}

// the pile-up encoding and option mapping of oracle/ref_harness.cpp
base_call make_call(const uint16_t raw)
{
    return base_call((raw >> 6) & 15, raw & 63, (raw >> 10) & 1, 0, 0, (raw >> 12) & 1, (raw >> 11) & 1, (raw >> 13) & 1);
}

void fill_pileup(const sx_pileup_batch* b, const uint32_t s, snp_pos_info& pi)
{
    pi.clear();
    pi.set_ref_base(b->ref_base[s]);
    for (uint32_t i = b->site_off[s]; i < b->site_off[s + 1]; ++i) pi.calls.push_back(make_call(b->calls[i]));
    if (b->t2_off)
        for (uint32_t i = b->t2_off[s]; i < b->t2_off[s + 1]; ++i) pi.tier2_calls.push_back(make_call(b->t2_calls[i]));
}
} // namespace

// records into out[n_sites]; the BED text of positions pos_begin + s (0-based) on chromosome `chrom` into bed[bed_cap] (NUL-terminated),
// its length into *bed_len.  Returns 0, 1 on an exception (message in err), or 2 when bed_cap is too small (*bed_len says how much is needed).
extern "C" int ref_site_gl_somatic_callable(const sx_params* p, const sx_pileup_batch* normal, const sx_pileup_batch* tumor, const uint8_t* is_forced_output,
                                            const char* chrom, int32_t pos_begin, sx_ssnv_result* out, char* bed, uint64_t bed_cap, uint64_t* bed_len, char* err,
                                            int errlen)
{
    try
    {
        strelka_options opt;
        opt.bsnp_diploid_theta = p->bsnp_diploid_theta;
        opt.bsnp_ssd_no_mismatch = p->bsnp_ssd_no_mismatch;
        opt.bsnp_ssd_one_mismatch = p->bsnp_ssd_one_mismatch;
        opt.is_min_vexp = (p->is_min_vexp != 0);
        opt.min_vexp = p->min_vexp;
        opt.hetVariantFrequencyExtension = p->hetVariantFrequencyExtension;
        opt.somatic_snv_rate = p->somatic_snv_rate;
        opt.shared_site_error_rate = p->shared_site_error_rate;
        opt.shared_site_error_strand_bias_fraction = p->shared_site_error_strand_bias_fraction;
        opt.ssnv_contam_tolerance = p->ssnv_contam_tolerance;
        const somatic_snv_caller_strand_grid caller(opt);
        PileupCleaner cleaner(opt);
        const bool is_tier2(normal->t2_off != nullptr && tumor->t2_off != nullptr);
        snp_pos_info npi, tpi;
        CleanedPileup ncpi[2], tcpi[2];
        std::ostringstream os;
        {
            SomaticCallableProcessor scall(&os);
            const std::string chrom_name(chrom);
            for (uint32_t s = 0; s < normal->n_sites; ++s)
            {
                sx_ssnv_result& o(out[s]);
                std::memset(&o, 0, sizeof(o));
                fill_pileup(normal, s, npi);
                fill_pileup(tumor, s, tpi);
                cleaner.CleanPileupFilter(npi, false, ncpi[0]);
                cleaner.CleanPileupFilter(tpi, false, tcpi[0]);
                if (is_tier2)
                {
                    cleaner.CleanPileupFilter(npi, true, ncpi[1]);
                    cleaner.CleanPileupFilter(tpi, true, tcpi[1]);
                }
                for (int t = 0; t < (is_tier2 ? 2 : 1); ++t)
                {
                    cleaner.CleanPileupErrorProb(ncpi[t]);
                    cleaner.CleanPileupErrorProb(tcpi[t]);
                }
                somatic_snv_genotype_grid sgt;
                sgt.is_forced_output = is_forced_output ? (is_forced_output[s] != 0) : false;
                const extended_pos_info* nt2(is_tier2 ? &ncpi[1].getExtendedPosInfo() : nullptr);
                const extended_pos_info* tt2(is_tier2 ? &tcpi[1].getExtendedPosInfo() : nullptr);
                caller.position_somatic_snv_call(ncpi[0].getExtendedPosInfo(), tcpi[0].getExtendedPosInfo(), nt2, tt2, true, sgt);
                scall.addToRegion(chrom_name, pos_begin + (int32_t)s + 1, sgt);
                // computed: every position whose reference base is not 'N' (the caller returns before setting ref_gt there)
                o.ref_gt = sgt.ref_gt;
                o.is_computed = (normal->ref_base[s] != 'N') ? 1 : 0;
                o.snv_tier = sgt.snv_tier;
                o.snv_from_ntype_tier = sgt.snv_from_ntype_tier;
                o.ntype = sgt.rs.ntype;
                o.max_gt = sgt.rs.max_gt;
                o.qphred = sgt.rs.qphred;
                o.from_ntype_qphred = sgt.rs.from_ntype_qphred;
                o.normal_alt_id = sgt.rs.normal_alt_id;
                o.tumor_alt_id = sgt.rs.tumor_alt_id;
                o.strandBias = sgt.rs.strandBias;
                o.nonsomatic_qphred = sgt.rs.nonsomatic_qphred;
            }
        } // (RegionProcessor flushes its last interval on destruction)
        const std::string text(os.str());
        *bed_len = text.size();
        if (text.size() + 1 > bed_cap) return 2;
        std::memcpy(bed, text.c_str(), text.size() + 1);
        return 0;
    }
    catch (const std::exception& e)
    {
        set_err(err, errlen, e.what());
        return 1;
    }
}
