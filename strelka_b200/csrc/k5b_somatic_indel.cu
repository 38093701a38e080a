// k5b_somatic_indel.cu -- K5b somatic_indel: the somatic caller's indel model, one warp per candidate indel.
//
// Replaces somatic_indel_caller_grid::get_somatic_indel (/root/reference/src/c++/lib/applications/strelka/somatic_indel_grid.cpp:181-361):
//   is_multi_indel_allele                 :100-175, with get_sum_path_pprob (starling_common/starling_indel_call_pprob_digt.cpp:186-235),
//                                         indel_lnp_to_pprob (starling_common/AlleleReportInfoUtil.cpp:220-297), is_indel_conflict (k6_conflict)
//   get_indel_digt_lhood                  starling_indel_call_pprob_digt.cpp:240-336
//   get_indel_het_grid_lhood              somatic_indel_grid.cpp:66-90 -> get_high_low_het_ratio_lhood :75-155
//   get_het_observed_allele_ratio         :40-71 ; integrateOutMappingStatus  starling_common/readMappingAdjustmentUtil.hh:46-56
//   calculate_result_set_grid             qscore_calculator.cpp:47-209 (sx_result_set_grid.cuh)
//
// Parity contract.  Lanes 0..20 each own one of the 21 likelihood states of a sample and add that state's term read by read, in
// read_path_lnp order, so every double sum is the reference's; the terms use the reference's libm restated (sx_log_sum.cuh,
// sx_libm_mirror_d.h).  The multi-indel filter's per-read posteriors are computed one read per lane and summed by lane 0 in read order,
// in float as ReadPathScores::score_t is.  Everything the reference derives from an option alone, and the shared-error terms of each
// indelToRefErrorProb (std::pow has no restatement here), are computed on the host.
#include "sx_device_util.cuh"
#include "sx_internal.h"
#include "sx_log_sum.cuh"
#include "sx_result_set_grid.cuh"
#include "k6_core.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>

namespace
{
constexpr int K5B_WARPS = 4;
constexpr unsigned FULL = 0xffffffffu;
constexpr int K5B_MAX_TOTAL = 2 * SX_SINDEL_MAX_ALTS; // total_pprob.alt_indel: the normal and the tumor pass each start their own map

// per-call constants (k5b_consts_of, on the host)
struct k5b_consts
{
    // calculate_result_set_grid's term lists at indel_contam_tolerance.  term_kind 0: lprior_freq is term_lprior; 1: the locus's
    // logSharedErrorRateComplement; 2: the locus's logSharedErrorRate + log_error_mod (a float sum)
    double term_lprior[6][44];
    uint8_t term_kind[6][44], term_tf[6][44], term_nf[6][44];
    uint32_t n_terms[6];
    float geno_prior[6];
    float log_error_mod;
    // likelihood lane k: the allele ratio it hands get_het_observed_allele_ratio and the log ratios that stand when total_path_term == 0
    double ratio[21], def_lr[21], def_li[21];
    double correctMappingLogPrior;
    double randomBaseMatchLogProb[2]; // [tier1 pass, tier2 pass]
    double allele_lnprior[5];         // std::log(1./n) for n = 2..4 alleles
    uint32_t min_flank[2];
    int32_t useTier2Evidence;
    int32_t pad;
};

struct k5b_terms // calculate_result_set_grid's terms of one locus
{
    const k5b_consts& C;
    double lcse, lse_mod;
    __device__ __forceinline__ uint32_t n_terms(uint32_t combo) const { return C.n_terms[combo]; }
    __device__ __forceinline__ double lprior(uint32_t combo, uint32_t i) const
    {
        const uint32_t k = C.term_kind[combo][i];
        return k == 0 ? C.term_lprior[combo][i] : k == 1 ? lcse : lse_mod;
    }
    __device__ __forceinline__ uint32_t nf(uint32_t combo, uint32_t i) const { return C.term_nf[combo][i]; }
    __device__ __forceinline__ uint32_t tf(uint32_t combo, uint32_t i) const { return C.term_tf[combo][i]; }
    __device__ __forceinline__ float geno_prior(uint32_t combo) const { return C.geno_prior[combo]; }
};

struct tier_rs // indel_result_set
{
    uint32_t ntype, max_gt;
    int qphred, from_ntype_qphred;
};

struct warp_scratch
{
    float nl[32], tl[32];
    double grid[44];
    // the filter: one read per lane, then lane 0's ordered sums
    float pp_ref[32], pp_indel[32], pp_alt[32][2];
    uint8_t used[32];
    float tot_alt[K5B_MAX_TOTAL];
    uint8_t tot_key[K5B_MAX_TOTAL];
    sx_indel_key alts[SX_SINDEL_MAX_ALTS];
};

// indel_lnp_to_pprob of one read (is_use_alt_indel = true): ReadPathScores of float values after double arithmetic
__device__ __forceinline__ void read_pprob(const k5b_consts& C, const sx_sindel_read& rd, const uint32_t pass, float& ref, float& indel, float* alt)
{
    const double lnprior = C.allele_lnprior[2 + rd.n_alt];
    float inc = static_cast<float>(d_mul(C.randomBaseMatchLogProb[pass], static_cast<double>(rd.non_ambig)));
    ref = static_cast<float>(d_add(d_add(static_cast<double>(rd.ref), C.correctMappingLogPrior), lnprior));
    indel = static_cast<float>(d_add(d_add(static_cast<double>(rd.indel), C.correctMappingLogPrior), lnprior));
    for (uint32_t k = 0; k < rd.n_alt; ++k) alt[k] = static_cast<float>(d_add(d_add(static_cast<double>(rd.alt_lnp[k]), C.correctMappingLogPrior), lnprior));
    const float m = (ref < indel) ? indel : ref;         // std::max(pprob.ref, pprob.indel)
    double scale = static_cast<double>((inc < m) ? m : inc); // std::max(pprob_readIncorrectlyMapped, ...)
    for (uint32_t k = 0; k < rd.n_alt; ++k)
        if (scale < static_cast<double>(alt[k])) scale = alt[k];
    inc = static_cast<float>(sx_exp(d_sub(static_cast<double>(inc), scale)));
    ref = static_cast<float>(sx_exp(d_sub(static_cast<double>(ref), scale)));
    indel = static_cast<float>(sx_exp(d_sub(static_cast<double>(indel), scale)));
    for (uint32_t k = 0; k < rd.n_alt; ++k) alt[k] = static_cast<float>(sx_exp(d_sub(static_cast<double>(alt[k]), scale)));
    double sum = static_cast<double>(f_add(f_add(inc, ref), indel)); // score_t + score_t + score_t, in float
    for (uint32_t k = 0; k < rd.n_alt; ++k) sum = d_add(sum, static_cast<double>(alt[k]));
    ref = static_cast<float>(d_div(static_cast<double>(ref), sum));
    indel = static_cast<float>(d_div(static_cast<double>(indel), sum));
    for (uint32_t k = 0; k < rd.n_alt; ++k) alt[k] = static_cast<float>(d_div(static_cast<double>(alt[k]), sum));
}

// is_multi_indel_allele (is_include_tier2 = pass); every lane returns the same answer
__device__ bool multi_indel_filter(const k5b_consts& C, warp_scratch& W, const sx_sindel_read* __restrict__ reads, const uint32_t* rb, const uint32_t pass,
                                   const uint32_t lane, bool& is_overlap)
{
    float tot_ref = 0.f, tot_indel = 0.f; // lane 0's
    uint32_t n_tot = 0;
    for (uint32_t s = 0; s < 2; ++s)
    {
        int8_t slot_of[SX_SINDEL_MAX_ALTS]; // get_sum_path_pprob's alt_indel_index, one per call
#pragma unroll
        for (int a = 0; a < SX_SINDEL_MAX_ALTS; ++a) slot_of[a] = -1;
        for (uint32_t r0 = rb[s]; r0 < rb[s + 1]; r0 += 32)
        {
            const uint32_t r = r0 + lane;
            W.used[lane] = 0;
            if (r < rb[s + 1])
            {
                const sx_sindel_read rd = reads[r];
                if (pass == 1 || rd.is_tier1)
                {
                    float alt[2] = {0.f, 0.f};
                    read_pprob(C, rd, pass, W.pp_ref[lane], W.pp_indel[lane], alt);
                    W.pp_alt[lane][0] = alt[0];
                    W.pp_alt[lane][1] = alt[1];
                    W.used[lane] = 1;
                }
            }
            __syncwarp();
            if (lane == 0)
            {
                const uint32_t n = min(32u, rb[s + 1] - r0);
                for (uint32_t k = 0; k < n; ++k)
                {
                    if (!W.used[k]) continue;
                    tot_indel = f_add(tot_indel, W.pp_indel[k]);
                    tot_ref = f_add(tot_ref, W.pp_ref[k]);
                    const sx_sindel_read& rd = reads[r0 + k];
                    for (uint32_t j = 0; j < rd.n_alt; ++j)
                    {
                        const uint32_t a = rd.alt[j];
                        if (slot_of[a] < 0)
                        {
                            slot_of[a] = static_cast<int8_t>(n_tot);
                            W.tot_key[n_tot] = static_cast<uint8_t>(a);
                            W.tot_alt[n_tot] = W.pp_alt[k][j];
                            ++n_tot;
                        }
                        else W.tot_alt[slot_of[a]] = f_add(W.tot_alt[slot_of[a]], W.pp_alt[k][j]);
                    }
                }
            }
            __syncwarp();
        }
    }
    uint32_t verdict = 0; // bit 0: filtered, bit 1: is_overlap
    if (lane == 0)
    {
        // scores: (-pprob, id) with INDEL = -2, REF = -1, alternates 0.. in first-seen order; std::sort order, ties broken on the id
        double sc[2 + K5B_MAX_TOTAL] = {};
        int id[2 + K5B_MAX_TOTAL] = {};
        uint32_t n = 0;
        auto push = [&](const double v, const int i) {
            uint32_t j = n++;
            while (j > 0 && (v < sc[j - 1] || (v == sc[j - 1] && i < id[j - 1])))
            {
                sc[j] = sc[j - 1];
                id[j] = id[j - 1];
                --j;
            }
            sc[j] = v;
            id[j] = i;
        };
        push(-static_cast<double>(tot_indel), -2);
        push(-static_cast<double>(tot_ref), -1);
        for (uint32_t i = 0; i < n_tot; ++i) push(-static_cast<double>(W.tot_alt[i]), static_cast<int>(i));
        while (id[0] >= 0 && id[1] >= 0)
        {
            if (k6_conflict(W.alts[W.tot_key[id[0]]], W.alts[W.tot_key[id[1]]])) break;
            for (uint32_t j = 1; j + 1 < n; ++j)
            {
                sc[j] = sc[j + 1];
                id[j] = id[j + 1];
            }
            --n;
        }
        bool filtered = (id[0] != -2) && (id[1] != -2);
        if (!filtered && n >= 3)
        {
            const double top_prob = d_add(sc[0], sc[1]);
            const double top_frac = d_div(top_prob, d_add(top_prob, sc[2]));
            if (top_frac < 0.9) filtered = true;
        }
        verdict = filtered ? 1u : ((id[0] != -1) && (id[1] != -1) ? 2u : 0u);
    }
    verdict = __shfl_sync(FULL, verdict, 0);
    if (verdict & 2u) is_overlap = true;
    return (verdict & 1u) != 0;
}

// get_indel_digt_lhood (lanes 0..2) and get_indel_het_grid_lhood (lanes 3..20) of one sample, cast to float; lanes 21.. return 0
__device__ __forceinline__ float sample_lhood(const k5b_consts& C, const sx_sindel_read* __restrict__ reads, const uint32_t r0, const uint32_t r1, const uint32_t pass,
                                              const uint32_t del_len, const uint32_t ins_len, const uint32_t min_overlap, const uint32_t lane)
{
    const bool active = lane < 21;
    const uint32_t li_ = active ? lane : 0;
    const double ratio = C.ratio[li_], def_lr = C.def_lr[li_], def_li = C.def_li[li_];
    const double rbm = C.randomBaseMatchLogProb[pass], cmlp = C.correctMappingLogPrior;
    double acc = 0.0;
    for (uint32_t r = r0; r < r1; ++r)
    {
        const sx_sindel_read rd = reads[r];
        if (pass == 0 && !rd.is_tier1) continue;
        double alt_path_lnp = rd.ref;
        for (uint32_t k = 0; k < rd.n_alt; ++k)
            if (static_cast<double>(rd.alt_lnp[k]) > alt_path_lnp) alt_path_lnp = rd.alt_lnp[k];
        const double noindel_lnp = alt_path_lnp, hom_lnp = rd.indel;
        double x;
        if (lane == 0) x = noindel_lnp;
        else if (lane == 1) x = hom_lnp;
        else
        {
            // get_het_observed_allele_ratio: unsigned base_expect; the defaults stand when total_path_term == 0
            double log_ref_prob = def_lr, log_indel_prob = def_li;
            const uint32_t rlen = rd.read_length;
            const uint32_t base_expect = ((rlen + 1) < (2 * min_overlap)) ? 0u : (rlen + 1) - (2 * min_overlap);
            const double ref_path_expect = static_cast<double>(base_expect + min(del_len, base_expect));
            const double indel_path_expect = static_cast<double>(base_expect + min(ins_len, base_expect));
            const double ref_path_term = d_mul(d_sub(1.0, ratio), ref_path_expect);
            const double indel_path_term = d_mul(ratio, indel_path_expect);
            const double total_path_term = d_add(ref_path_term, indel_path_term);
            if (total_path_term > 0)
            {
                const double indel_prob = d_div(indel_path_term, total_path_term);
                log_ref_prob = sx_log(d_sub(1.0, indel_prob));
                log_indel_prob = sx_log(indel_prob);
            }
            x = get_log_sum(d_add(noindel_lnp, log_ref_prob), d_add(hom_lnp, log_indel_prob));
        }
        // integrateOutMappingStatus; the incorrect-mapping term follows the pass, not the read (isTier2 = is_tier2_pass)
        if (active) acc = d_add(acc, get_log_sum(d_add(x, cmlp), d_mul(rbm, static_cast<double>(rd.non_ambig))));
    }
    return active ? static_cast<float>(acc) : 0.f;
}

__global__ void __launch_bounds__(K5B_WARPS * 32)
    k5b_somatic_indel_kernel(const sx_sindel_batch b, const k5b_consts* __restrict__ consts, const float2* __restrict__ err_terms, const uint32_t n_err,
                             sx_sindel_result* __restrict__ out, int* __restrict__ status)
{
    __shared__ k5b_consts C;
    __shared__ warp_scratch S[K5B_WARPS];
    for (uint32_t i = threadIdx.x; i < sizeof(k5b_consts) / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(&C)[i] = reinterpret_cast<const uint32_t*>(consts)[i];
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    warp_scratch& W = S[warp];

    for (uint32_t l = blockIdx.x * K5B_WARPS + warp; l < b.n_loci; l += gridDim.x * K5B_WARPS)
    {
        sx_sindel_result* res = out + l;
        {
            uint32_t* w = reinterpret_cast<uint32_t*>(res);
            for (uint32_t i = lane; i < sizeof(sx_sindel_result) / 4; i += 32) w[i] = 0u;
        }
        __syncwarp();
        const sx_indel_key key = b.key[l];
        const uint32_t eidx = b.err_idx[l];
        if (key.type != SX_INDEL_TYPE_INDEL || eidx >= n_err)
        {
            if (lane == 0) atomicOr(status, SX_ST_SINDEL_ARG);
            continue;
        }
        const bool forced = b.is_forced_output[l] != 0;
        const uint32_t a0 = b.alt_off[l], n_alts = b.alt_off[l + 1] - a0;
        const uint32_t rb[3] = {b.read_off[2 * l], b.read_off[2 * l + 1], b.read_off[2 * l + 2]};
        // capacities: the alternate table, and every read's alternates (at most two, each in the table)
        bool over = n_alts > SX_SINDEL_MAX_ALTS;
        for (uint32_t r = rb[0] + lane; r < rb[2] && !over; r += 32)
        {
            const sx_sindel_read& rd = b.reads[r];
            if (rd.n_alt > 2 || (rd.n_alt > 0 && rd.alt[0] >= n_alts) || (rd.n_alt > 1 && rd.alt[1] >= n_alts)) over = true;
        }
        if (__any_sync(FULL, over))
        {
            if (lane == 0) res->status = SX_ST_SINDEL_CAP;
            continue;
        }
        if (lane < n_alts) W.alts[lane] = b.alts[a0 + lane];
        __syncwarp();
        const float2 et = err_terms[eidx]; // (float) logSharedIndelErrorRate, (float) logSharedIndelErrorRateComplement
        const k5b_terms terms{C, static_cast<double>(et.y), static_cast<double>(f_add(et.x, C.log_error_mod))};

        tier_rs trs[2] = {{0, 0, 0, 0}, {0, 0, 0, 0}};
        bool overlap[2] = {false, false}, multi[2] = {false, false};
        for (uint32_t i = 0; i < 2; ++i)
        {
            if (i == 1)
            {
                if (!C.useTier2Evidence) continue;
                if (trs[0].qphred == 0 && !forced)
                {
                    trs[1].qphred = 0;
                    continue;
                }
            }
            const bool filtered = multi_indel_filter(C, W, b.reads, rb, i, lane, overlap[i]);
            multi[i] = filtered;
            if (filtered && !forced)
            {
                trs[i].qphred = 0;
                continue;
            }
            const float nl = sample_lhood(C, b.reads, rb[0], rb[1], i, key.del_len, key.ins_len, C.min_flank[0], lane);
            const float tl = sample_lhood(C, b.reads, rb[1], rb[2], i, key.del_len, key.ins_len, C.min_flank[1], lane);
            W.nl[lane] = nl;
            W.tl[lane] = tl;
            __syncwarp();
            result_set_grid(terms, W.nl, W.tl, W.grid, lane, trs[i]);
            if (filtered) trs[i].qphred = 0;
            sx_sindel_tier& t = res->tier[i];
            if (lane < 21)
            {
                t.normal_lhood[lane] = nl;
                t.tumor_lhood[lane] = tl;
            }
            if (lane == 0)
            {
                t.qphred = trs[i].qphred;
                t.from_ntype_qphred = trs[i].from_ntype_qphred;
                t.ntype = trs[i].ntype;
                t.max_gt = trs[i].max_gt;
                t.evaluated = 1;
            }
            __syncwarp();
        }
        if (lane == 0)
        {
            res->tier[0].is_overlap = overlap[0];
            res->tier[1].is_overlap = overlap[1];
            res->tier[0].multi_indel = multi[0];
            res->tier[1].multi_indel = multi[1];
        }
        if (!forced && (trs[0].qphred == 0 || trs[1].qphred == 0)) continue;
        uint32_t sindel_tier = 0, from_tier = 0;
        if (C.useTier2Evidence)
        {
            if (trs[0].qphred > trs[1].qphred) sindel_tier = 1;
            if (trs[0].from_ntype_qphred > trs[1].from_ntype_qphred) from_tier = 1;
        }
        tier_rs rs = trs[from_tier];
        if (trs[0].ntype != trs[1].ntype)
        {
            rs.ntype = 3; // NTYPE::CONFLICT
            rs.from_ntype_qphred = 0;
        }
        else rs.ntype = rs.ntype == 0 ? 0u : rs.ntype == 1 ? 1u : 2u; // SOMATIC_DIGT -> NTYPE
        rs.qphred = trs[sindel_tier].qphred;
        if (lane == 0)
        {
            res->is_output = 1;
            res->sindel_tier = static_cast<uint8_t>(sindel_tier);
            res->sindel_from_ntype_tier = static_cast<uint8_t>(from_tier);
            res->is_overlap = overlap[from_tier];
            res->ntype = rs.ntype;
            res->max_gt = rs.max_gt;
            res->qphred = rs.qphred;
            res->from_ntype_qphred = rs.from_ntype_qphred;
        }
    }
}

// the per-call constants, with the host libm in the reference's expression shapes
void k5b_consts_of(const sx_sindel_opts& o, k5b_consts& C)
{
    typedef float blt_float_t;
    memset(&C, 0, sizeof(C));
    const blt_float_t RATIO_INCREMENT = 0.5f / static_cast<blt_float_t>(9 + 1); // strelka_digt_states.hh:98
    // calculate_result_set_grid's loop (qscore_calculator.cpp:63-123), unrolled into ordered term lists
    {
        const blt_float_t contam_tolerance = static_cast<blt_float_t>(o.indel_contam_tolerance);
        static const blt_float_t ln_one_half(std::log(1. / 2.));
        static const blt_float_t log_error_mod = -std::log(static_cast<double>(21 - 1));
        C.log_error_mod = log_error_mod;
        auto fraction_of = [&](int index) -> blt_float_t { // strelka_digt_states.cpp:34-41
            if (index == 0) return 0.f;
            if (index == 1) return 1.f;
            if (index == 2) return 0.5f;
            if (index < 3 + 9) return RATIO_INCREMENT * (index - 3 + 1);
            return RATIO_INCREMENT * (index - 3 + 2);
        };
        // somatic_indel_caller_grid ctor (somatic_indel_grid.cpp:58-64) and calculateGermlineGenotypeLogPrior (qscore_calculator.cpp:33-42)
        const blt_float_t ln_som_match = static_cast<blt_float_t>(log1p_switch(-o.somatic_indel_rate));
        const blt_float_t ln_som_mismatch = static_cast<blt_float_t>(std::log(o.somatic_indel_rate));
        const double theta = o.bindel_diploid_theta;
        const blt_float_t lnprior[3] = {(blt_float_t)log1p_switch(-(3. * theta) / 2.), (blt_float_t)std::log(theta / 2.), (blt_float_t)std::log(theta)};
        for (unsigned ngt = 0; ngt < 3; ++ngt)
            for (unsigned tgt = 0; tgt < 2; ++tgt)
            {
                const unsigned combo = ngt * 2 + tgt;
                unsigned index = 0;
                for (unsigned tumor_freq_index = 0; tumor_freq_index < 21; ++tumor_freq_index)
                {
                    const blt_float_t tumor_freq = fraction_of(tumor_freq_index);
                    const bool consider_norm_contam = contam_tolerance * tumor_freq >= RATIO_INCREMENT;
                    for (unsigned normal_freq_index = 0; normal_freq_index < 21; ++normal_freq_index)
                    {
                        double lprior_freq = 0;
                        uint8_t kind = 0;
                        if (tgt == 0)
                        {
                            if (normal_freq_index != tumor_freq_index) continue;
                            kind = (normal_freq_index == ngt) ? 1 : 2;
                        }
                        else
                        {
                            if (normal_freq_index == tumor_freq_index) continue;
                            if (ngt != 0)
                            {
                                if (normal_freq_index != ngt) continue;
                                lprior_freq = log_error_mod;
                            }
                            else if (!consider_norm_contam)
                            {
                                if (normal_freq_index != 0) continue;
                                lprior_freq = log_error_mod;
                            }
                            else
                            {
                                if ((normal_freq_index != ngt) && (normal_freq_index != 3)) continue;
                                lprior_freq = log_error_mod + ln_one_half;
                            }
                        }
                        C.term_lprior[combo][index] = lprior_freq;
                        C.term_kind[combo][index] = kind;
                        C.term_tf[combo][index] = tumor_freq_index;
                        C.term_nf[combo][index] = normal_freq_index;
                        ++index;
                    }
                }
                C.n_terms[combo] = index;
                C.geno_prior[combo] = lnprior[ngt] + ((tgt == 0) ? ln_som_match : ln_som_mismatch);
            }
    }
    // lanes 0, 1: NOINDEL, HOM (no ratio); 2: HET at 0.5, defaults loghalf (starling_indel_call_pprob_digt.cpp:250,288-295);
    // 3 + i: lhood_low of het_ratio i, 20 - i: its lhood_high (somatic_indel_grid.cpp:80-89, starling_indel_call_pprob_digt.cpp:88-153)
    static const double loghalf(-std::log(2.));
    C.ratio[2] = 0.5;
    C.def_lr[2] = C.def_li[2] = loghalf;
    for (unsigned i = 0; i < 9; ++i)
    {
        const double het_ratio((i + 1) * RATIO_INCREMENT); // a float product, widened
        const double chet_ratio(1. - het_ratio);
        const double log_het_ratio(std::log(het_ratio)), log_chet_ratio(std::log(chet_ratio));
        C.ratio[3 + i] = het_ratio;
        C.def_lr[3 + i] = log_chet_ratio;
        C.def_li[3 + i] = log_het_ratio;
        C.ratio[20 - i] = chet_ratio;
        C.def_lr[20 - i] = log_het_ratio;
        C.def_li[20 - i] = log_chet_ratio;
    }
    C.correctMappingLogPrior = std::log(1.7e-10); // starling_base_shared.cpp:64
    C.randomBaseMatchLogProb[0] = std::log(o.randomBaseMatchProb);
    C.randomBaseMatchLogProb[1] = std::log(o.tier2RandomBaseMatchProb);
    for (unsigned n = 2; n <= 4; ++n) C.allele_lnprior[n] = std::log(1. / static_cast<double>(n));
    C.min_flank[0] = static_cast<uint32_t>(o.min_read_bp_flank[0]);
    C.min_flank[1] = static_cast<uint32_t>(o.min_read_bp_flank[1]);
    C.useTier2Evidence = o.useTier2Evidence ? 1 : 0;
}

// the shared-error terms of every table entry (somatic_indel_grid.cpp:273-275), as the float pair calculate_result_set_grid receives
void k5b_err_terms_of(const sx_sindel_opts& o, const double* err_prob, const uint32_t n_err, std::vector<float2>& out)
{
    out.resize(n_err);
    for (uint32_t i = 0; i < n_err; ++i)
    {
        const double sharedIndelErrorRate(std::pow(err_prob[i], o.shared_indel_error_factor));
        const double logSharedIndelErrorRate(std::log(sharedIndelErrorRate));
        const double logSharedIndelErrorRateComplement(log1p_switch(-sharedIndelErrorRate));
        out[i] = make_float2(static_cast<float>(logSharedIndelErrorRate), static_cast<float>(logSharedIndelErrorRateComplement));
    }
}
} // namespace

int sx_k5b_check(sx_ctx* ctx, const char* what, const sx_sindel_opts* o, const sx_sindel_batch* b, const double* err_prob, const uint32_t n_err, const void* out)
{
    if (!o || !b || !out) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL argument", what);
    if (o->min_read_bp_flank[0] < 0 || o->min_read_bp_flank[1] < 0) return sx_fail(ctx, SX_ERR_ARG, "%s: negative min_read_bp_flank", what);
    if (b->n_loci && (!err_prob || n_err == 0)) return sx_fail(ctx, SX_ERR_ARG, "%s: no error-rate table", what);
    if (b->n_loci && (!b->key || !b->is_forced_output || !b->err_idx || !b->alt_off || !b->read_off)) return sx_fail(ctx, SX_ERR_ARG, "%s: NULL batch array", what);
    return SX_OK;
}

// K5b's launcher: uploads the per-call constants and error terms (host staging slots 0 and 1) and launches
int sx_k5b_run(sx_ctx* ctx, const sx_sindel_opts* o, const sx_sindel_batch* d, const double* err_prob, const uint32_t n_err, sx_sindel_result* out_dev, unsigned* launches)
{
    static_assert(sizeof(k5b_consts) % 4 == 0, "k5b_consts is copied in words");
    k5b_consts C;
    k5b_consts_of(*o, C);
    std::vector<float2> et;
    k5b_err_terms_of(*o, err_prob, n_err, et);
    const k5b_consts* d_consts = nullptr;
    const float2* d_et = nullptr;
    int rc;
    if ((rc = sx_upload(ctx, sx_host_slot(0), &C, 1, d_consts, 0))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(1), et.data(), et.size(), d_et, 0))) return rc;
    // (C and et are pageable: cudaMemcpyAsync has staged them by the time it returns, so they may go out of scope here)
    const int grid = static_cast<int>(std::min<uint32_t>((d->n_loci + K5B_WARPS - 1) / K5B_WARPS, (uint32_t)ctx->sm_count * 8));
    k5b_somatic_indel_kernel<<<grid, K5B_WARPS * 32, 0, ctx->s_compute>>>(*d, d_consts, d_et, n_err, out_dev, ctx->d_status);
    SX_CUDA(ctx, cudaGetLastError());
    *launches += 1;
    return SX_OK;
}

extern "C" void sx_default_sindel_opts(sx_sindel_opts* o)
{
    memset(o, 0, sizeof(*o));
    o->somatic_indel_rate = 0.000001;     // applications/strelka/strelka_shared.hh:130
    o->bindel_diploid_theta = 0.0001;     // starling_common/starling_base_shared.hh:95
    o->indel_contam_tolerance = 0.15;     // strelka_shared.hh:151
    o->shared_indel_error_factor = 1.65;  // :142
    o->randomBaseMatchProb = 0.5;         // :74
    o->tier2RandomBaseMatchProb = 0.25;   // starling_common/Tier2Options.hh:49
    o->useTier2Evidence = 1;              // strelka_shared.hh:78
    o->min_read_bp_flank[0] = 1;          // normal_sample_min_read_bp_flank, strelka_shared.hh:159
    o->min_read_bp_flank[1] = 5;          // default_min_read_bp_flank, starling_base_shared.hh:108
}

extern "C" int sx_somatic_indel_dev(sx_ctx* ctx, const sx_sindel_opts* opts, const sx_sindel_batch* d, const double* err_prob_host, uint32_t n_err,
                                    sx_sindel_result* out_dev)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc = sx_k5b_check(ctx, "sx_somatic_indel_dev", opts, d, err_prob_host, n_err, out_dev);
    if (rc) return rc;
    if (d->n_loci == 0) return SX_OK;
    if ((rc = sx_run_timed(ctx, [&](unsigned* launches) { return sx_k5b_run(ctx, opts, d, err_prob_host, n_err, out_dev, launches); }))) return rc;
    return sx_check_status(ctx, "sx_somatic_indel_dev", SX_ST_SINDEL_ARG);
}

extern "C" int sx_somatic_indel(sx_ctx* ctx, const sx_sindel_opts* opts, const sx_sindel_batch* b, const double* err_prob_host, uint32_t n_err,
                                sx_sindel_result* out_host)
{
    if (!ctx) return SX_ERR_ARG;
    ctx->timing = sx_timing{};
    int rc = sx_k5b_check(ctx, "sx_somatic_indel", opts, b, err_prob_host, n_err, out_host);
    if (rc) return rc;
    if (b->n_loci == 0) return SX_OK;
    const size_t n_loci = b->n_loci, n_alts = b->alt_off[n_loci], n_reads = b->read_off[2 * n_loci];
    if ((n_alts && !b->alts) || (n_reads && !b->reads)) return sx_fail(ctx, SX_ERR_ARG, "sx_somatic_indel: NULL batch array");
    for (size_t l = 0; l < n_loci; ++l)
        if (b->err_idx[l] >= n_err) return sx_fail(ctx, SX_ERR_ARG, "sx_somatic_indel: locus %zu: error-rate index %u past the table (%u)", l, b->err_idx[l], n_err);
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    sx_call_timer t(ctx);
    sx_sindel_batch d = *b;
    if ((rc = sx_upload(ctx, sx_host_slot(2), b->key, n_loci, d.key, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(3), b->is_forced_output, n_loci, d.is_forced_output, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(4), b->err_idx, n_loci, d.err_idx, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(5), b->alt_off, n_loci + 1, d.alt_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(6), b->alts, n_alts, d.alts, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(7), b->read_off, 2 * n_loci + 1, d.read_off, 16))) return rc;
    if ((rc = sx_upload(ctx, sx_host_slot(8), b->reads, n_reads, d.reads, 16))) return rc;
    sx_sindel_result* d_out = nullptr;
    if ((rc = sx_take(ctx, sx_host_slot(9), n_loci, d_out, 0))) return rc;
    unsigned launches = 0;
    if ((rc = sx_k5b_run(ctx, opts, &d, err_prob_host, n_err, d_out, &launches))) return rc;
    if ((rc = sx_download(ctx, out_host, d_out, n_loci))) return rc;
    if ((rc = t.finish(launches))) return rc;
    return sx_check_status(ctx, "sx_somatic_indel", SX_ST_SINDEL_ARG);
}
