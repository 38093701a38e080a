// sx_context.cu -- ctx lifetime, host-computed tables, memory helpers, timing.
#include "sx_internal.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>

int sx_fail(sx_ctx* ctx, int code, const char* fmt, ...)
{
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf;
    else fprintf(stderr, "strelka_b200: %s\n", buf);
    return code;
}

// ABI layout pins (mirrored by strelka_b200/_abi.py and checked in tests/test_abi.py)
static_assert(sizeof(sx_aln_seg) == 4 && sizeof(sx_aln) == 16 && sizeof(sx_region) == 48, "K1 POD layout");
static_assert(sizeof(sx_ga_result) == 16 && sizeof(sx_ga_scores) == 32, "K3 POD layout");
static_assert(sizeof(sx_digt_result_set) == 24 && sizeof(sx_digt_result) == 152, "K2a POD layout");
static_assert(sizeof(sx_ssnv_result) == 288, "K2b POD layout");
static_assert(sizeof(sx_params) == 104, "sx_params layout");
static_assert(sizeof(sx_indel_result) == 152, "K5 POD layout");
static_assert(sizeof(sx_sindel_read) == 24 && sizeof(sx_sindel_opts) == 64 && sizeof(sx_sindel_tier) == 188 && sizeof(sx_sindel_result) == 400, "K5b POD layout");

static thread_local std::string g_create_err;

extern "C" const char* sx_last_error(const sx_ctx* ctx)
{
    return ctx ? ctx->err.c_str() : g_create_err.c_str();
}

extern "C" int sx_abi_version(void) { return SX_ABI_VERSION; }

extern "C" void sx_default_params(sx_params* p)
{
    memset(p, 0, sizeof(*p));
    p->bsnp_diploid_theta = 0.001;   // blt_common/blt_shared.hh:82
    p->bsnp_ssd_no_mismatch = 0.35;  // applications/starling/starling_shared.hh:34
    p->bsnp_ssd_one_mismatch = 0.6;  // :35
    p->is_min_vexp = 1;              // :38
    p->is_bsnp_diploid = 1;
    p->min_vexp = 0.25;              // :39
    p->hetVariantFrequencyExtension = 0;
    p->somatic_snv_rate = 0.0001;               // configureStrelkaSomaticWorkflow.py.ini (ssnvPrior)
    p->shared_site_error_rate = 0.0000000005;   // (ssnvNoise)
    p->shared_site_error_strand_bias_fraction = 0.0;
    p->ssnv_contam_tolerance = 0.15;
    p->pipeline_chunks = 0;
    p->min_read_bp_flank = 5;              // starling_common/starling_base_shared.hh:108
    p->randomBaseMatchProb = 0.25;         // :177
    p->readConfidentSupportThreshold = 0.51; // :245
}

extern "C" void sx_ga_active_region_scores(sx_ga_scores* s)
{
    // starling_common/ActiveRegionDetector.hh:62-66 + ctor starling_common/ActiveRegionDetector.cpp:41
    s->match = 1;
    s->mismatch = -4;
    s->open = -5;
    s->extend = -1;
    s->offEdge = -100;
    s->insertDelete = -5;
    s->isAllowEdgeInsertion = 1;
    s->isRequireEdgeDeletion = 1;
}

// --------------------------------------------------------------------------------------------------------------
// tables.  Expression shapes follow the reference literally (including float/double mixing), see sx_internal.h.
// This translation unit is compiled with -fmad=false equivalents on the host side: nvcc passes it to g++ with
// -ffp-contract=off (Makefile), so no host FMA contraction can change a table value.
// --------------------------------------------------------------------------------------------------------------
double log1p_switch(const double x) // blt_util/math_util.hh:33-47 (boost::math::log1p<double> == ::log1p with glibc)
{
    if (std::abs(x) < 0.01) return ::log1p(x);
    return std::log(1 + x);
}

namespace
{
typedef float blt_float_t;

inline double digt_expect(const int base_id, const int gt) // blt_util/digt.hh:94-113
{
    static const double ex[10][4] = {{1.0, 0.0, 0.0, 0.0}, {0.0, 1.0, 0.0, 0.0}, {0.0, 0.0, 1.0, 0.0}, {0.0, 0.0, 0.0, 1.0}, {0.5, 0.5, 0.0, 0.0},
                                     {0.5, 0.0, 0.5, 0.0}, {0.5, 0.0, 0.0, 0.5}, {0.0, 0.5, 0.5, 0.0}, {0.0, 0.5, 0.0, 0.5}, {0.0, 0.0, 0.5, 0.5}};
    return ex[gt][base_id];
}

void fill_priors(const blt_float_t theta, float out[2][5][2][10]) // position_snp_call_pprob_digt.cpp:50-248
{
    const blt_float_t one_third(1. / 3.);
    blt_float_t pr[2][5][2][10];
    memset(pr, 0, sizeof(pr));
    for (unsigned ref_gt = 0; ref_gt < 4; ++ref_gt)
    {
        {
            blt_float_t* prior = pr[0][ref_gt][0]; // get_genomic_prior
            blt_float_t prior_sum(0.);
            for (unsigned gt(0); gt < 10; ++gt)
            {
                if (gt == ref_gt) continue;
                prior[gt] = (theta * one_third);
                if (gt >= 4)
                {
                    if (digt_expect(ref_gt, gt) <= 0.) prior[gt] *= theta;
                }
                else
                {
                    prior[gt] *= .5;
                }
                prior_sum += prior[gt];
            }
            prior[ref_gt] = (1. - prior_sum);
        }
        {
            blt_float_t* prior = pr[0][ref_gt][1]; // get_poly_prior
            const blt_float_t ctheta(1. - theta);
            for (unsigned gt(0); gt < 10; ++gt)
            {
                if (gt == ref_gt) prior[gt] = 0.25 * (ctheta);
                else if (gt >= 4)
                {
                    if (digt_expect(ref_gt, gt) <= 0.) prior[gt] = theta * one_third;
                    else prior[gt] = 0.5 * one_third * ctheta;
                }
                else prior[gt] = 0.25 * one_third * ctheta;
            }
        }
        {
            blt_float_t* prior = pr[1][ref_gt][0]; // get_haploid_genomic_prior
            blt_float_t prior_sum(0.);
            for (unsigned gt(0); gt < 10; ++gt)
            {
                if (gt == ref_gt) continue;
                if (gt >= 4) prior[gt] = 0;
                else prior[gt] = (theta * one_third);
                prior_sum += prior[gt];
            }
            prior[ref_gt] = (1. - prior_sum);
        }
        {
            blt_float_t* prior = pr[1][ref_gt][1]; // get_haploid_poly_prior
            for (unsigned gt(0); gt < 10; ++gt)
            {
                if (gt == ref_gt) prior[gt] = 0.5;
                else if (gt >= 4) prior[gt] = 0;
                else prior[gt] = 0.5 * one_third;
            }
        }
    }
    for (int h = 0; h < 2; ++h) // finish_prior
    {
        for (int k = 0; k < 2; ++k)
        {
            blt_float_t* nps = pr[h][4][k];
            for (unsigned i(0); i < 4; ++i)
                for (unsigned gt(0); gt < 10; ++gt) nps[gt] += pr[h][i][k][gt];
        }
        for (int k = 0; k < 2; ++k)
        {
            blt_float_t* x = pr[h][4][k];
            blt_float_t sum(0);
            for (unsigned gt(0); gt < 10; ++gt) sum += x[gt];
            sum = 1. / sum;
            for (unsigned gt(0); gt < 10; ++gt) x[gt] *= sum;
        }
        for (unsigned i(0); i < 5; ++i)
            for (int k = 0; k < 2; ++k)
                for (unsigned gt(0); gt < 10; ++gt) out[h][i][k][gt] = std::log(pr[h][i][k][gt]);
    }
}

blt_float_t get_dependent_eprob(const double q2p, const blt_float_t vexp) // adjust_joint_eprob.cpp:60-70
{
    static const blt_float_t dep_converge_prob(0.75);
    const blt_float_t eprob(q2p);
    const blt_float_t val(std::pow(eprob, vexp));
    const blt_float_t frac((1 - val) / (1 - eprob));
    return std::max(eprob, frac * val + (1 - frac) * dep_converge_prob);
}

void build_tables(const sx_params& p, sx_tables& t)
{
    memset(&t, 0, sizeof(t));
    double q2p[SX_MAX_QSCORE + 1], q2lncompe[SX_MAX_QSCORE + 1], q2lne[SX_MAX_QSCORE + 1];
    {
        static const double q2lnp(-std::log(10.) / 10.); // qscore_cache.cpp:36
        for (int i(0); i <= SX_MAX_QSCORE; ++i)
        {
            q2p[i] = std::pow(10., -static_cast<double>(i) / 10.); // phred_to_error_prob, qscore.hh:76-80
            q2lncompe[i] = log1p_switch(-q2p[i]);
            q2lne[i] = static_cast<double>(i) * q2lnp;
        }
    }
    // K1: starling_read_align_score.cpp:118-135 (terms), :453 (soft clip), :483 (non-candidate penalty)
    {
        static const double lnthird(-std::log(3.));
        for (int q = 0; q <= SX_MAX_QSCORE; ++q)
        {
            t.k1_tab[2 * q + 0] = q2lne[q] + lnthird;
            t.k1_tab[2 * q + 1] = q2lncompe[q];
            t.k1_tab[2 * (SX_K1_ROW_EQ + q) + 0] = q2lncompe[q];
            t.k1_tab[2 * (SX_K1_ROW_EQ + q) + 1] = q2lncompe[q];
        }
        t.k1_tab[2 * SX_K1_ROW_ZERO + 0] = 0.0;
        t.k1_tab[2 * SX_K1_ROW_ZERO + 1] = 0.0;
        t.k1_softclip = std::log(0.25);
        t.k1_noncand = std::log(1e-5);
    }
    // K4: mappedq[j][i] = error_prob_to_qphred(phred_to_mapped_error_prob(i, j))  (qscore_cache.cpp:44-47, qscore.hh:40-63,107-113)
    {
        static const double minlog10(static_cast<double>(std::numeric_limits<double>::min_exponent10));
        for (int i(0); i <= SX_MAX_QSCORE; ++i)
            for (int j(0); j <= 90; ++j)
            {
                const double be(std::pow(10., -static_cast<double>(i) / 10.));
                const double me(std::pow(10., -static_cast<double>(j) / 10.));
                const double prob(((1. - me) * be) + (me * 0.75));
                t.mappedq[j][i] = static_cast<uint8_t>(static_cast<int>(std::floor(-10. * std::max(minlog10, std::log10(prob)) + 0.5)));
            }
    }
    // germline: position_snp_call_pprob_digt.cpp:40-43,343-355 ; adjust_joint_eprob.cpp:112-121
    {
        const blt_float_t one_third(1. / 3.);
        const blt_float_t log_one_third(std::log(one_third));
        const blt_float_t one_half(1. / 2.);
        const blt_float_t log_one_half(std::log(one_half));
        static const blt_float_t lnran(std::log(0.75));
        for (int q = 0; q <= SX_MAX_QSCORE; ++q)
        {
            t.g_eprob[q] = static_cast<float>(q2p[q]);
            const blt_float_t ceprob(1. - q2p[q]);
            t.g_val1[q] = std::log((ceprob) + ((1. - ceprob) * one_third)) + log_one_half;
            t.g_val2[q] = q2lncompe[q];
            const blt_float_t weight(lnran - q2lne[q]);
            t.g_weight[q] = weight;
            t.g_depmin[q] = get_dependent_eprob(q2p[q], static_cast<blt_float_t>(p.min_vexp));
        }
        t.g_log_one_third = log_one_third;
        t.g_ln10f = std::log(static_cast<blt_float_t>(10));
        t.g_min_vexp = static_cast<blt_float_t>(p.min_vexp);
        t.g_ssd_no_mismatch = p.bsnp_ssd_no_mismatch;
        t.g_ssd_one_mismatch = p.bsnp_ssd_one_mismatch;
        t.g_is_dependent_eprob = (p.is_bsnp_diploid && (p.bsnp_ssd_no_mismatch > 0. || p.bsnp_ssd_one_mismatch > 0)) ? 1 : 0; // blt_shared.hh:76-81
        t.g_is_min_vexp = p.is_min_vexp ? 1 : 0;
        fill_priors(static_cast<blt_float_t>(p.bsnp_diploid_theta), t.g_lnprior);
    }
    // indel genotype model: starling_base_shared.cpp:44,66 ; AlleleGroupGenotype.cpp:76-77
    {
        t.i_randomBaseMatchLogProb = std::log(p.randomBaseMatchProb);
        t.i_correctMappingLogPrior = std::log(1.7e-10);
        t.i_loghalf = std::log(0.5);
        t.i_readSupportThreshold = p.readConfidentSupportThreshold;
        t.i_min_flank = p.min_read_bp_flank;
    }
    // somatic: position_somatic_snv_strand_grid_lhood_cached.cpp ; position_somatic_snv_strand_grid.cpp:42-55 ; qscore_calculator.cpp:33-60
    {
        static const blt_float_t one_third(1. / 3.);
        static const blt_float_t ln_one_third(std::log(one_third));
        static const blt_float_t one_half(1. / 2.);
        static const blt_float_t ln_one_half(std::log(one_half));
        const blt_float_t RATIO_INCREMENT = 0.5f / static_cast<blt_float_t>(9 + 1);
        for (int q = 0; q <= SX_MAX_QSCORE; ++q)
        {
            {
                const blt_float_t eprob(q2p[q]);
                const blt_float_t ceprob(1 - eprob);
                const blt_float_t lne(q2lne[q]);
                const blt_float_t lnce(q2lncompe[q]);
                t.s_simple[q][0] = lne + ln_one_third;
                t.s_simple[q][1] = std::log((ceprob) + ((eprob)*one_third)) + ln_one_half;
                t.s_simple[q][2] = lnce;
            }
            for (unsigned hetIndex = 0; hetIndex < 9; ++hetIndex)
            {
                const blt_float_t het_ratio((hetIndex + 1) * RATIO_INCREMENT);
                {
                    const blt_float_t chet_ratio(1. - het_ratio);
                    const blt_float_t eprob(q2p[q]);
                    const blt_float_t ceprob(1 - eprob);
                    t.s_het[hetIndex][q][0] = std::log((ceprob)*het_ratio + ((eprob)*one_third) * chet_ratio);
                    t.s_het[hetIndex][q][1] = std::log((ceprob)*chet_ratio + ((eprob)*one_third) * het_ratio);
                }
                {
                    const blt_float_t chet_ratio(1. - het_ratio);
                    const blt_float_t eprob(q2p[q]);
                    const blt_float_t ceprob(1. - eprob);
                    t.s_strand[hetIndex][q][0] = (std::log((ceprob)*chet_ratio + ((eprob)*one_third) * het_ratio));
                    t.s_strand[hetIndex][q][1] = (std::log((ceprob)*het_ratio + ((eprob)*one_third) * chet_ratio));
                }
            }
            {
                const blt_float_t val_off_ref(q2lncompe[q]);
                const blt_float_t val_off_alt(q2lne[q] + ln_one_third);
                t.s_off_ref[q] = val_off_ref;
                t.s_off_alt[q] = val_off_alt;
            }
        }
        const double theta(p.bsnp_diploid_theta);
        t.s_lnprior[0] = (blt_float_t)log1p_switch(-(3. * theta) / 2.);
        t.s_lnprior[1] = (blt_float_t)std::log(theta / 2.);
        t.s_lnprior[2] = (blt_float_t)std::log(theta);
        t.s_contam_tolerance = static_cast<blt_float_t>(p.ssnv_contam_tolerance);
        t.s_ln_csse_rate = static_cast<blt_float_t>(log1p_switch(-p.shared_site_error_rate));
        t.s_ln_som_match = static_cast<blt_float_t>(log1p_switch(-p.somatic_snv_rate));
        t.s_ln_som_mismatch = static_cast<blt_float_t>(std::log(p.somatic_snv_rate));
        const blt_float_t strand_sse_rate(p.shared_site_error_rate * p.shared_site_error_strand_bias_fraction);
        const blt_float_t nostrand_sse_rate(p.shared_site_error_rate - strand_sse_rate);
        t.s_ln_sse_rate = std::log(nostrand_sse_rate);
        t.s_ln_one_half = static_cast<blt_float_t>(std::log(1. / 2.));
        t.s_log_error_mod = static_cast<blt_float_t>(-std::log(static_cast<double>(21 - 1)));
        t.s_ratio_increment = RATIO_INCREMENT;

        // unroll the double loop of calculate_result_set_grid (qscore_calculator.cpp:63-123) into ordered term lists
        {
            const blt_float_t contam_tolerance(t.s_contam_tolerance);
            const blt_float_t logSharedErrorRate(t.s_ln_sse_rate), logSharedErrorRateComplement(t.s_ln_csse_rate);
            static const blt_float_t grid_ln_one_half(std::log(1. / 2.));
            static const blt_float_t log_error_mod = -std::log(static_cast<double>(21 - 1));
            auto fraction_of = [&](int index) -> blt_float_t { // strelka_digt_states.cpp:34-41
                if (index == 0) return 0.f;
                if (index == 1) return 1.f;
                if (index == 2) return 0.5f;
                if (index < 3 + 9) return RATIO_INCREMENT * (index - 3 + 1);
                return RATIO_INCREMENT * (index - 3 + 2);
            };
            for (unsigned ngt(0); ngt < 3; ++ngt)
                for (unsigned tgt(0); tgt < 2; ++tgt)
                {
                    const unsigned combo(ngt * 2 + tgt);
                    unsigned index(0);
                    for (unsigned tumor_freq_index(0); tumor_freq_index < 21; ++tumor_freq_index)
                    {
                        blt_float_t tumor_freq = fraction_of(tumor_freq_index);
                        bool consider_norm_contam = contam_tolerance * tumor_freq >= RATIO_INCREMENT;
                        for (unsigned normal_freq_index(0); normal_freq_index < 21; ++normal_freq_index)
                        {
                            double lprior_freq;
                            if (tgt == 0)
                            {
                                if (normal_freq_index != tumor_freq_index) continue;
                                lprior_freq = (normal_freq_index == ngt) ? logSharedErrorRateComplement : logSharedErrorRate + log_error_mod;
                            }
                            else
                            {
                                if (normal_freq_index == tumor_freq_index) continue;
                                if (ngt != 0)
                                {
                                    if (normal_freq_index != ngt) continue;
                                    lprior_freq = log_error_mod;
                                }
                                else
                                {
                                    if (!consider_norm_contam)
                                    {
                                        if (normal_freq_index == 0) lprior_freq = log_error_mod;
                                        else continue;
                                    }
                                    else
                                    {
                                        if ((normal_freq_index == ngt) || (normal_freq_index == 3)) lprior_freq = log_error_mod + grid_ln_one_half;
                                        else continue;
                                    }
                                }
                            }
                            t.s_term_lprior[combo][index] = lprior_freq;
                            t.s_term_tf[combo][index] = tumor_freq_index;
                            t.s_term_nf[combo][index] = normal_freq_index;
                            ++index;
                        }
                    }
                    t.s_n_terms[combo] = index;
                    t.s_geno_prior[combo] = t.s_lnprior[ngt] + ((tgt == 0) ? t.s_ln_som_match : t.s_ln_som_mismatch);
                }
        }
    }
}
} // namespace

extern "C" int sx_set_host_wait_policy(int cuda_device, int blocking)
{
    cudaError_t e = cudaSetDevice(cuda_device);
    if (e == cudaSuccess) e = cudaSetDeviceFlags(blocking ? cudaDeviceScheduleBlockingSync : cudaDeviceScheduleAuto);
    if (e != cudaSuccess)
    {
        g_create_err = std::string("sx_set_host_wait_policy: ") + cudaGetErrorString(e);
        (void)cudaGetLastError();
        return SX_ERR_CUDA;
    }
    return SX_OK;
}

extern "C" int sx_create(int cuda_device, const sx_params* p, sx_ctx** out)
{
    if (!p || !out)
    {
        g_create_err = "sx_create: NULL argument";
        return SX_ERR_ARG;
    }
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
    {
        g_create_err = std::string("sx_create: no usable CUDA device (") + cudaGetErrorString(e) + "); strelka_b200 has no CPU fallback";
        return SX_ERR_CUDA;
    }
    if (cuda_device < 0 || cuda_device >= ndev)
    {
        g_create_err = "sx_create: cuda_device out of range";
        return SX_ERR_ARG;
    }
    if (p->hetVariantFrequencyExtension > 0)
    {
        g_create_err = "sx_create: hetVariantFrequencyExtension > 0 (RNA het-extension model, increment_het_ratio_lhood) is outside the accelerated path";
        return SX_ERR_UNSUPPORTED;
    }
    sx_ctx* ctx = new sx_ctx();
    ctx->device = cuda_device;
    ctx->params = *p;
    auto bail = [&](const char* what, cudaError_t ce) {
        g_create_err = std::string("sx_create: ") + what + ": " + cudaGetErrorString(ce);
        sx_destroy(ctx); // releases whatever was created so far (streams, events, tables)
        return SX_ERR_CUDA;
    };
    if ((e = cudaSetDevice(cuda_device)) != cudaSuccess) return bail("cudaSetDevice", e);
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, cuda_device)) != cudaSuccess) return bail("cudaGetDeviceProperties", e);
    if (prop.major != 9 || prop.minor != 0) // sm_90a code loads on compute capability 9.0 only
    {
        g_create_err = "sx_create: this library is built for sm_90a (H100) only";
        sx_destroy(ctx);
        return SX_ERR_CUDA;
    }
    ctx->sm_count = prop.multiProcessorCount;
    ctx->smem_optin = prop.sharedMemPerBlockOptin;
    if ((e = cudaStreamCreateWithFlags(&ctx->s_compute, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
    if ((e = cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
    if ((e = cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking)) != cudaSuccess) return bail("cudaStreamCreate", e);
    cudaEventCreate(&ctx->ev_a);
    cudaEventCreate(&ctx->ev_b);
    build_tables(*p, ctx->tables);
    if ((e = cudaMalloc(&ctx->d_tables, sizeof(sx_tables))) != cudaSuccess) return bail("cudaMalloc", e);
    if ((e = cudaMemcpy(ctx->d_tables, &ctx->tables, sizeof(sx_tables), cudaMemcpyHostToDevice)) != cudaSuccess) return bail("cudaMemcpy", e);
    if ((e = sx_k2a_init_tables(ctx->d_tables)) != cudaSuccess) return bail("K2a tables", e);
    if ((e = cudaMemcpy(&ctx->tables, ctx->d_tables, sizeof(sx_tables), cudaMemcpyDeviceToHost)) != cudaSuccess) return bail("cudaMemcpy", e);
    if ((e = cudaMalloc(&ctx->d_status, sizeof(int))) != cudaSuccess) return bail("cudaMalloc", e);
    cudaMemset(ctx->d_status, 0, sizeof(int));
    *out = ctx;
    return SX_OK;
}

extern "C" void sx_destroy(sx_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    sx_comm_release(ctx);
    for (auto& b : ctx->buf)
        if (b.p) cudaFree(b.p);
    if (ctx->d_tables) cudaFree(ctx->d_tables);
    if (ctx->d_status) cudaFree(ctx->d_status);
    for (auto ev : ctx->ev_pool) cudaEventDestroy(ev);
    for (auto& ev : ctx->ev_win)
        if (ev) cudaEventDestroy(ev);
    for (auto& ev : ctx->ev_swin)
        if (ev) cudaEventDestroy(ev);
    for (auto& ev : ctx->ev_user)
        if (ev) cudaEventDestroy(ev);
    if (ctx->ev_a) cudaEventDestroy(ctx->ev_a);
    if (ctx->ev_b) cudaEventDestroy(ctx->ev_b);
    if (ctx->s_compute) cudaStreamDestroy(ctx->s_compute);
    if (ctx->s_h2d) cudaStreamDestroy(ctx->s_h2d);
    if (ctx->s_d2h) cudaStreamDestroy(ctx->s_d2h);
    delete ctx;
}

int sx_ensure(sx_ctx* ctx, sx_slot slot, size_t bytes, void** out)
{
    if (slot < 0 || slot >= SX_SLOT_COUNT) return sx_fail(ctx, SX_ERR_ARG, "device buffer slot %d outside the context's %d", (int)slot, (int)SX_SLOT_COUNT);
    sx_buf& b = ctx->buf[slot];
    if (b.cap < bytes)
    {
        if (b.p) cudaFree(b.p);
        b.p = nullptr;
        b.cap = 0;
        const size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&b.p, want);
        if (e != cudaSuccess)
        {
            cudaGetLastError();
            return sx_fail(ctx, SX_ERR_NOMEM, "cudaMalloc(%zu) failed: %s", want, cudaGetErrorString(e));
        }
        b.cap = want;
    }
    *out = b.p;
    return SX_OK;
}

#define SX_STR_(x) #x
#define SX_STR(x) SX_STR_(x)
namespace
{
// every status bit with its error.  A capacity bit has a second message that quotes the stage's first n_totals totals.
struct sx_status_entry
{
    int bit, code;
    const char* msg;
    const char* msg_totals;
    int n_totals;
};
constexpr sx_status_entry k_status[] = {
    {SX_ST_QUAL, SX_ERR_RANGE, "%s: quality score above " SX_STR(SX_MAX_QSCORE) " (qphred_cache::qscore_check would throw)", nullptr, 0},
    {SX_ST_TILE, SX_ERR_ARG, "%s: a region does not fit the shared-memory tile the kernel was launched with", nullptr, 0},
    {SX_ST_SEG_KIND, SX_ERR_ARG, "%s: unknown segment kind", nullptr, 0},
    {SX_ST_READ_OVERRUN, SX_ERR_ARG, "%s: alignment path consumes more read bases than the read holds", nullptr, 0},
    {SX_ST_SITE_DEPTH, SX_ERR_UNSUPPORTED, "%s: a site holds more calls than the kernel handles", nullptr, 0},
    {SX_ST_INDEL_ALLELES, SX_ERR_ARG, "%s: allele count outside 1.." SX_STR(SX_INDEL_MAX_ALLELES) " or ploidy outside {1,2}", nullptr, 0},
    {SX_ST_READ_ORDER, SX_ERR_ARG, "%s: reads are not in position order, or an alignment spans more reference than max_ref_span", nullptr, 0},
    {SX_ST_BASE, SX_ERR_ARG, "%s: unknown base code (bam_seq_code_to_id would throw)", nullptr, 0},
    {SX_ST_READ_LIMIT, SX_ERR_UNSUPPORTED, "%s: a read is longer, or has more path segments, than the kernel handles", nullptr, 0},
    {SX_ST_K6_SEG_KIND, SX_ERR_UNSUPPORTED, "%s: a path segment kind outside score_indels' domain (SKIP / REFSKIP / unknown)", nullptr, 0},
    {SX_ST_K6_ALNS, SX_ERR_ARG, "%s: a read has more alignments than the scratch was sized for", nullptr, 0},
    {SX_ST_K6_EVAL, SX_ERR_UNSUPPORTED, "%s: a read evaluates more than 64 indels", nullptr, 0},
    {SX_ST_K6_REC_CAP, SX_ERR_NOMEM, "%s: rec_off leaves too few record slots for a read", nullptr, 0},
    {SX_ST_K6_KEY, SX_ERR_ARG, "%s: an alignment key index outside its region's window, or an unsupported key type", nullptr, 0},
    {SX_ST_K8_NO_KEY, SX_ERR_ARG, "%s: a path gap matches no indel key of its alignment (getMatchingIndelKey would assert)", nullptr, 0},
    {SX_ST_K8_KIND, SX_ERR_ARG, "%s: can't handle cigar code", nullptr, 0},
    {SX_ST_K8_CAP, SX_ERR_CAPACITY, "%s: output capacity too small (totals[] holds the needed sizes)", "%s: output capacity too small: %u segments, %u insert bytes needed", 2},
    {SX_ST_K7_CAP, SX_ERR_CAPACITY, "%s: output capacity too small (totals[] holds the needed sizes)",
     "%s: output capacity too small: the batch produces %u alignments, %u segments, %u keys", 3},
    {SX_ST_K7A_CAP, SX_ERR_CAPACITY, "%s: cap_keys too small (totals[0] holds the needed size)", "%s: cap_keys too small: %u keys needed", 1},
    {SX_ST_K9_CAP, SX_ERR_CAPACITY, "%s: cap_segs too small (totals[0] holds the needed size)", "%s: cap_segs too small: %u segment slots needed", 1},
    {SX_ST_SINDEL_CAP, SX_ERR_CAPACITY, "%s: a locus over the alternate-allele caps", nullptr, 0}, // (per-locus status only; listed for the disjointness check)
    {SX_ST_SINDEL_ARG, SX_ERR_ARG, "%s: a candidate indel that is not of type INDEL, or an error-rate index past the table", nullptr, 0},
    {SX_ST_INDEL_READS_DUP, SX_ERR_ARG, "%s: a read id twice in one locus's list", nullptr, 0}, // (per-locus status only; listed for the disjointness check)
    {SX_ST_K6B_ID, SX_ERR_ARG, "%s: a record's window index outside its region's window, or an indel id at or past n_gid", nullptr, 0},
    {SX_ST_K6G_GROUP, SX_ERR_ARG, "%s: an allele group with an allele count outside 1.." SX_STR(SX_INDEL_MAX_ALLELES)
                                  ", a ploidy outside {1,2}, an id at or past n_gid, or offsets that do not start at 0 and ascend", nullptr, 0},
};

constexpr bool status_bits_disjoint()
{
    int seen = 0;
    for (const sx_status_entry& e : k_status)
    {
        if (e.bit <= 0 || (e.bit & (e.bit - 1)) || (seen & e.bit)) return false;
        seen |= e.bit;
    }
    return true;
}
static_assert(status_bits_disjoint(), "every status bit is one bit, and no two overlap");
} // namespace

int sx_check_status(sx_ctx* ctx, const char* what, int first, const uint32_t* totals)
{
    int st = 0;
    SX_CUDA(ctx, cudaMemcpyAsync(&st, ctx->d_status, sizeof(int), cudaMemcpyDeviceToHost, ctx->s_compute));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    if (st == 0) return SX_OK;
    cudaMemsetAsync(ctx->d_status, 0, sizeof(int), ctx->s_compute);
    for (const int pass_first : {1, 0})
        for (const sx_status_entry& e : k_status)
        {
            if (!(st & e.bit) || ((first & e.bit) != 0) != (pass_first != 0)) continue;
            if (!totals || !e.msg_totals || !(first & e.bit)) return sx_fail(ctx, e.code, e.msg, what); // (the totals are the caller's stage's)
            if (e.n_totals == 1) return sx_fail(ctx, e.code, e.msg_totals, what, totals[0]);
            if (e.n_totals == 2) return sx_fail(ctx, e.code, e.msg_totals, what, totals[0], totals[1]);
            return sx_fail(ctx, e.code, e.msg_totals, what, totals[0], totals[1], totals[2]);
        }
    return sx_fail(ctx, SX_ERR_ARG, "%s: device status %d", what, st);
}

extern "C" void* sx_host_alloc(size_t bytes)
{
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess)
    {
        cudaGetLastError();
        return nullptr;
    }
    return p;
}
extern "C" void sx_host_free(void* p)
{
    if (p) cudaFreeHost(p);
}
extern "C" void* sx_dev_alloc(sx_ctx* ctx, size_t bytes)
{
    void* p = nullptr;
    cudaSetDevice(ctx->device);
    if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess)
    {
        cudaGetLastError();
        sx_fail(ctx, SX_ERR_NOMEM, "cudaMalloc(%zu) failed", bytes);
        return nullptr;
    }
    return p;
}
extern "C" void sx_dev_free(sx_ctx* ctx, void* p)
{
    if (p)
    {
        cudaSetDevice(ctx->device);
        cudaFree(p);
    }
}
extern "C" int sx_memcpy_h2d(sx_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes)
{
    SX_CUDA(ctx, cudaMemcpyAsync(dst_dev, src_host, bytes, cudaMemcpyHostToDevice, ctx->s_compute));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    return SX_OK;
}
extern "C" int sx_memcpy_d2h(sx_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes)
{
    SX_CUDA(ctx, cudaMemcpyAsync(dst_host, src_dev, bytes, cudaMemcpyDeviceToHost, ctx->s_compute));
    SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
    return SX_OK;
}
extern "C" int sx_memcpy_d2d(sx_ctx* ctx, void* dst_dev, const void* src_dev, size_t bytes)
{
    if (!ctx) return SX_ERR_ARG;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    SX_CUDA(ctx, cudaMemcpyAsync(dst_dev, src_dev, bytes, cudaMemcpyDeviceToDevice, ctx->s_compute));
    return SX_OK;
}

// Two marks on the compute stream and the device time between them: how a caller times a run of entry points on the device instead of by the
// host clock (bench.py's timed region).
extern "C" int sx_timer_mark(sx_ctx* ctx, int which)
{
    if (!ctx || which < 0 || which > 1) return SX_ERR_ARG;
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!ctx->ev_user[which]) SX_CUDA(ctx, cudaEventCreate(&ctx->ev_user[which]));
    SX_CUDA(ctx, cudaEventRecord(ctx->ev_user[which], ctx->s_compute));
    return SX_OK;
}
extern "C" int sx_stream_join(sx_ctx* waiter, sx_ctx* other)
{
    if (!waiter || !other) return SX_ERR_ARG;
    if (waiter == other) return SX_OK;
    if (waiter->device != other->device) return sx_fail(waiter, SX_ERR_ARG, "sx_stream_join: the two contexts are on different devices");
    SX_CUDA(waiter, cudaSetDevice(waiter->device));
    cudaEvent_t ev;
    SX_CUDA(waiter, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    cudaError_t e = cudaEventRecord(ev, other->s_compute);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(waiter->s_compute, ev, 0);
    cudaEventDestroy(ev); // (released when the wait has been satisfied)
    SX_CUDA(waiter, e);
    return SX_OK;
}
extern "C" int sx_timer_elapsed_ms(sx_ctx* ctx, double* ms)
{
    if (!ctx || !ms) return SX_ERR_ARG;
    if (!ctx->ev_user[0] || !ctx->ev_user[1]) return sx_fail(ctx, SX_ERR_ARG, "sx_timer_elapsed_ms: both marks must have been set (sx_timer_mark 0 and 1)");
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    SX_CUDA(ctx, cudaEventSynchronize(ctx->ev_user[1]));
    float f = 0.f;
    SX_CUDA(ctx, cudaEventElapsedTime(&f, ctx->ev_user[0], ctx->ev_user[1]));
    *ms = f;
    return SX_OK;
}

extern "C" int sx_synchronize(sx_ctx* ctx)
{
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    SX_CUDA(ctx, cudaDeviceSynchronize());
    return SX_OK;
}
extern "C" int sx_last_timing(const sx_ctx* ctx, sx_timing* out)
{
    if (!ctx || !out) return SX_ERR_ARG;
    *out = ctx->timing;
    return SX_OK;
}
extern "C" uint64_t sx_total_launches(const sx_ctx* ctx) { return ctx ? ctx->total_launches : 0; }
