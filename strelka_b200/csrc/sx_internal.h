// sx_internal.h -- shared declarations of libstrelka_b200.so (not part of the ABI)
#pragma once

#include "strelka_b200.h"

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <string>
#include <vector>

#define SX_MAX_QSCORE 70

// ---------------------------------------------------------------------------------------------------------------
// host-computed tables (sx_create): every value the reference derives from an option or a quality score alone.
// They are evaluated with the HOST libm in exactly the reference's expression shapes, so that on a given machine
// they are bit-identical to what the reference process would hold in its own caches:
//   qphred_cache          blt_util/qscore_cache.cpp:33-49
//   het_ratio_cache       strelka_common/het_ratio_cache.hh (values: position_somatic_snv_strand_grid_lhood_cached.cpp)
//   dependent_prob_cache  blt_common/adjust_joint_eprob.cpp:75-88
//   pprob_digt_caller priors  blt_common/position_snp_call_pprob_digt.cpp:50-248
// ---------------------------------------------------------------------------------------------------------------
#define SX_K1_ROWS 143           /* 0..70: (mismatch, match) of q; 71..141: '=' read base (match, match); 142: 'N' read base (0, 0) */
#define SX_K1_ROW_EQ 71
#define SX_K1_ROW_ZERO 142

struct sx_tables
{
    // K1
    double k1_tab[SX_K1_ROWS * 2];  // [row][0] mismatch term q2lne+ln(1/3), [row][1] match term q2lncompe
    double k1_softclip;             // ln(0.25)
    double k1_noncand;              // ln(1e-5)
    // K4: qphred_cache::mappedq[mapq 0..90][basecall q 0..70] (blt_util/qscore_cache.cpp:44-47)
    uint8_t mappedq[91][SX_MAX_QSCORE + 1];
    // germline site model
    float g_eprob[SX_MAX_QSCORE + 1];     // (float) q2p
    float g_val1[SX_MAX_QSCORE + 1];      // (float)( log(ceprob + (1-ceprob)/3) + ln 1/2 )
    float g_val2[SX_MAX_QSCORE + 1];      // (float) q2lncompe
    float g_weight[SX_MAX_QSCORE + 1];    // (float)( ln(0.75)f - q2lne )
    float g_depmin[SX_MAX_QSCORE + 1];    // get_dependent_eprob(q, min_vexp)
    float g_lnprior[2][5][2][10];         // [haploid][ref base incl N][genome,poly][gt]
    float g_log_one_third, g_min_vexp;
    double g_ssd_no_mismatch, g_ssd_one_mismatch;
    int g_is_dependent_eprob, g_is_min_vexp;
    // val0 = logf(de) + ln(1/3) of a call (position_snp_call_pprob_digt.cpp:352) wherever de is a function of q alone.  Filled on the
    // device right after the upload (sx_k2a_init_tables, k2a_germline.cu) with the kernel's own device functions:
    //   g_val0_plain[q]     de = eprob[q]                (q < 3, or no dependent error model)
    //   g_val0_min[q]       de = depmin[q]               (ranks at or past the exponent clamp)
    //   g_val0_clean[k][q]  de = dependent_eprob(eprob[q], vexp_k), k < g_clean_ranks, in a group without a neighbour-mismatch call
    //                       (its vexp_frac is (float)bsnp_ssd_no_mismatch, so the exponents vexp_k are the same in every such group)
    // g_clean_ok: the clean-group rows apply (dependent model on, exponent clamp on, clamp reached within SX_K2_CLEAN_RANKS ranks).
#define SX_K2_CLEAN_RANKS 8
    float g_val0_plain[SX_MAX_QSCORE + 1], g_val0_min[SX_MAX_QSCORE + 1];
    float g_val0_clean[SX_K2_CLEAN_RANKS][SX_MAX_QSCORE + 1];
    int g_clean_ranks, g_clean_ok;
    // somatic site model
    float s_simple[SX_MAX_QSCORE + 1][3];     // val[0..2] of get_diploid_gt_lhood_cached_simple
    float s_het[9][SX_MAX_QSCORE + 1][2];     // val[0..1] of get_high_low_het_ratio_lhood_cached for ratio index 0..8
    float s_strand[9][SX_MAX_QSCORE + 1][2];  // val[0..1] of get_strand_ratio_lhood_spi
    float s_off_ref[SX_MAX_QSCORE + 1];       // (float) q2lncompe
    float s_off_alt[SX_MAX_QSCORE + 1];       // (float) q2lne + ln(1/3)f
    float s_lnprior[3];                       // germlineGenotypeLogPrior
    float s_ln_sse_rate, s_ln_csse_rate, s_ln_som_match, s_ln_som_mismatch, s_contam_tolerance, s_ln_one_half;
    float s_log_error_mod, s_ratio_increment;
    float g_ln10f; // std::log(10.f), the FloatType=float ln10 of ln_error_prob_to_phred (blt_util/qscore.hh:54)
    // calculate_result_set_grid (qscore_calculator.cpp:47-145) unrolled on the host: for each (normal gt, somatic state) the
    // ordered list of (tumor freq index, normal freq index, ln prior) terms its double loop visits
    double s_term_lprior[6][44];
    uint8_t s_term_tf[6][44], s_term_nf[6][44];
    uint32_t s_n_terms[6];
    float s_geno_prior[6]; // germlineGenotypeLogPrior[ngt] + (tgt==0 ? lnmatch : lnmismatch), float add
    float pad2_[2];
    // indel genotype model
    double i_randomBaseMatchLogProb, i_correctMappingLogPrior, i_loghalf, i_readSupportThreshold;
    int32_t i_min_flank, i_pad;
};

int sx_upload_pileup(sx_ctx* ctx, const sx_pileup_batch* b, int slot_base, sx_pileup_batch* d, uint32_t* max_site, cudaStream_t st);
cudaError_t sx_k2a_init_tables(sx_tables* d_tables); // fills the g_val0_* rows of the device copy (synchronous)

struct sx_buf
{
    void* p = nullptr;
    size_t cap = 0;
};

struct sx_ctx
{
    int device = 0;
    sx_params params;
    sx_tables tables;        // host copy
    sx_tables* d_tables = nullptr;
    int* d_status = nullptr; // device-side error word (0 = ok)
    cudaStream_t s_compute = nullptr, s_h2d = nullptr, s_d2h = nullptr;
    cudaEvent_t ev_a = nullptr, ev_b = nullptr;
    std::vector<cudaEvent_t> ev_pool;
    int sm_count = 0;
    size_t smem_optin = 0;
    std::string err;
    sx_timing timing{};
    uint64_t total_launches = 0;
    sx_buf buf[192];         // grow-only device arenas, one per logical pool (host entries 0..29, K7 family 40..63, K4 64, pipeline 70..)
    void* nccl = nullptr;    // ncclComm_t
    void* nccl_lib = nullptr;
    int rank = 0, world = 1;
    cudaEvent_t ev_user[2] = {};     // sx_timer_mark
    cudaEvent_t ev_win[16] = {};     // stage boundaries of sx_process_window_dev (created on first use)
    float win_ms[16] = {};
    cudaStream_t s_comm = nullptr;   // the gather's own stream (created by sx_comm_init)
    cudaEvent_t ev_comm = nullptr;   // compute -> comm ordering
    std::vector<unsigned long long> comm_counts; // per-rank byte counts of the last gather (root: receive offsets)
    void* d_comm_counts = nullptr;
};
void sx_comm_release(sx_ctx* ctx); // sx_comm.cu: ncclCommDestroy + the comm stream (no-op without a communicator)

int sx_fail(sx_ctx* ctx, int code, const char* fmt, ...);
#define SX_CUDA(ctx, call)                                                                                        \
    do                                                                                                            \
    {                                                                                                             \
        cudaError_t e_ = (call);                                                                                  \
        if (e_ != cudaSuccess) return sx_fail((ctx), SX_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
    } while (0)

int sx_ensure(sx_ctx* ctx, int slot, size_t bytes, void** out);
int sx_check_status(sx_ctx* ctx, const char* what);

// timing helpers: record kernel time on the compute stream
struct sx_kernel_timer
{
    sx_ctx* ctx;
    explicit sx_kernel_timer(sx_ctx* c) : ctx(c) { cudaEventRecord(c->ev_a, c->s_compute); }
    void stop(unsigned launches)
    {
        cudaEventRecord(ctx->ev_b, ctx->s_compute);
        pending = launches;
    }
    int finish()
    {
        cudaError_t e = cudaEventSynchronize(ctx->ev_b);
        if (e != cudaSuccess) return sx_fail(ctx, SX_ERR_CUDA, "kernel failed: %s", cudaGetErrorString(e));
        float ms = 0;
        cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b);
        ctx->timing.kernel_ms += ms;
        ctx->timing.launches += pending;
        ctx->total_launches += pending;
        return SX_OK;
    }
    unsigned pending = 0;
};

// kernels' host launchers (each in its own .cu)
int sx_k1_launch(sx_ctx* ctx, const sx_align_batch* dev, uint32_t region_begin, uint32_t region_end, double* lnp_dev, size_t smem_bytes, size_t smem_fast,
                 cudaStream_t st);
size_t sx_k1_region_smem(const sx_region* r0, const sx_region* r1, const sx_aln* alns);

// asynchronous stage launchers of the device-resident pipeline (sx_pipeline.cu); each lives beside its kernels
int sx_k7g_run(sx_ctx* ctx, const sx_gate_batch* d, const sx_gate_out* o, unsigned* launches);
int sx_k7a_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_region* regions, const uint8_t* seq4, const char* ref, const uint32_t* key_ins_off, const char* key_ins,
               const sx_prep_out* o, unsigned* launches);
int sx_k7_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* o, unsigned* launches);
int sx_k8_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* e, uint32_t n_alns, const uint32_t* key_ins_off, const char* key_ins, const sx_link_out* o,
              unsigned* launches);
int sx_k1_run_dev(sx_ctx* ctx, const sx_align_batch* d, double* lnp_dev, unsigned* launches);
int sx_k6_run(sx_ctx* ctx, const sx_score_indels_batch* d, const double* lnp_dev, const sx_score_indels_out* out_dev, unsigned* launches);
int sx_k9_run(sx_ctx* ctx, const sx_realign_batch* d, const double* lnp, const sx_realign_out* o, unsigned* launches);
int sx_k4_run(sx_ctx* ctx, const sx_pileup_reads_batch* d, const sx_pileup_columns* out, unsigned* launches);
int sx_k2a_run(sx_ctx* ctx, const sx_pileup_batch* d, int is_always_test, sx_digt_result* out_dev, unsigned* launches);
