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

double log1p_switch(double x); // blt_util/math_util.hh:33-47 with the host libm (sx_context.cu)

int sx_upload_pileup(sx_ctx* ctx, const sx_pileup_batch* b, int host_base, sx_pileup_batch* d, uint32_t* max_site); // host slots host_base..+5
cudaError_t sx_k2a_init_tables(sx_tables* d_tables); // fills the g_val0_* rows of the device copy (synchronous)

// ---------------------------------------------------------------------------------------------------------------
// device buffers: sx_ctx::buf holds one grow-only buffer per slot.  Every buffer the library allocates has its slot here.
// ---------------------------------------------------------------------------------------------------------------
enum sx_slot : int
{
    // host staging: what a host-array entry point (sx_score_alignments, sx_site_gl_germline, ...) uploads and downloads, as
    // sx_host_slot(i).  The running entry owns the whole block; no stage launcher allocates in it.
    SX_SLOT_HOST = 0,
    SX_SLOT_HOST_END = SX_SLOT_HOST + 32,
    // stage scratch, owned by the stage's launcher while its launches run
    SX_SLOT_K1_SMEM_NEED = SX_SLOT_HOST_END,
    SX_SLOT_K2A_SCRATCH, SX_SLOT_K2A_MAX_SITE,
    SX_SLOT_K2B_REGION_OFF, SX_SLOT_K2B_REGION_SUMS,
    SX_SLOT_K2C_COUNTS, SX_SLOT_K2C_REC_OFF, SX_SLOT_K2C_TOTAL, SX_SLOT_K2C_SUMS,
    SX_SLOT_K3_INFO, SX_SLOT_K3_CURSOR, SX_SLOT_K3_ORDER, SX_SLOT_K3_SCRATCH,
    SX_SLOT_K4_SCAN_S, SX_SLOT_K4_SCAN_B, SX_SLOT_K4_TILE_SUMS, SX_SLOT_K4_MAX_CAND,
    SX_SLOT_K6_MAX, SX_SLOT_K6_LIST, SX_SLOT_K6_ARENA, SX_SLOT_K6_CLASS, SX_SLOT_K6_HIST, SX_SLOT_K6_LIST_BY_CLASS,
    // the list builder of K6b and K6g (k6_lists.cuh), and the tile sums of both links' second scan.  Each link's scratch is dead once its
    // write kernel is enqueued, and both links run on the compute stream, so their lifetimes cannot overlap.
    SX_SLOT_K6L_OFF, SX_SLOT_K6L_CURSOR, SX_SLOT_K6L_TOTAL64, SX_SLOT_K6L_SUMS, SX_SLOT_K6L_ID, SX_SLOT_K6L_REC, SX_SLOT_K6L_READ, SX_SLOT_K6L_ORDER,
    SX_SLOT_K6B_LOCUS_OF, SX_SLOT_K6B_ALT_IDS,
    // K6b's output where the library owns it: the sx_sindel_batch between the link and K5b (sx_somatic_indel_from_records_dev), and the
    // device side of sx_link_indel_reads
    SX_SLOT_K6B_OUT_ALT_OFF, SX_SLOT_K6B_OUT_ALTS, SX_SLOT_K6B_OUT_READ_OFF, SX_SLOT_K6B_OUT_READS, SX_SLOT_K6B_OUT_STATUS, SX_SLOT_K6B_OUT_TOTALS,
    SX_SLOT_K6G_LIST_OF, SX_SLOT_K6G_DUP, SX_SLOT_K6G_LNP64,
    // K6g's output where the library owns it: the sx_indel_batch between the link and K5 (sx_indel_gl_from_records_dev)
    SX_SLOT_K6G_OUT_READ_OFF, SX_SLOT_K6G_OUT_LNP_OFF, SX_SLOT_K6G_OUT_ALLELE_OFF, SX_SLOT_K6G_OUT_PLOIDY, SX_SLOT_K6G_OUT_DEL_LEN, SX_SLOT_K6G_OUT_INS_LEN,
    SX_SLOT_K6G_OUT_LNP, SX_SLOT_K6G_OUT_READ_LENGTH, SX_SLOT_K6G_OUT_NON_AMBIG, SX_SLOT_K6G_OUT_IS_FWD, SX_SLOT_K6G_OUT_STATUS, SX_SLOT_K6G_OUT_TOTALS,
    SX_SLOT_K7_READ_REGION, SX_SLOT_K7_ARENA, SX_SLOT_K7_ARENA_DEEP, SX_SLOT_K7_CNT_SEG, SX_SLOT_K7_CNT_KEY, SX_SLOT_K7_SUMS,
    SX_SLOT_K7_LOG, SX_SLOT_K7_LOG_OFF, SX_SLOT_K7_LOG_CURSOR, SX_SLOT_K7_RETRY1, SX_SLOT_K7_RETRY2, SX_SLOT_K7_RETRY_N, SX_SLOT_K7_ACTIVE,
    SX_SLOT_K7_CLASS, SX_SLOT_K7_HIST, SX_SLOT_K7_ACTIVE_BY_CLASS,
    SX_SLOT_K7A_READ_REGION, SX_SLOT_K7A_STAGE, SX_SLOT_K7A_ACTIVE,
    SX_SLOT_K8_ALN_READ, SX_SLOT_K8_READ_REGION, SX_SLOT_K8_SEG_N, SX_SLOT_K8_INS_N, SX_SLOT_K8_REG_SEG, SX_SLOT_K8_REG_INS, SX_SLOT_K8_SUMS,
    // per-read scratch shared by K7a and K9: a per-read word (K7a's entry: read byte offset, K9's entry: read region) and the tile sums of their scan.
    // These are O(reads) and every context that runs the window pass holds them.  Their lifetimes cannot overlap: K7a's are dead once its
    // write kernel has run, and K9 is enqueued after K7a on the same stream (sx_process_window_dev) or by its own entry point.
    SX_SLOT_K7A_K9_READ_WORD, SX_SLOT_K7A_K9_SUMS,
    // window pass: the intermediates of sx_process_window_dev
    SX_SLOT_WIN_READ_REGION, SX_SLOT_WIN_SEQ_OFF, SX_SLOT_WIN_QUAL_OFF, SX_SLOT_WIN_BPOS, SX_SLOT_WIN_NON_AMBIG, SX_SLOT_WIN_PIN, SX_SLOT_WIN_MAXIMA,
    SX_SLOT_WIN_GATE, SX_SLOT_WIN_IN_POS, SX_SLOT_WIN_IN_SEGS,
    SX_SLOT_WIN_KEY_TOTALS, SX_SLOT_WIN_IN_KEY_OFF, SX_SLOT_WIN_IN_KEYS, SX_SLOT_WIN_IN_LEAD, SX_SLOT_WIN_IN_TRAIL,
    SX_SLOT_WIN_ENUM_TOTALS, SX_SLOT_WIN_ALN_OFF, SX_SLOT_WIN_ENUM_STATUS, SX_SLOT_WIN_ALN_POS, SX_SLOT_WIN_ALN_SEG_OFF, SX_SLOT_WIN_SEGS,
    SX_SLOT_WIN_ALN_KEY_OFF, SX_SLOT_WIN_ALN_KEYS, SX_SLOT_WIN_ALN_LEAD, SX_SLOT_WIN_ALN_TRAIL,
    SX_SLOT_WIN_LINK_TOTALS, SX_SLOT_WIN_LINK_ALNS, SX_SLOT_WIN_LINK_SEGS, SX_SLOT_WIN_LINK_INS, SX_SLOT_WIN_K6_SEGS, SX_SLOT_WIN_LNP,
    SX_SLOT_WIN_RECS, SX_SLOT_WIN_N_REC, SX_SLOT_WIN_MAX_ALN, SX_SLOT_WIN_EVAL_ALN,
    SX_SLOT_WIN_BEST_TOTALS, SX_SLOT_WIN_BEST_SEG_OFF, SX_SLOT_WIN_BEST_POS, SX_SLOT_WIN_BEST_N_SEG, SX_SLOT_WIN_REALIGN_STATUS, SX_SLOT_WIN_BEST_ALN,
    SX_SLOT_WIN_BEST_SEGS, SX_SLOT_WIN_PILEUP_READS,
    SX_SLOT_WIN_SITE_OFF, SX_SLOT_WIN_T2_OFF, SX_SLOT_WIN_N_SPANDEL, SX_SLOT_WIN_N_SUBMAPPED, SX_SLOT_WIN_CALLS, SX_SLOT_WIN_T2_CALLS,
    SX_SLOT_WIN_SITE_GL, SX_SLOT_WIN_VARIANT_CHUNKS, SX_SLOT_WIN_VARIANT_SUMS,
    // somatic window pass (sx_process_somatic_window_dev): the normal sample's results that the later stages read, kept apart from the
    // tumor sample's pass (which uses the SX_SLOT_WIN_* buffers), and the somatic stages' own outputs and scratch
    SX_SLOT_SWIN_NON_AMBIG, SX_SLOT_SWIN_RECS, SX_SLOT_SWIN_N_REC, SX_SLOT_SWIN_SITE_OFF, SX_SLOT_SWIN_T2_OFF, SX_SLOT_SWIN_CALLS, SX_SLOT_SWIN_T2_CALLS,
    SX_SLOT_SWIN_SITE_SNV, SX_SLOT_SWIN_INDEL, SX_SLOT_SWIN_SNV_CHUNKS, SX_SLOT_SWIN_SNV_SUMS, SX_SLOT_SWIN_INDEL_CHUNKS, SX_SLOT_SWIN_INDEL_SUMS,
    // window pass: what sx_process_window uploads (the window batch's arrays) and the outputs it downloads
    SX_SLOT_WUP_REGION_READ_OFF, SX_SLOT_WUP_REGION_KEY_OFF, SX_SLOT_WUP_KEYS, SX_SLOT_WUP_KEY_HAP, SX_SLOT_WUP_KEY_INS_OFF, SX_SLOT_WUP_KEY_INS,
    SX_SLOT_WUP_REALIGN_BEGIN, SX_SLOT_WUP_REALIGN_END, SX_SLOT_WUP_RAW_POS, SX_SLOT_WUP_RAW_SEG_OFF, SX_SLOT_WUP_RAW_SEGS, SX_SLOT_WUP_READ_LEN,
    SX_SLOT_WUP_READ_FLAGS, SX_SLOT_WUP_MAPQ, SX_SLOT_WUP_USE_KEY_OFF, SX_SLOT_WUP_USE_KEYS, SX_SLOT_WUP_REC_OFF, SX_SLOT_WUP_REGIONS,
    SX_SLOT_WUP_SEQ4, SX_SLOT_WUP_QUAL, SX_SLOT_WUP_REF, SX_SLOT_WUP_CAND_SNV,
    SX_SLOT_WDN_GATE, SX_SLOT_WDN_ENUM_STATUS, SX_SLOT_WDN_REALIGN_STATUS, SX_SLOT_WDN_BEST_POS, SX_SLOT_WDN_BEST_SEG_OFF, SX_SLOT_WDN_BEST_N_SEG,
    SX_SLOT_WDN_BEST_SEGS, SX_SLOT_WDN_RECS, SX_SLOT_WDN_N_REC, SX_SLOT_WDN_SITE_OFF, SX_SLOT_WDN_T2_OFF, SX_SLOT_WDN_N_SPANDEL,
    SX_SLOT_WDN_N_SUBMAPPED, SX_SLOT_WDN_CALLS, SX_SLOT_WDN_T2_CALLS, SX_SLOT_WDN_SITE_GL, SX_SLOT_WDN_VARIANT_SITES,
    SX_SLOT_COUNT
};

// slot i of the host staging block (SX_SLOT_COUNT, which sx_ensure refuses, past its end)
constexpr sx_slot sx_host_slot(int i) { return i >= 0 && i < SX_SLOT_HOST_END - SX_SLOT_HOST ? sx_slot(SX_SLOT_HOST + i) : SX_SLOT_COUNT; }

// ---------------------------------------------------------------------------------------------------------------
// device status word (sx_ctx::d_status): the bits the kernels raise.  sx_check_status (sx_context.cu) reports each with its own
// error code and message, and clears the word.
// ---------------------------------------------------------------------------------------------------------------
enum sx_status_bit : int
{
    SX_ST_QUAL = 1,              // K1, K4: a quality score above SX_MAX_QSCORE
    SX_ST_TILE = 2,              // K1: a region does not fit the shared-memory tile of the launch
    SX_ST_SEG_KIND = 4,          // K1, K4: an unknown segment kind
    SX_ST_READ_OVERRUN = 8,      // K1: a path consumes more read bases than the read holds
    SX_ST_SITE_DEPTH = 16,       // K2a: a site deeper than the kernel handles
    SX_ST_INDEL_ALLELES = 32,    // K5: allele count or ploidy outside the model
    SX_ST_READ_ORDER = 64,       // K4: reads out of position order, or an alignment wider than max_ref_span
    SX_ST_BASE = 128,            // K4: an unknown base code
    SX_ST_READ_LIMIT = 256,      // K4: a read longer, or with more segments, than the kernel handles
    SX_ST_K6_SEG_KIND = 1 << 9,  // K6 (K6_ST_* of k6_core.cuh, shifted by 9)
    SX_ST_K6_ALNS = 1 << 10,
    SX_ST_K6_EVAL = 1 << 11,
    SX_ST_K6_REC_CAP = 1 << 12,
    SX_ST_K6_KEY = 1 << 13,
    SX_ST_K7_CAP = 1 << 14,      // K7: an output capacity is too small
    SX_ST_K8_NO_KEY = 1 << 15,   // K8 (K8_ST_* of k8_core.cuh, shifted by 15)
    SX_ST_K8_KIND = 1 << 16,
    SX_ST_K8_CAP = 1 << 17,      // K8: an output capacity is too small
    SX_ST_K7A_CAP = 1 << 18,     // K7a: cap_keys is too small
    SX_ST_K9_CAP = 1 << 19,      // K9: cap_segs is too small
    SX_ST_SINDEL_CAP = 1 << 20,  // K5b: a locus over the alternate caps.  Written to that locus's result status (SX_SINDEL_ST_CAP), never to
                                 // the device word: the locus gets no result and the call goes on.
    SX_ST_SINDEL_ARG = 1 << 21,  // K5b: a candidate that is not SX_INDEL_TYPE_INDEL, or an error-rate index past the table
    SX_ST_INDEL_READS_DUP = 1 << 22, // K6b: one read id twice in a locus's list.  Like SX_ST_SINDEL_CAP a per-locus status (SX_INDEL_READS_ST_DUP_READ),
                                     // never in the device word
    SX_ST_K6B_ID = 1 << 23,      // K6b: a window index past its region's window, or an id at or past n_gid
    SX_ST_K6G_GROUP = 1 << 24,   // K6g: a group with an allele count outside 1..SX_INDEL_MAX_ALLELES, a ploidy outside {1,2}, an id at or past n_gid,
                                 // or offsets that do not start at 0 and ascend
    SX_ST_CONT_TIE = 1 << 25,    // K2c: a qscore within its error bound of a rounding boundary.  A per-entry status (SX_CONT_ST_QSCORE_TIE), never in
                                 // the device word
};
static_assert(SX_ST_SINDEL_CAP == SX_SINDEL_ST_CAP, "the per-locus capacity status of K5b is its status bit");
static_assert(SX_ST_CONT_TIE == SX_CONT_ST_QSCORE_TIE, "the per-entry tie status of K2c is its status bit");

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
    sx_buf buf[SX_SLOT_COUNT]; // grow-only device buffers, one per sx_slot
    void* nccl = nullptr;    // ncclComm_t
    void* nccl_lib = nullptr;
    int rank = 0, world = 1;
    cudaEvent_t ev_user[2] = {};     // sx_timer_mark
    cudaEvent_t ev_win[16] = {};     // stage boundaries of sx_process_window_dev (created on first use)
    float win_ms[16] = {};
    cudaEvent_t ev_swin[16] = {};    // stage boundaries of sx_process_somatic_window_dev (created on first use)
    float swin_ms[16] = {};
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

int sx_ensure(sx_ctx* ctx, sx_slot slot, size_t bytes, void** out);

// the slot's buffer as `count` elements of T plus `slack` bytes
template <typename T> int sx_take(sx_ctx* ctx, sx_slot slot, size_t count, T*& p, size_t slack)
{
    void* q(nullptr);
    const int rc(sx_ensure(ctx, slot, count * sizeof(T) + slack, &q));
    p = static_cast<T*>(q);
    return rc;
}

// host staging of a host-array entry point: `count` elements of `src` into the slot's buffer (sized with `slack` extra bytes) on the
// compute stream; `dst` is the device copy.  An empty array is allocated but not copied.
template <typename T> int sx_upload(sx_ctx* ctx, sx_slot slot, const T* src, size_t count, const T*& dst, size_t slack)
{
    T* p(nullptr);
    const int rc(sx_take(ctx, slot, count, p, slack));
    if (rc) return rc;
    if (count) SX_CUDA(ctx, cudaMemcpyAsync(p, src, count * sizeof(T), cudaMemcpyHostToDevice, ctx->s_compute));
    dst = p;
    return SX_OK;
}
template <typename T> int sx_upload(sx_ctx* ctx, sx_slot slot, const T* src, size_t count, T*& dst, size_t slack)
{
    const T* p(nullptr);
    const int rc(sx_upload(ctx, slot, src, count, p, slack));
    dst = const_cast<T*>(p);
    return rc;
}
// ... and back: `count` elements of `src` into `dst` (nothing for an empty array)
template <typename T> int sx_download(sx_ctx* ctx, T* dst, const T* src, size_t count)
{
    if (count) SX_CUDA(ctx, cudaMemcpyAsync(dst, src, count * sizeof(T), cudaMemcpyDeviceToHost, ctx->s_compute));
    return SX_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// prefix sums (sx_scan.cu): 1..SX_SCAN_MAX uint32 arrays scanned in place, each with its own length and flavour.  One call enqueues
// three launches on the compute stream and adds them to *launches; `sums_slot` is the calling stage's own buffer for the tile sums.
// ---------------------------------------------------------------------------------------------------------------
constexpr uint32_t SX_SCAN_TILE = 4096, SX_SCAN_THREADS = 256;
constexpr int SX_SCAN_MAX = 8;
enum sx_scan_flag : uint32_t
{
    SX_SCAN_EXCLUSIVE = 1, // data[i] = the sum of the elements before i (else up to and including i)
    SX_SCAN_CLOSE = 2,     // also data[n] = the sum of all n (the array holds n + 1 words)
};
struct sx_scan_array
{
    uint32_t* data;
    uint32_t n;
    uint32_t flags;  // sx_scan_flag bits
    uint32_t* total; // device word for the sum of all n, or NULL
};
struct sx_scan_set
{
    int n_arrays;
    sx_scan_array a[SX_SCAN_MAX];
};
int sx_scan(sx_ctx* ctx, sx_slot sums_slot, const sx_scan_set& job, unsigned* launches);

// Reports and clears the device status word: SX_OK when it is 0, else the error of its first set bit.  The bits in `first` (a stage's
// own) are tested before the others.  `totals`, when the caller has them, are the stage's totals the capacity messages quote.
int sx_check_status(sx_ctx* ctx, const char* what, int first = 0, const uint32_t* totals = nullptr);

// The body of a *_dev entry point: on the context's device, `run(unsigned* launches)` enqueues a stage through its launcher, between two
// events on the compute stream.  Once the stream has passed the second, the time between them and the launches are added to ctx->timing and
// ctx->total_launches.  An error from `run` is returned at once, with nothing added.
template <typename F> int sx_run_timed(sx_ctx* ctx, F&& run)
{
    SX_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaEventRecord(ctx->ev_a, ctx->s_compute);
    unsigned launches = 0;
    const int rc = run(&launches);
    if (rc) return rc;
    cudaEventRecord(ctx->ev_b, ctx->s_compute);
    const cudaError_t e = cudaEventSynchronize(ctx->ev_b);
    if (e != cudaSuccess) return sx_fail(ctx, SX_ERR_CUDA, "kernel failed: %s", cudaGetErrorString(e));
    float ms = 0;
    cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b);
    ctx->timing.kernel_ms += ms;
    ctx->timing.launches += launches;
    ctx->total_launches += launches;
    return SX_OK;
}

// the host-array counterpart: the whole call on the compute stream, ev_a before the uploads and ev_b after the downloads
struct sx_call_timer
{
    sx_ctx* ctx;
    cudaError_t start; // (reported by finish)
    explicit sx_call_timer(sx_ctx* c) : ctx(c), start(cudaEventRecord(c->ev_a, c->s_compute)) {}
    int finish(unsigned launches)
    {
        SX_CUDA(ctx, start);
        SX_CUDA(ctx, cudaEventRecord(ctx->ev_b, ctx->s_compute));
        SX_CUDA(ctx, cudaStreamSynchronize(ctx->s_compute));
        float ms = 0;
        cudaEventElapsedTime(&ms, ctx->ev_a, ctx->ev_b);
        ctx->timing.kernel_ms = ms;
        ctx->timing.launches = launches;
        ctx->total_launches += launches;
        return SX_OK;
    }
};

// kernels' host launchers (each in its own .cu)
int sx_k1_launch(sx_ctx* ctx, const sx_align_batch* dev, uint32_t region_begin, uint32_t region_end, double* lnp_dev, size_t smem_bytes, size_t smem_fast,
                 cudaStream_t st);
size_t sx_k1_region_smem(const sx_region* r0, const sx_region* r1, const sx_aln* alns);

// The stage launchers, each beside its kernels and the only code that launches them.  A launcher enqueues its stage on ctx->s_compute
// (device pointers in and out) and adds the stage's launches to *launches; it does no timing, reads no status word and leaves the device
// as the caller set it.  The *_dev entries run them under sx_run_timed, the host-array entries after their uploads (K1's and K2a's
// through sx_k1_launch and germline_run, as their batches are measured on the host), and sx_process_window_dev one after another.
int sx_k1_run(sx_ctx* ctx, const sx_align_batch* d, double* lnp_dev, unsigned* launches);
int sx_k1_read_max_run(sx_ctx* ctx, const sx_align_batch* d, const double* lnp_dev, double* max_lnp_dev, uint32_t* max_aln_dev, unsigned* launches);
int sx_k2a_run(sx_ctx* ctx, const sx_pileup_batch* d, int is_always_test, sx_digt_result* out_dev, unsigned* launches);
// `callable`: isComputeNonSomatic (sx_site_gl_somatic_callable_dev)
int sx_k2b_run(sx_ctx* ctx, const sx_pileup_batch* n, const sx_pileup_batch* t, const uint8_t* forced_dev, sx_ssnv_result* out_dev, bool callable,
               unsigned* launches);
// the callable regions of site_snv[n_pos] (n_pos > 0); *total_host (host memory) receives their number once the stream has passed the copy
int sx_k2b_regions_run(sx_ctx* ctx, const sx_ssnv_result* site_snv, uint32_t n_pos, int32_t pos_begin, int32_t* region_begin, int32_t* region_end,
                       uint32_t cap, uint32_t* total_host, unsigned* launches);
int sx_k3_run(sx_ctx* ctx, const sx_ga_scores* sc, const sx_ga_batch* d, sx_ga_result* res_dev, uint32_t* cigar_dev, unsigned* launches);
int sx_k4_run(sx_ctx* ctx, const sx_pileup_reads_batch* d, const sx_pileup_columns* out, unsigned* launches);
int sx_k5_run(sx_ctx* ctx, const sx_indel_batch* d, sx_indel_result* out_dev, unsigned* launches);
int sx_k5b_run(sx_ctx* ctx, const sx_sindel_opts* o, const sx_sindel_batch* d, const double* err_prob, uint32_t n_err, sx_sindel_result* out_dev, unsigned* launches);
// K5b's argument checks, reported under `what` (the K5b entries, and sx_somatic_indel_from_records_dev before its K5b run)
int sx_k5b_check(sx_ctx* ctx, const char* what, const sx_sindel_opts* o, const sx_sindel_batch* b, const double* err_prob, uint32_t n_err, const void* out);
int sx_k6_run(sx_ctx* ctx, const sx_score_indels_batch* d, const double* lnp_dev, const sx_score_indels_out* out_dev, unsigned* launches);
int sx_k6b_run(sx_ctx* ctx, const char* what, const sx_indel_reads_sample* normal, const sx_indel_reads_sample* tumor, const sx_indel_loci* loci, sx_indel_reads_out* out_dev,
               uint32_t* totals_host, bool own_out, unsigned* launches);
// K6b's argument checks of the loci, reported under `what`
int sx_k6b_check_loci(sx_ctx* ctx, const char* what, const sx_indel_loci* loci);
// ... of one sample (K6b and K6g), and the host staging of one sample's arrays into host slots base .. base + 9 (ids checked against n_gid)
int sx_k6b_check_sample(sx_ctx* ctx, const char* what, const sx_indel_reads_sample* s);
int sx_k6b_upload_sample(sx_ctx* ctx, const char* what, const sx_indel_reads_sample* h, int base, uint32_t n_gid, sx_indel_reads_sample* d);
// The link's offset, status and totals arrays in the context's SX_SLOT_K6B_OUT_* buffers (its entries and alternates are taken by sx_k6b_run
// with own_out once their totals are known), and the sx_sindel_batch they form with the loci
int sx_k6b_own_out(sx_ctx* ctx, uint32_t n_loci, sx_indel_reads_out* o);
sx_sindel_batch sx_sindel_batch_of(const sx_indel_loci* loci, const sx_indel_reads_out* o);
// K5b -> the link's flags into the results, enqueued on the compute stream behind the link (sx_k6b_run with own_out into `o`, from
// sx_k6b_own_out): the second half of sx_somatic_indel_from_records_dev and of the somatic window pass.  The arguments are checked by the
// caller (sx_k5b_check); the status word is the caller's to read.
int sx_sindel_from_links_run(sx_ctx* ctx, const sx_sindel_opts* opts, const sx_indel_loci* loci, const sx_indel_reads_out* o, const double* err_prob, uint32_t n_err,
                             sx_sindel_result* out_dev, unsigned* launches);
// K6g: one sample's K6 records -> K5's per-group read lists.  totals_host receives {reads, allele_lnp floats} (also on SX_ERR_CAPACITY).
// own_out: the allele and per-read arrays are taken from the context's SX_SLOT_K6G_OUT_* buffers once the totals are known, instead of checked
// against the caller's capacities.  The status word (SX_ST_K6G_GROUP, SX_ST_K6B_ID) is the caller's to read.
int sx_k6g_run(sx_ctx* ctx, const char* what, const sx_indel_reads_sample* sample, const sx_allele_groups* groups, sx_allele_group_reads_out* out_dev,
               uint32_t* totals_host, bool own_out, unsigned* launches);
// K2c on device arrays: count, scan, write.  totals_host[0] receives the record count (also on SX_ERR_CAPACITY, which leaves site_rec_off
// written and no record).  One host synchronisation (the count).
int sx_k2c_run(sx_ctx* ctx, const sx_cont_opts* o, const sx_cont_batch* d, const sx_cont_out* out, uint32_t* totals_host, unsigned* launches);
// The read index (sx_read_index.cu): one pass, a warp per region.  Every output array is optional (NULL: not computed); seq_off / qual_off
// (which need read_len and regions) are byte offsets in the pools -- the region's seq_off / qual_off plus the sizes of the reads before it in
// the region -- closed by [n_reads].
struct sx_read_index_in
{
    uint32_t n_regions, n_reads, qual_bits;
    const uint32_t* region_read_off;
    const uint16_t* read_len;
    const sx_region* regions;
};
struct sx_read_index
{
    uint32_t* region;   // [n_reads] the read's region
    uint32_t* seq_off;  // [n_reads + 1] byte offset of its packed bases
    uint32_t* qual_off; // [n_reads + 1] ... of its qualities (qual_bits 4: packed like the bases; else one byte per base)
};
int sx_read_index_run(sx_ctx* ctx, const sx_read_index_in* in, const sx_read_index* o, unsigned* launches);
// ... only the region of every read (the stages' own entry points)
int sx_read_region_run(sx_ctx* ctx, uint32_t n_regions, uint32_t n_reads, const uint32_t* region_read_off, uint32_t* region, unsigned* launches);
// The per-read stages take the region of every read (and K7a the byte offset of its packed bases) from the window's read index.  NULL (a
// stage's own entry points): K7a and K7b build them with the index's kernel in place of the one launch they always had for it; the gates and
// K9, which had none, search region_read_off per read.
int sx_k7g_run(sx_ctx* ctx, const sx_gate_batch* d, const sx_gate_out* o, const uint32_t* read_region, unsigned* launches);
int sx_k7a_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_region* regions, const uint8_t* seq4, const char* ref, const uint32_t* key_ins_off, const char* key_ins,
               const sx_prep_out* o, const uint32_t* read_region, const uint32_t* read_seq_off, unsigned* launches);
int sx_k7_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* o, unsigned* launches);
// K7 and K7a: the reads whose gate lets them into the search (SX_GATE_REALIGN) as a dense list, *count of them (one launch)
int sx_k7_active_reads(sx_ctx* ctx, uint32_t n_reads, const uint8_t* gate, uint32_t* list, uint32_t* count);
int sx_k8_run(sx_ctx* ctx, const sx_enum_batch* d, const sx_enum_out* e, uint32_t n_alns, const uint32_t* key_ins_off, const char* key_ins, const sx_link_out* o,
              const uint32_t* read_region, unsigned* launches);
int sx_k9_run(sx_ctx* ctx, const sx_realign_batch* d, const double* lnp, const sx_realign_out* o, const uint32_t* read_region, unsigned* launches);
