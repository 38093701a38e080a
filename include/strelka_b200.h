/*
 * strelka_b200.h -- C ABI of the GPU-native Strelka2 per-locus scoring hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b).  The reference (Illumina/strelka,
 * paths relative to /root/reference/src/c++/lib/) has no FFI of its own; each entry point
 * below names the reference call site whose work it takes over.  INTEGRATION.md shows the
 * C++ shim a reference maintainer adds at each of those call sites.
 *
 * Conventions
 *   - plain pointers and sizes only; every input/output buffer is HOST memory owned by the
 *     caller for the duration of the call (pinned memory from sx_host_alloc() makes the
 *     transfers true DMA).  `*_dev` variants take DEVICE pointers (inputs already in HBM).
 *   - return value 0 == SX_OK, negative == failure; sx_last_error(ctx) gives the text.
 *     The library never calls exit() and never falls back to a CPU implementation: without
 *     a usable CUDA device sx_create() fails with SX_ERR_CUDA.
 *   - one sx_ctx per (GPU, host thread).  No process globals: unlike the reference's
 *     function-local static caches (strelka_common/position_snp_call_grid_lhood_cached.cpp:136,
 *     applications/strelka/position_somatic_snv_strand_grid_lhood_cached.cpp:46,139) a ctx is
 *     re-entrant.
 */
#ifndef STRELKA_B200_H
#define STRELKA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SX_ABI_VERSION 2

enum {
    SX_OK = 0,
    SX_ERR_CUDA = -1,        /* CUDA runtime/driver failure (incl. "no device") */
    SX_ERR_ARG = -2,         /* NULL / inconsistent argument */
    SX_ERR_ALIGNMENT = -3,   /* a region slice violates the 16-byte staging alignment rule */
    SX_ERR_UNSUPPORTED = -4, /* option combination outside the accelerated path */
    SX_ERR_RANGE = -5,       /* value outside the reference's own asserted range (e.g. qscore > 70) */
    SX_ERR_NOMEM = -6,
    SX_ERR_NCCL = -7
};

typedef struct sx_ctx sx_ctx;

/* ------------------------------------------------------------------------------------------
 * Options snapshot: every option field the hot-path functions read.
 *   blt_options            blt_common/blt_shared.hh:82-128
 *   starling_options       applications/starling/starling_shared.hh:34-39 (ssd 0.35/0.6, min_vexp 0.25)
 *   strelka_options        applications/strelka/strelka_shared.hh:126-151
 * sx_default_params() fills the reference defaults for the germline (starling2) caller and the
 * workflow defaults of configureStrelkaSomaticWorkflow.py.ini for the somatic one.
 * ---------------------------------------------------------------------------------------- */
typedef struct sx_params {
    /* germline site model */
    double bsnp_diploid_theta;           /* 0.001 */
    double bsnp_ssd_no_mismatch;         /* 0.35  (0 disables dependent error probs) */
    double bsnp_ssd_one_mismatch;        /* 0.6 */
    int32_t is_min_vexp;                 /* 1 */
    int32_t is_bsnp_diploid;             /* 1 for starling; is_dependent_eprob() needs it (blt_shared.hh:76-81) */
    double min_vexp;                     /* 0.25 */
    double hetVariantFrequencyExtension; /* 0; >0 (RNA mode) -> SX_ERR_UNSUPPORTED */
    /* somatic site model */
    double somatic_snv_rate;                         /* 1e-4  */
    double shared_site_error_rate;                   /* 5e-10 */
    double shared_site_error_strand_bias_fraction;   /* 0 */
    double ssnv_contam_tolerance;                    /* 0.15 */
    /* runtime knobs (not reference options) */
    int32_t pipeline_chunks;   /* host-buffer entry points split a batch into this many H2D/compute/D2H chunks; 0 = auto */
    /* indel genotype model (starling_base_options, starling_common/starling_base_shared.hh:108,177,245) */
    int32_t min_read_bp_flank;             /* 5 */
    double randomBaseMatchProb;            /* 0.25 */
    double readConfidentSupportThreshold;  /* 0.51 */
} sx_params;

void sx_default_params(sx_params* p);

int sx_create(int cuda_device, const sx_params* p, sx_ctx** out);
/* How this process's host threads wait for `cuda_device` (a runtime knob, not a reference option): blocking = 1 makes every wait of a context on
 * that device yield the CPU instead of spinning (cudaDeviceScheduleBlockingSync) -- for hosts whose CPU quota is smaller than the number of waiting
 * threads (8 ranks x several contexts on a 16-CPU cgroup: spinning waiters exhaust the quota and every rank stalls); 0 restores the driver's choice.
 * Call it before the first sx_create on the device.  Returns SX_OK or SX_ERR_CUDA. */
int sx_set_host_wait_policy(int cuda_device, int blocking);
void sx_destroy(sx_ctx* ctx);
const char* sx_last_error(const sx_ctx* ctx); /* valid until the next call on ctx; ctx may be NULL for create errors */
int sx_abi_version(void);

/* pinned host memory helpers (cudaHostAlloc / cudaFreeHost) */
void* sx_host_alloc(size_t bytes);
void sx_host_free(void* p);
/* device memory helpers for the *_dev entry points (cudaMalloc/cudaFree/cudaMemcpy on ctx's device) */
void* sx_dev_alloc(sx_ctx* ctx, size_t bytes);
void sx_dev_free(sx_ctx* ctx, void* p);
int sx_memcpy_h2d(sx_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes);
int sx_memcpy_d2h(sx_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes);
int sx_memcpy_d2d(sx_ctx* ctx, void* dst_dev, const void* src_dev, size_t bytes); /* on ctx's compute stream, asynchronous */
int sx_synchronize(sx_ctx* ctx);
/* Device-side timing of a run of entry points: sx_timer_mark(ctx, 0) and (ctx, 1) record CUDA events on ctx's compute stream where they are
 * called; sx_timer_elapsed_ms waits for mark 1 and returns the device time between the two (host gaps between launches included). */
int sx_timer_mark(sx_ctx* ctx, int which);
/* Everything enqueued so far on `other`'s compute stream becomes a prerequisite of whatever `waiter` enqueues next (an event on one stream, a
 * wait on the other; no host synchronisation): lets a caller that runs windows on several contexts close a device-timed region on one of them. */
int sx_stream_join(sx_ctx* waiter, sx_ctx* other);
int sx_timer_elapsed_ms(sx_ctx* ctx, double* ms);

/* ==========================================================================================
 * K1  score_alignments
 *   replaces the loop  for (cal : candAlignments) scoreCandidateAlignment(opt,indelBuffer,rseg,cal,ref)
 *   starling_common/starling_read_align.cpp:1568-1571 calling
 *   starling_common/starling_read_align_score.cpp:260-499.
 *
 * A batch is a list of REGIONS (the reads buffered around one candidate locus / realignment
 * window).  Each region owns a slice of the reference, a contiguous run of reads and the
 * contiguous run of candidate alignments of those reads.
 *
 * Staging rule (the kernel moves each region into shared memory with TMA bulk copies):
 *   region.seq_off, region.qual_off, region.ref_off and the first insert-pool byte of a region
 *   are multiples of 16; the first segment index of a region is a multiple of 4; every pool is
 *   allocated with SX_POOL_SLACK spare bytes after its last used byte.  Violations return
 *   SX_ERR_ALIGNMENT.  The C++ host mirror (strelka_b200/host/strelka_b200.hh, sx::ReadAlignBatch) builds
 *   conforming batches from reference-shaped objects.
 * ======================================================================================== */
#define SX_POOL_SLACK 64

/* flattened path segment kinds (host flattens ALIGNPATH::align_t + IndelKey lookups, see
 * starling_read_align_score.cpp:306-499 and INTEGRATION.md) */
enum {
    SX_SEG_MATCH = 0,    /* MATCH / SEQ_MATCH: read base vs reference base; advances read and ref */
    SX_SEG_INSERT = 1,   /* INSERT, the insert half of a swap, or SEQ_MISMATCH: read base vs next bases of the
                            alignment's insert-pool slice (already tail-adjusted for leading-edge insertions,
                            score.cpp:334-338,394-398); advances read only */
    SX_SEG_REFSKIP = 2,  /* DELETE / SKIP / delete half of a swap / ref half of SEQ_MISMATCH: advances ref only */
    SX_SEG_SOFTCLIP = 3, /* adds len*ln(0.25) (score.cpp:453-454); advances read */
    SX_SEG_HARDCLIP = 4  /* no-op */
};
#define SX_SEGF_NONCANDIDATE 0x1 /* add ln(1e-5) after this segment (score.cpp:473-485) */

typedef struct sx_aln_seg {
    uint16_t len;
    uint8_t kind;
    uint8_t flags;
} sx_aln_seg;

typedef struct sx_aln {
    uint32_t read;    /* read index in the batch */
    int32_t ref_pos;  /* cal.al.pos: contig coordinate of the first reference base of the path */
    uint32_t seg_off; /* index of first segment in seg pool; segments end at the next alignment's seg_off */
    uint32_t ins_off; /* byte offset of this alignment's inserted bases in the insert pool */
} sx_aln;

/* Compact wire formats (sx_align_batch.format bits).  The scoring entry points are PCIe-bound from host buffers, so bytes are
 * throughput: a batch may send its alignment headers and segments in half the space.  Semantics are identical; the builder falls
 * back to the wide structs when a field would not fit. */
#define SX_FMT_ALN8 0x1u /* `alns` points to sx_aln8[n_alns + 1] */
#define SX_FMT_SEG2 0x2u /* `segs` points to sx_aln_seg2[n_segs]; every region's seg_begin is a multiple of 8 */
/* SX_FMT_BASEQ: base and quality in ONE nibble per base.  The seq4 pool keeps its layout (reads back to back, byte-aligned, high
 * nibble first) but a nibble is (base << 2) | quality code, base A C G T = 0..3, quality code an index into qual_dict[0..3]
 * (qual_bits must be 2, every dictionary quality <= 70); the qual pool is not read.  The few bases that are not A/C/G/T are listed
 * per region in `exc` (their nibble still carries the quality code).  Halves the read bytes again: 75 bytes per 150 bp read. */
#define SX_FMT_BASEQ 0x4u
/* SX_FMT_REF4: the ref pool holds BAM 4-bit codes, two bases per byte, high nibble first (anything that is not A/C/G/T as 15);
 * region.ref_off is the byte offset of the window's first packed byte (multiple of 16), ref_len stays in bases. */
#define SX_FMT_REF4 0x8u
#define SX_EXC(pos, bam_code) ((uint32_t)(pos) | ((uint32_t)(bam_code) << 24)) /* exception: nibble position in the region's seq4 slice (< 2^24), bam_seq code */

typedef struct sx_aln8 {  /* every field relative to the alignment's region; an alignment's segments end at the next alignment's */
    uint16_t read;        /* seg_off, the last alignment's at the region's last segment                                          */
    int16_t ref_pos;      /* ref_pos - region.ref_begin */
    uint16_t seg_off;     /* seg_off - region.seg_begin */
    uint16_t ins_off;     /* ins_off - region.ins_begin */
} sx_aln8;

typedef uint16_t sx_aln_seg2; /* len (bits 0-11, <= 4095) | kind << 12 (3 bits) | flags << 15 */

typedef struct sx_region {
    uint64_t seq_off;    /* byte offset in seq4 pool of the region's first read (multiple of 16) */
    uint64_t qual_off;   /* byte offset in qual pool (multiple of 16) */
    uint64_t ref_off;    /* byte offset in ref pool (multiple of 16) */
    uint32_t read_begin; /* first read; reads end at next region's read_begin */
    uint32_t aln_begin;  /* first alignment; ends at next region's aln_begin */
    uint32_t seg_begin;  /* == alns[aln_begin].seg_off rounded down to the region's first (possibly pad) segment; multiple of 4 */
    uint32_t ins_begin;  /* first insert-pool byte of the region; multiple of 16 */
    int32_t ref_begin;   /* contig coordinate of ref pool byte ref_off */
    uint32_t ref_len;    /* bases available; positions outside read as 'N' (reference_contig_segment::get_base) */
} sx_region;

typedef struct sx_align_batch {
    uint32_t n_regions;
    uint32_t n_reads;
    uint32_t n_alns;
    uint32_t n_segs;
    const sx_region* regions;  /* [n_regions + 1]; entry n_regions is a sentinel carrying the end offsets */
    const uint16_t* read_len;  /* [n_reads] */
    const uint8_t* seq4;       /* BAM-native 4-bit packed bases ('=':0 A:1 C:2 G:4 T:8 N:15, high nibble first,
                                  htsapi/bam_seq.hh:38-47); within a region reads are packed back to back,
                                  each read starting on a byte boundary */
    const uint8_t* qual;       /* 1 byte per base, reads back to back within a region; values <= 70 */
    const char* ref;           /* ASCII reference bases */
    const sx_aln* alns;        /* [n_alns + 1], sorted by region; sentinel carries end offsets */
    const sx_aln_seg* segs;    /* [n_segs] */
    const char* ins;           /* ASCII inserted bases */
    uint64_t seq4_bytes, qual_bytes, ref_bytes, ins_bytes; /* used bytes of each pool (without slack) */
    /* Quality wire format.  qual_bits 0 or 8: `qual` holds one byte per base.  qual_bits 4: a batch whose reads use at most 16
     * distinct quality values (binned Illumina qualities do) may send them dictionary-coded, two per byte, high nibble first,
     * each read starting on a byte boundary exactly like seq4; nibble v stands for quality qual_dict[v].  Lossless; it cuts the
     * host->device bytes of a 150 bp read from 225 to 150 and selects the byte-entry scoring kernel (k1_score4.cu).
     * qual_bits 2: at most 4 distinct values (NovaSeq-style binning): one 2-bit code per NIBBLE POSITION of the region's seq4
     * slice, pad nibbles included -- the code of the nibble at position p (counted from the region's seq_off, two per byte) is
     * bits 7-2*(p&3) .. 6-2*(p&3) of byte region.qual_off + p/4; a region's quality slice is half its seq4 slice. */
    uint32_t qual_bits;
    uint8_t qual_dict[16];
    uint32_t format; /* SX_FMT_* bits; 0 = sx_aln / sx_aln_seg */
    /* SX_FMT_BASEQ only: exceptions of region i are exc[exc_off[i] .. exc_off[i+1]), SX_EXC words in any order */
    const uint32_t* exc_off; /* [n_regions + 1] */
    const uint32_t* exc;
} sx_align_batch;

/* lnp_out[n_alns] <- ln P(read | alignment path); bit-identical to the reference's double. */
int sx_score_alignments(sx_ctx* ctx, const sx_align_batch* batch_host, double* lnp_out_host);
/* same, every pointer inside *batch_dev and lnp_out_dev is a DEVICE pointer (the struct itself is host) */
int sx_score_alignments_dev(sx_ctx* ctx, const sx_align_batch* batch_dev, double* lnp_out_dev);
/* cell updates in a batch = sum over alignments of read bases in MATCH/INSERT segments (SURVEY 8a GCUPS def.) */
uint64_t sx_align_batch_cells(const sx_align_batch* batch_host);

/* K1 epilogue (starling_read_align.cpp:1535-1593): per read, the maximum path score and the index of the first
 * alignment attaining it in batch order; ties are resolved by the caller with isFirstCandidateAlignmentPreferred
 * (:1352) among alignments whose score equals max.  max_aln[n_reads] (UINT32_MAX for a read without alignments). */
int sx_read_max_dev(sx_ctx* ctx, const sx_align_batch* batch_dev, const double* lnp_dev,
                    double* max_lnp_dev, uint32_t* max_aln_dev);

/* ==========================================================================================
 * K3  global_align
 *   replaces _aligner.align(hap.begin,end, ref.begin,end, result)
 *   starling_common/ActiveRegionProcessor.cpp:591 -> alignment/GlobalAlignerImpl.hh:36-228,
 *   alignment/SingleRefAlignerSharedImpl.hh:80-170 (traceback, '='/'X' expansion).
 * ======================================================================================== */
typedef struct sx_ga_scores { /* alignment/AlignmentScores.hh:24-53 */
    int32_t match, mismatch, open, extend, offEdge, insertDelete;
    int32_t isAllowEdgeInsertion, isRequireEdgeDeletion;
} sx_ga_scores;

/* the scores ActiveRegionDetector constructs its aligner with (ActiveRegionDetector.hh:62-66, .cpp:41) */
void sx_ga_active_region_scores(sx_ga_scores* s);

typedef struct sx_ga_batch {
    uint32_t n;
    const char* query;         /* ASCII pool */
    const char* ref;           /* ASCII pool */
    const uint32_t* query_off; /* [n+1] */
    const uint32_t* ref_off;   /* [n+1] */
    uint32_t max_ops;          /* capacity (in ops) of each result's cigar slot */
} sx_ga_batch;

/* cigar op = (len << 4) | code with BAM codes M0 I1 D2 N3 S4 H5 P6 =7 X8 */
typedef struct sx_ga_result {
    int32_t score;
    int32_t beginPos;
    uint32_t n_ops; /* > max_ops: overflow, cigar truncated */
    uint32_t status; /* 0 ok; 1 cigar overflow; 2 problem too large for the kernel's shared-memory tile */
} sx_ga_result;

#define SX_GA_MAX_QUERY 1023
#define SX_GA_MAX_CELLS (200 * 1024) /* (Q+1)*(R+1) pointer bytes must fit one CTA's shared memory */

int sx_global_align(sx_ctx* ctx, const sx_ga_scores* scores, const sx_ga_batch* batch_host,
                    sx_ga_result* res_host /*[n]*/, uint32_t* cigar_host /*[n*max_ops]*/);
int sx_global_align_dev(sx_ctx* ctx, const sx_ga_scores* scores, const sx_ga_batch* batch_dev,
                        sx_ga_result* res_dev, uint32_t* cigar_dev);

/* ==========================================================================================
 * K2a  site_gl_germline
 *   replaces CleanPileupFilter + CleanPileupErrorProb + position_snp_call_pprob_digt:
 *   starling_common/PileupCleaner.cpp:30-75, blt_common/adjust_joint_eprob.cpp:60-243,
 *   blt_common/position_snp_call_pprob_digt.cpp:326-539, called from
 *   applications/starling/starling_pos_processor.cpp:178,254-267.
 *
 * A pileup batch is CSR over sites.  `calls` uses the reference's own 16-bit base_call layout
 * (blt_common/snp_pos_info.hh:109-118): bits 0-5 qscore, 6-9 base_id (A0 C1 G2 T3), 10 is_fwd_strand,
 * 11 is_neighbor_mismatch, 12 is_call_filter, 13 is_tier_specific_call_filter.
 * ======================================================================================== */
#define SX_CALL(q, base_id, fwd, nbr_mm, filt, tfilt) \
    ((uint16_t)(((q) & 63) | (((base_id) & 15) << 6) | (((fwd) & 1) << 10) | (((nbr_mm) & 1) << 11) | (((filt) & 1) << 12) | (((tfilt) & 1) << 13)))

typedef struct sx_pileup_batch {
    uint32_t n_sites;
    const uint32_t* site_off;   /* [n_sites+1] offsets into calls */
    const uint16_t* calls;      /* snp_pos_info::calls of every site, in pileup order */
    const uint32_t* t2_off;     /* [n_sites+1] offsets into t2_calls, or NULL (no tier2 data) */
    const uint16_t* t2_calls;   /* snp_pos_info::tier2_calls */
    const char* ref_base;       /* [n_sites] 'A','C','G','T' or 'N' */
    const uint8_t* ploidy;      /* [n_sites] 2 (diploid) or 1 (haploid); NULL = all 2 */
} sx_pileup_batch;

typedef struct sx_digt_result_set { /* diploid_genotype::result_set, position_snp_call_pprob_digt.hh:72-90 */
    double ref_pprob;
    uint32_t max_gt;
    int32_t snp_qphred;
    int32_t max_gt_qphred;
    int32_t pad;
} sx_digt_result_set;

typedef struct sx_digt_result { /* diploid_genotype, position_snp_call_pprob_digt.hh:39-110 */
    sx_digt_result_set genome;
    sx_digt_result_set poly;
    double strand_bias;
    float lhood[10];          /* ln P(pileup | gt), DIGT order AA CC GG TT AC AG AT CG CT GT (blt_util/digt.hh) */
    uint32_t phredLoghood[10];
    uint32_t ref_gt;
    uint32_t is_computed;     /* 0: early return (ref 'N', or all-ref site without is_always_test): fields are the reset() values */
    uint32_t n_used_calls;    /* calls left after CleanPileupFilter */
    uint32_t pad;
} sx_digt_result;

int sx_site_gl_germline(sx_ctx* ctx, const sx_pileup_batch* batch_host, int is_always_test,
                        sx_digt_result* out_host /*[n_sites]*/);
int sx_site_gl_germline_dev(sx_ctx* ctx, const sx_pileup_batch* batch_dev, int is_always_test,
                            sx_digt_result* out_dev);
/* the dependent error probs alone (adjust_joint_eprob), one float per *cleaned* call, CSR by out_off[n_sites+1] */
int sx_dependent_eprob(sx_ctx* ctx, const sx_pileup_batch* batch_host, uint32_t* out_off_host, float* de_host);

/* ==========================================================================================
 * K2b  site_gl_somatic
 *   replaces sscaller_strand_grid().position_somatic_snv_call(nepi,tepi,nepi_t2,tepi_t2,false,sgtg)
 *   applications/strelka/strelka_pos_processor.cpp:213-219 ->
 *   applications/strelka/position_somatic_snv_strand_grid.cpp:228-363,
 *   position_somatic_snv_strand_grid_lhood_cached.cpp:41-234, qscore_calculator.cpp:47-209.
 * ======================================================================================== */
typedef struct sx_ssnv_result { /* somatic_snv_genotype_grid + snv_result_set */
    float normal_lhood[30];  /* tier selected by snv_from_ntype_tier; DIGT_GRID order (strelka_digt_states.hh:89-98); 21..29 unused (0) */
    float tumor_lhood[30];
    float strandBias;
    uint32_t ref_gt;
    uint32_t is_computed;        /* 0: early return; nothing below is meaningful */
    uint32_t snv_tier;
    uint32_t snv_from_ntype_tier;
    uint32_t ntype;              /* NTYPE: REF 0, HOM 1, HET 2, CONFLICT 3 */
    uint32_t max_gt;
    int32_t qphred;              /* QSS */
    int32_t from_ntype_qphred;   /* QSS_NT */
    uint32_t normal_alt_id;
    uint32_t tumor_alt_id;
    uint32_t pad;
} sx_ssnv_result;

/* normal and tumor must have the same n_sites and ref_base; is_forced_output may be NULL (all 0);
 * tier2 evaluation happens when both batches carry t2_off */
int sx_site_gl_somatic(sx_ctx* ctx, const sx_pileup_batch* normal_host, const sx_pileup_batch* tumor_host,
                       const uint8_t* is_forced_output_host, sx_ssnv_result* out_host /*[n_sites]*/);
int sx_site_gl_somatic_dev(sx_ctx* ctx, const sx_pileup_batch* normal_dev, const sx_pileup_batch* tumor_dev,
                           const uint8_t* is_forced_output_dev, sx_ssnv_result* out_dev);

/* ==========================================================================================
 * K5  indel_gl
 *   replaces the per-read loop of getVariantAlleleGroupGenotypeLhoodsForSample
 *   starling_common/AlleleGroupGenotype.cpp:184-258 (updateGenotypeLogLhoodFromAlleleLogLhood :34-111,
 *   updateSupportingReadStats :122-152), with integrateOutMappingStatus
 *   (starling_common/readMappingAdjustmentUtil.hh:46-56) and get_het_observed_allele_ratio
 *   (starling_common/starling_indel_call_pprob_digt.cpp:40-71), called from
 *   applications/starling/starling_pos_processor.cpp:1335 (updateIndelLocusWithSampleInfo).
 *
 * Per locus: an orthogonal allele group of A non-reference indel alleles (1 <= A <= SX_INDEL_MAX_ALLELES) and,
 * per supporting read in readId order, the allele log-likelihoods the host takes out of the ReadPathScores maps
 * (getAlleleLogLhoodFromRead, OrthogonalVariantAlleleCandidateGroupUtil.cpp:132-196: index 0 = reference).
 * ======================================================================================== */
#define SX_INDEL_MAX_ALLELES 4
#define SX_INDEL_MAX_GT 15 /* (A+1)(A+2)/2 at A = 4 */

typedef struct sx_indel_batch {
    uint32_t n_loci;
    const uint32_t* read_off;       /* [n_loci+1] offsets into the per-read arrays */
    const uint32_t* lnp_off;        /* [n_loci+1] offsets into allele_lnp; a locus holds n_reads*(A+1) floats, read-major */
    const uint32_t* allele_off;     /* [n_loci+1] offsets into the per-allele arrays (A = allele_off[l+1]-allele_off[l]) */
    const uint8_t* ploidy;          /* [n_loci] callerPloidy 1 or 2 */
    const uint16_t* allele_del_len; /* per non-ref allele: IndelKey::delete_length() */
    const uint16_t* allele_ins_len; /* per non-ref allele: IndelKey::insert_length() */
    const float* allele_lnp;        /* ReadPathScores::score_t values: [read][0] = ref path, [read][1+a] = allele a */
    const uint16_t* read_length;    /* per read: ReadPathScores::read_length */
    const uint16_t* non_ambig;      /* per read: ReadPathScores::nonAmbiguousBasesInRead */
    const uint8_t* is_fwd;          /* per read: ReadPathScores::is_fwd_strand */
} sx_indel_batch;

typedef struct sx_indel_result {
    double gt_lhood[SX_INDEL_MAX_GT];                 /* genotypeLogLhood, VcfGenotypeUtil::getGenotypeIndex order (htsapi/vcf_util.hh:373-390) */
    uint16_t support[2][SX_INDEL_MAX_ALLELES + 2];    /* LocusSupportingReadStats: [rev=0|fwd=1][ref, alt1.., last = nonConfidentCount] */
    uint32_t n_gt;
} sx_indel_result;

int sx_indel_gl(sx_ctx* ctx, const sx_indel_batch* batch_host, sx_indel_result* out_host /*[n_loci]*/);
int sx_indel_gl_dev(sx_ctx* ctx, const sx_indel_batch* batch_dev, sx_indel_result* out_dev);

/* ==========================================================================================
 * K4  pileup_reads   (SURVEY 8f1: the producer of K2's input)
 *   replaces  starling_pos_processor_base::pileup_read_segment
 *   (starling_common/starling_pos_processor_base.cpp:1127-1421) called for every read buffered at a position
 *   (pileup_pos_reads :1096-1123), with create_mismatch_filter_map (starling_read_util.cpp:120-217),
 *   getReadAmbiguousEndLength (htsapi/bam_seq_read_util.cpp:29-54) and qphred_to_mapped_qphred (blt_util/qscore.hh:117).
 *
 * Input: the reads of one contig segment with their BEST alignment (the host keeps the decisions that need its containers:
 * is_any_nonovermax, the largest-indel-span check; realigned vs input alignment is K9's output when it is given the mapper's alignments),
 * in the order the reference piles them up (read-buffer order: see buffer_pos below).  Output: for every position of the report range the
 * column of base_call words in exactly that order -- the tier1 buffer (`calls`) and the tier2 buffer (`t2_calls`) of
 * pos_basecall_buffer::insert_pos_basecall -- i.e. an sx_pileup_batch ready for K2, plus the spanning-deletion and
 * sub-mapped read counts of each position.  Not produced: MAPQ tallies and the EVS feature accumulators (out of scope).
 * ======================================================================================== */
enum { SX_SEG_DELETE = 5, SX_SEG_SKIP = 6 }; /* K4 paths keep DELETE and SKIP apart: only a DELETE is a spanning deletion */

#define SX_PRF_FWD 0x01u        /* best_al.is_fwd_strand */
#define SX_PRF_TIER1 0x02u      /* rseg.is_tier1_mapping() */
#define SX_PRF_TIER1OR2 0x04u   /* rseg.is_tier1or2_mapping(); clear = sub-mapped read */
#define SX_PRF_PIN_FIRST 0x08u  /* rseg.get_segment_edge_pin().first  (an exon borders the leading edge) */
#define SX_PRF_PIN_SECOND 0x10u /* ... .second */
#define SX_PRF_SKIP 0x20u       /* buffered (it keeps its place in the order) but not piled up: a read that was not realigned and has no alignment
                                   with indels the caller handles (! is_any_nonovermax, :1147), or whose realignment left the stage buffer
                                   (is_invalid_realignment, :1171) */

typedef struct sx_pileup_read {
    uint32_t seq_off;  /* byte offset of the read's first packed byte in seq4 (reads start on byte boundaries) */
    uint32_t qual_off; /* byte offset of its first quality (one byte per base) */
    uint32_t seg_off;  /* first segment of its alignment path in `segs`; the path ends at the next read's seg_off */
    int32_t pos;       /* best_al.pos */
    uint16_t len;      /* rseg.read_size() */
    uint8_t mapq;
    uint8_t flags;     /* SX_PRF_* */
} sx_pileup_read;

typedef struct sx_pileup_opts { /* blt_options / starling_base_options fields read by the pileup */
    int32_t isBasecallQualAdjustedForMapq;         /* 1 */
    int32_t minBasecallErrorPhredProb;             /* 17 */
    uint32_t mismatchDensityFilterFlankSize;       /* 0 = filter off (blt_shared.hh:116-119) */
    uint32_t mismatchDensityFilterMaxMismatchCount;
    int32_t useTier2Evidence;                      /* 0 */
    int32_t tier2MismatchDensityFilterMaxMismatchCount; /* 10 */
    uint32_t minDistanceFromReadEdge;              /* 0 */
    uint32_t reserved_;
} sx_pileup_opts;

typedef struct sx_pileup_reads_batch {
    uint32_t n_reads;
    uint32_t n_segs;
    const sx_pileup_read* reads; /* [n_reads + 1]; sorted by pos; the sentinel carries the end offsets */
    const uint8_t* seq4;         /* BAM 4-bit packed bases */
    const uint8_t* qual;
    const sx_aln_seg* segs;      /* kinds MATCH, INSERT, DELETE, SKIP, SOFTCLIP, HARDCLIP */
    const char* ref;             /* reference_contig_segment: ASCII, ref[i] is contig position ref_begin + i; 'N' outside */
    int32_t ref_begin;
    uint32_t ref_len;
    int32_t report_begin, report_end; /* _reportRange, half open; output site i is position report_begin + i */
    const uint32_t* cand_snv;    /* sorted keys ((pos - report_begin) << 2) | base id: CandidateSnvBuffer::isCandidateSnvAnySample */
    uint32_t n_cand_snv;
    uint32_t max_ref_span;       /* >= the reference span of every read's alignment; the kernel tiles the range by windows >= this */
    uint32_t max_read_len;       /* >= every read's length (0 = unknown: the kernel's limit of 1024 is assumed) */
    uint32_t reserved_;
    sx_pileup_opts opts;
    /* The order key.  The reference piles reads up in read-buffer order -- rseg.buffer_pos = the MAPPER's alignment position minus its
     * unaligned prefix (starling_read_buffer.cpp:68-78, starling_read_util.cpp:30-35), read index within a position -- while a read
     * contributes through its best alignment, whose start a realignment may have moved.  buffer_pos[n_reads] (ascending; NULL: the
     * reads are ordered by reads[].pos itself) carries that key; max_pos_shift >= |reads[r].pos - buffer_pos[r]| for every read. */
    const int32_t* buffer_pos;
    uint32_t max_pos_shift;
    /* qual_bits 0 / 8: one byte per base.  4: dictionary-coded, two per byte, high nibble first, every read on a byte boundary (the
     * layout of seq4 and of sx_align_batch.qual with qual_bits 4); reads[].qual_off is then the offset of the read's first packed byte. */
    uint32_t qual_bits;
    uint8_t qual_dict[16];
} sx_pileup_reads_batch;

typedef struct sx_pileup_columns { /* caller-allocated; n_sites = report_end - report_begin */
    uint32_t* site_off;   /* [n_sites + 1] */
    uint16_t* calls;      /* [calls_capacity]   tier1 buffer, base_call words (blt_common/snp_pos_info.hh:109-118) */
    uint32_t* t2_off;     /* [n_sites + 1] */
    uint16_t* t2_calls;   /* [t2_capacity]      tier2 buffer */
    uint32_t* n_spandel;  /* [n_sites] insert_pos_spandel_count */
    uint32_t* n_submapped; /* [n_sites] insert_pos_submap_count */
    uint64_t calls_capacity, t2_capacity; /* in words; the total read bases of the batch always suffices for each */
} sx_pileup_columns;

void sx_default_pileup_opts(sx_pileup_opts* o);
/* SX_ERR_NOMEM if a capacity is too small (site_off / t2_off are still filled, so the caller can size and retry) */
int sx_pileup_reads(sx_ctx* ctx, const sx_pileup_reads_batch* batch_host, sx_pileup_columns* out_host);
int sx_pileup_reads_dev(sx_ctx* ctx, const sx_pileup_reads_batch* batch_dev, sx_pileup_columns* out_dev);

/* ==========================================================================================
 * K6  score_indels   (SURVEY 8f2: the consumer of K1's scores)
 *   replaces, per read segment that is a tier1 or tier2 mapping,
 *     the arg-max epilogue of scoreCandidateAlignments   starling_common/starling_read_align.cpp:1573-1593
 *       (ties by isFirstCandidateAlignmentPreferred :1352-1377, getExtraPathInfo :1295-1320, getCandidateIndelCount :1324-1336)
 *     score_indels                                        starling_common/starling_read_align_score_indels.cpp:454-1079
 *       with late_indel_normalization_filter :281-450, is_equiv_candidate :247-276, is_first_indel_dominant :285-300,
 *       get_alignment_indel_bp_overlap :131-234, which_interfering_indel :100-118, is_indel_conflict (indel_util.cpp:29-45),
 *       IndelBuffer::rangeIterator (IndelBuffer.cpp:76-91), get_soft_clip_alignment_range (alignment_util.cpp:45-55),
 *       getLowestFwdReadPosForRefRange (alignment_util.cpp:272-302), ReadPathScores::insertAlt (IndelData.cpp:42-68)
 *   called from scoreCandidateAlignmentsAndIndels (starling_read_align.cpp:1750-1812).
 *
 * Input: K1's scores where K1 left them (device, one double per candidate alignment) plus the small integer description the
 * reference's containers hold: per region the IndelBuffer entries of its window in IndelKey order, per alignment its path and the
 * keys of its indels.  Output: what score_indels writes into the IndelBuffer -- one record per (read, evaluated indel): the
 * ReadPathScores entry (read_path_lnp[readId]) or the suboverlap mark -- in IndelKey order per read.
 * The std::map / std::set bookkeeping of the reference becomes per-read maxima over its alignments.
 * ======================================================================================== */
#define SX_INDEL_TYPE_INDEL 0u    /* INDEL::INDEL */
#define SX_INDEL_TYPE_MISMATCH 1u /* INDEL::MISMATCH (never evaluated, never "interfering", conflicts without the +1 margin) */
#define SX_IKF_CANDIDATE 0x1u     /* indelBuffer.isCandidateIndel(key) */

typedef struct sx_indel_key { /* one IndelBuffer entry; a region's entries are in IndelKey order (IndelKey.hh:53-76) */
    int32_t pos;
    uint16_t del_len;          /* IndelKey::delete_length() */
    uint16_t ins_len;          /* IndelKey::insert_length() */
    uint32_t ins_id;           /* within a region: equal insert sequences <=> equal ins_id (0 = empty) */
    uint8_t type;              /* SX_INDEL_TYPE_* ; breakends are not supported (SX_ERR_UNSUPPORTED) */
    uint8_t flags;             /* SX_IKF_* */
    uint16_t pad;
    double ref_to_indel_lnp;   /* getSampleData(sample).getErrorRates().refToIndelErrorProb.getLogValue() */
    double indel_to_ref_lnp;   /* ... indelToRefErrorProb.getLogValue() */
} sx_indel_key;

#define SX_SIF_FWD 0x01u        /* cal.al.is_fwd_strand (the same for every candidate alignment of a read) */
#define SX_SIF_TIER1 0x02u      /* rseg.is_tier1_mapping(); clear = tier2 (reads that are neither are not sent) */
#define SX_SIF_INCOMPLETE 0x04u /* is_incomplete_search (starling_read_align.cpp:2100) */

typedef struct sx_score_indels_opts {
    uint32_t max_indel_size;         /* opt.maxIndelSize, 49 */
    uint32_t upstream_oligo_size;    /* 0 */
    int32_t min_read_bp_flank;       /* sample_opt.min_read_bp_flank, 5 */
    int32_t is_smoothed_alignments;  /* 1 */
    double smoothed_lnp_range;       /* std::log(10.) */
} sx_score_indels_opts;

typedef struct sx_score_indels_batch {
    uint32_t n_regions, n_reads, n_alns, n_keys;
    const uint32_t* region_read_off; /* [n_regions + 1] the reads of a region */
    const uint32_t* region_key_off;  /* [n_regions + 1] its IndelBuffer window: every entry a rangeIterator() over any of its
                                        alignments can visit, at most 65535 per region */
    const sx_indel_key* keys;        /* [n_keys] */
    const uint32_t* aln_off;         /* [n_reads + 1] read r owns scores lnp[aln_off[r] .. aln_off[r+1]) -- K1's alignment order,
                                        which is the iteration order of std::set<CandidateAlignment> */
    const int32_t* aln_pos;          /* [n_alns] cal.al.pos */
    const uint32_t* aln_seg_off;     /* [n_alns + 1] */
    const sx_aln_seg* segs;          /* cal.al.path: MATCH (also SEQ_MATCH / SEQ_MISMATCH), INSERT, SX_SEG_DELETE, SOFTCLIP, HARDCLIP;
                                        flags unused; SX_SEG_SKIP is outside score_indels' domain (its assert, :176) */
    const uint32_t* aln_key_off;     /* [n_alns + 1] */
    const uint16_t* aln_keys;        /* cal.getIndels(): indices into the region's window, ascending */
    const uint16_t* read_len;        /* [n_reads] rseg.read_size() */
    const uint16_t* non_ambig;       /* [n_reads] bases of the segment that are not 'N' (:866-875) */
    const uint16_t* full_len;        /* [n_reads] rseg.full_read_size();   NULL: == read_len  */
    const uint16_t* full_off;        /* [n_reads] rseg.full_read_offset(); NULL: 0            */
    const uint8_t* read_flags;       /* [n_reads] SX_SIF_* */
    const uint32_t* rec_off;         /* [n_reads + 1] output slots of each read; a read never needs more than the number of
                                        window entries with pos in [min soft-clip begin - max_indel_size, max soft-clip end) */
    sx_score_indels_opts opts;
} sx_score_indels_batch;

#define SX_RIS_SCORED 0x1u        /* read_path_lnp[readId] = ReadPathScores(...) (:1069) */
#define SX_RIS_SUBOVERLAP 0x2u    /* suboverlap_tier{1,2}_read_ids.insert(readId) (:640-648); the tier is the read's */

typedef struct sx_read_indel_score { /* 32 bytes */
    uint16_t key;            /* index into the region's window */
    uint8_t flags;           /* SX_RIS_* */
    uint8_t n_alt;           /* ReadPathScores::alt_indel.size(), <= 2 */
    int16_t read_pos;        /* ReadPathScores::read_pos */
    int16_t dist_from_edge;  /* ReadPathScores::distanceFromClosestReadEdge */
    float ref_lnp;           /* ReadPathScores::ref   */
    float indel_lnp;         /* ReadPathScores::indel */
    uint16_t alt_key[2];     /* alt_indel[i].first, as window index */
    float alt_lnp[2];        /* alt_indel[i].second */
    uint32_t pad;
} sx_read_indel_score;

typedef struct sx_score_indels_out { /* caller-allocated */
    sx_read_indel_score* recs; /* [rec_off[n_reads]]; read r's records are recs[rec_off[r] .. rec_off[r] + n_rec[r]) */
    uint32_t* n_rec;           /* [n_reads] */
    uint32_t* max_aln;         /* [n_reads] maxCandAlignmentPtr after scoreCandidateAlignments (:1593), as alignment index */
    uint32_t* eval_aln;        /* [n_reads] ... after late_indel_normalization_filter (:430-449): the alignment score_indels evaluates */
} sx_score_indels_out;

void sx_default_score_indels_opts(sx_score_indels_opts* o);
/* lnp: the K1 scores, [n_alns].  Host variant copies everything; the _dev variant takes device pointers inside *batch_dev,
 * lnp_dev (typically the buffer sx_score_alignments_dev just wrote) and *out_dev. */
int sx_score_indels(sx_ctx* ctx, const sx_score_indels_batch* batch_host, const double* lnp_host, sx_score_indels_out* out_host);
int sx_score_indels_dev(sx_ctx* ctx, const sx_score_indels_batch* batch_dev, const double* lnp_dev, sx_score_indels_out* out_dev);

/* ==========================================================================================
 * K7  enumerate_alignments   (SURVEY 8a row a3 / 8f3: the producer of K1's and K6's input)
 *   replaces  getCandidateAlignments           starling_common/starling_read_align.cpp:1816-1994
 *   with      candidate_alignment_search       :857-1277  (the recursive toggle search)
 *             make_start_pos_alignment         :393-584,  get_end_pin_start_pos :593-719
 *             add_indels_in_range              :311-375,  sort_remove_only_indels_last :724-749
 *             addKeysToCandidateAlignment      :789-804,  HaplotypeStatus / getCurIndelHaplotypeIds :56-179, :811-849
 *   and the container semantics around them: std::set<CandidateAlignment> (CandidateAlignment.hh:38-49,
 *   alignment.hh:73-91, align_path.hh:184-196), IndelBuffer::rangeIterator (IndelBuffer.cpp:76-91),
 *   is_range_{intersect,adjacent}_indel_breakpoints (indel_util.cpp:49-76), is_indel_conflict (:29-45),
 *   starling_align_limit::get_max_toggle (starling_align_limit.hh:41-52).
 *
 * Input, per region (the reads buffered around one realignment window): the IndelBuffer window in IndelKey order (the
 * sx_indel_key table K6 reads, plus what the search consults of IndelData: SX_IKF_NOT_DISCOVERED / SX_IKF_FORCED_OUTPUT and the
 * optional sx_key_hap rows); per read the NORMALIZED input alignment realignAndScoreRead hands to getCandidateAlignments
 * (:2049-2057: edge indels matchified, soft clips matchified -- by the host, or by K7g sx_realign_gates from the mapper's alignment),
 * the window entries that alignment already contains (getAlignmentIndels(..., includeMismatches = true), CandidateAlignment.cpp:58-173,
 * as window indices -- by the host, or by K7a sx_alignment_indels from the read bases and the reference where K1 keeps them) and the
 * non-candidate entries this read is an observation of (is_usable_indel :289-305).  The chain K7g -> K7a -> K7 -> K7b -> K1 -> K6 / K9 is
 * realignAndScoreRead for a batch of reads with every intermediate in device memory.
 * Output, per read: the std::set<CandidateAlignment> in ITS iteration order -- which is K1's and K6's alignment order -- as CSR
 * arrays shaped like sx_score_indels_batch's (aln_pos / path segments / cal.getIndels() as window indices) + the leading / trailing
 * edge keys + the warn flags that make is_incomplete_search.
 *
 * Path segments carry the reference's own ALIGNPATH::align_t values (SX_AP_*, blt_util/align_path.hh:36-48) because the set's
 * order compares them numerically.
 * ======================================================================================== */
enum { SX_AP_MATCH = 1, SX_AP_INSERT = 2, SX_AP_DELETE = 3, SX_AP_SKIP = 4, SX_AP_SOFT_CLIP = 5, SX_AP_HARD_CLIP = 6, SX_AP_PAD = 7, SX_AP_SEQ_MATCH = 8, SX_AP_SEQ_MISMATCH = 9 };

#define SX_IKF_NOT_DISCOVERED 0x2u /* IndelData::status.notDiscoveredFromReads */
#define SX_IKF_FORCED_OUTPUT 0x4u  /* IndelData::isForcedOutput */
#define SX_ENUM_MAX_SAMPLES 4
#define SX_NO_KEY 0xFFFFu          /* leading_indel_key / trailing_indel_key of type INDEL::NONE */

typedef struct sx_key_hap { /* the active-region phasing data of one window entry (IndelData.hh) */
    int32_t active_region_id;                  /* IndelData::activeRegionId, < 0 = none */
    int8_t haplotype_id[SX_ENUM_MAX_SAMPLES];  /* IndelSampleData::haplotypeId per sample (0, 1, 2, 3) */
    uint8_t bypass_mask;                       /* bit s: IndelSampleData::isHaplotypingBypassed of sample s */
    uint8_t pad[3];
} sx_key_hap;

#define SX_ENUM_ST_ORIGIN_SKIP 0x01u /* mca_warnings::origin_skip  (:1248)                                      */
#define SX_ENUM_ST_MAX_TOGGLE 0x02u  /* mca_warnings::max_toggle_depth (:971, :1135); either => is_incomplete_search (:2100) */
#define SX_ENUM_ST_EXCEPTION 0x04u   /* the reference throws blt_exception for this read (:446, :493, :572, :658, :676, :709, :1872);
                                        no alignments are returned for it */
#define SX_ENUM_ST_LIMIT 0x08u       /* more indels / alignments / segments than this build's per-read scratch holds; no alignments are
                                        returned and the caller runs the read through its own getCandidateAlignments */

typedef struct sx_enum_opts {
    uint32_t max_indel_size;             /* opt.maxIndelSize, 49 (rangeIterator) */
    int32_t max_read_indel_toggle;       /* opt.max_read_indel_toggle, 5 (starling_base_shared.hh:139) */
    double max_candidate_indel_density;  /* 0.15 (:145) */
    uint32_t n_max_toggle;               /* starling_align_limit::_max_toggle.size() */
    uint8_t max_toggle[100];             /* ... its values for opt.max_realignment_candidates = 5000 (starling_align_limit.cpp:64-88);
                                            indices >= n_max_toggle mean 1 */
    int32_t is_haplotyping_enabled;      /* opt.isHaplotypingEnabled */
    uint32_t n_samples;                  /* opt.getSampleCount(), <= SX_ENUM_MAX_SAMPLES */
    uint32_t sample_id;                  /* the sample the reads belong to */
    uint32_t max_alns_per_read;          /* scratch capacity per read, 0 = 64; reads that need more get SX_ENUM_ST_LIMIT */
    uint32_t flags;                      /* SX_ENUM_F_* */
} sx_enum_opts;

/* SX_ENUM_F_FAST (the default of sx_default_enum_opts): ordinary reads (<= 11 nested toggles, <= 16 alignments) search in per-lane-interleaved
 * local memory, the others in a global arena; every read is searched ONCE, its alignments appended to a log and gathered into read order
 * after the scan.  flags = 0 selects the first launch plan (per-thread arena, count / scan / write: the search runs twice) -- same results,
 * several times slower on cfg2-shaped loci; kept as a cross-check of the fast plan. */
#define SX_ENUM_F_FAST 0x1u

typedef struct sx_enum_batch {
    uint32_t n_regions, n_reads, n_keys;
    const uint32_t* region_read_off;   /* [n_regions + 1] */
    const uint32_t* region_key_off;    /* [n_regions + 1] the IndelBuffer window of a region, IndelKey order, <= 65535 entries */
    const sx_indel_key* keys;          /* [n_keys] (the error-rate fields are not read) */
    const sx_key_hap* key_hap;         /* [n_keys] or NULL: no entry lies in an active region */
    const int32_t* realign_begin;      /* [n_regions] realign_buffer_range (starling_pos_processor_base.cpp:735) */
    const int32_t* realign_end;        /* [n_regions] */
    const int32_t* in_pos;             /* [n_reads] normalizedInputAlignment.pos (>= 0, :2062) */
    const uint32_t* in_seg_off;        /* [n_reads + 1] */
    const sx_aln_seg* in_segs;         /* normalizedInputAlignment.path, kind = SX_AP_* */
    const uint32_t* in_key_off;        /* [n_reads + 1] */
    const uint16_t* in_keys;           /* window indices of getAlignmentIndels(cal, ref, rseg, maxIndelSize, true), ascending; mismatches
                                          that are not window entries are dropped (:1865), as the reference does; SX_NO_KEY = an indel of
                                          the alignment that is no window entry: the read gets SX_ENUM_ST_EXCEPTION (:1866-1872).  K7a
                                          (sx_alignment_indels) computes this array and the two below on the device */
    const uint32_t* use_key_off;       /* [n_reads + 1] */
    const uint16_t* use_keys;          /* window indices of the entries whose tier1/tier2/submap/noise read-id sets hold this read */
    const uint16_t* in_lead_key;       /* [n_reads] leading_indel_key of getCandidateAlignment (:1481-1522) as window index, or SX_NO_KEY */
    const uint16_t* in_trail_key;      /* [n_reads] trailing_indel_key */
    const uint16_t* read_len;          /* [n_reads] rseg.read_size() */
    const uint8_t* gate;               /* [n_reads] or NULL: K7g's output; a read whose SX_GATE_REALIGN bit is clear is answered with no alignments
                                          and status 0 (realignAndScoreRead returned before the search), by K7a with no keys */
    sx_enum_opts opts;
} sx_enum_batch;

typedef struct sx_enum_out { /* caller-allocated, capacities stated */
    uint32_t cap_alns, cap_segs, cap_keys;
    uint32_t* totals;        /* [3] alignments, segments, keys the batch produces (written even when a capacity is too small) */
    uint32_t* aln_off;       /* [n_reads + 1] */
    uint8_t* status;         /* [n_reads] SX_ENUM_ST_* */
    int32_t* aln_pos;        /* [cap_alns] */
    uint32_t* aln_seg_off;   /* [cap_alns + 1] */
    sx_aln_seg* segs;        /* [cap_segs] kind = SX_AP_* */
    uint32_t* aln_key_off;   /* [cap_alns + 1] */
    uint16_t* aln_keys;      /* [cap_keys] cal.getIndels() as ascending window indices */
    uint16_t* aln_lead_key;  /* [cap_alns] */
    uint16_t* aln_trail_key; /* [cap_alns] */
} sx_enum_out;

#define SX_ERR_CAPACITY (-8) /* an sx_enum_out capacity is too small: totals[] says what the batch needs */

void sx_default_enum_opts(sx_enum_opts* o);
int sx_enumerate_alignments(sx_ctx* ctx, const sx_enum_batch* batch_host, sx_enum_out* out_host);
int sx_enumerate_alignments_dev(sx_ctx* ctx, const sx_enum_batch* batch_dev, sx_enum_out* out_dev /* device pointers; totals too */);

/* ==========================================================================================
 * K7a  alignment_indels   (the first step of getCandidateAlignments: which window entries the input alignment already contains)
 *   replaces  getCandidateAlignment              starling_common/starling_read_align.cpp:1481-1522 (the edge keys)
 *             getAlignmentIndels(cal, ref, rseg, opt.maxIndelSize, includeMismatches = true)
 *                                                starling_common/CandidateAlignment.cpp:58-173, called at starling_read_align.cpp:1857
 *   i.e. the per-BASE host loop in front of K7: every aligned read base is compared with the reference (a mismatch that is a
 *   window entry is a key of the alignment), every insert / delete / swap of the path is looked up by position, lengths and
 *   inserted bases.
 *
 * Input: the sx_enum_batch being prepared (window, region offsets, in_pos / in_segs / read_len), the read bases and reference
 * windows where K1 keeps them (the wide formats: seq4 = BAM 4-bit codes, reads of a region back to back from regions[g].seq_off,
 * each read starting on a byte boundary; ref = ASCII from regions[g].ref_off, positions outside read as 'N') and the insert
 * sequences of the window entries.  Output: the batch's own in_key_off / in_keys / in_lead_key / in_trail_key arrays.  An indel of
 * the alignment that is no window entry is written as SX_NO_KEY: K7 then answers the read as the reference does (blt_exception,
 * :1866-1872 -> SX_ENUM_ST_EXCEPTION); a mismatch that is no window entry is dropped (:1865).
 * ======================================================================================== */
typedef struct sx_prep_out { /* caller-allocated */
    uint32_t cap_keys;
    uint32_t* totals;        /* [1] keys produced (written even when cap_keys is too small: SX_ERR_CAPACITY) */
    uint32_t* in_key_off;    /* [n_reads + 1] */
    uint16_t* in_keys;       /* [cap_keys] ascending per read */
    uint16_t* in_lead_key;   /* [n_reads] */
    uint16_t* in_trail_key;  /* [n_reads] */
} sx_prep_out;

int sx_alignment_indels(sx_ctx* ctx, const sx_enum_batch* batch_host, const sx_region* regions_host /*[n_regions + 1]*/, const uint8_t* seq4_host, const char* ref_host,
                        const uint32_t* key_ins_off_host, const char* key_ins_host, sx_prep_out* out_host);
int sx_alignment_indels_dev(sx_ctx* ctx, const sx_enum_batch* batch_dev, const sx_region* regions_dev, const uint8_t* seq4_dev, const char* ref_dev,
                            const uint32_t* key_ins_off_dev, const char* key_ins_dev, sx_prep_out* out_dev);

/* ==========================================================================================
 * K7g  realign_gates   (the front of realignAndScoreRead, starling_common/starling_read_align.cpp:2045-2062: which reads go into the
 *   search at all, and with which input alignment)
 *   replaces  alignment::is_realignable / is_overmax        starling_common/alignment.cpp:34-50
 *             check_for_candidate_indel_overlap             starling_read_align.cpp:222-283 (get_alignment_zone, alignment_util.cpp:76-85)
 *             normalizeInputAlignmentIndels                 :2000-2021 (matchify_edge_indels = remove_edge_deletions + matchify_edge_insertions,
 *                                                           alignment_util.cpp:89-198; is_edge_readref_len_segment, align_path.cpp:827-846)
 *             matchify_edge_soft_clip                       alignment_util.cpp:203-207 (:2051-2057), the negative-start test :2062
 * Input: the mapper's alignment of every read (pos + path, SX_AP_* kinds) in the CSR the K7 batch will use, the window, the realignment
 * range.  Output: gate[r] and -- for the reads that pass -- the normalized alignment written into the same CSR slots (a normalized path
 * is never longer than the original; unused slots become zero-length HARD_CLIP segments, which the search strips like any clip).
 * ======================================================================================== */
#define SX_GATE_REALIGN 0x01u      /* the read goes on to getCandidateAlignments */
#define SX_GATE_SOFT_CLIPPED 0x02u /* isSoftClippedInputAlignment (:2051): the caller's retain-optimal-soft-clipping test wants to know */

typedef struct sx_gate_batch {
    uint32_t n_regions, n_reads;
    const uint32_t* region_read_off;  /* [n_regions + 1] */
    const uint32_t* region_key_off;   /* [n_regions + 1] */
    const sx_indel_key* keys;         /* window entries (pos, lengths, type, SX_IKF_CANDIDATE) */
    const int32_t* realign_begin;     /* [n_regions] */
    const int32_t* realign_end;
    const int32_t* raw_pos;           /* [n_reads] rseg.getInputAlignment().pos */
    const uint32_t* seg_off;          /* [n_reads + 1] */
    const sx_aln_seg* raw_segs;       /* rseg.getInputAlignment().path */
    const uint16_t* read_len;         /* [n_reads] rseg.read_size() */
    const uint8_t* pin_flags;         /* [n_reads] or NULL: bit 0 / 1 = rseg.get_segment_edge_pin().first / .second */
    uint32_t max_indel_size;          /* opt.maxIndelSize */
} sx_gate_batch;

typedef struct sx_gate_out { /* caller-allocated */
    uint8_t* gate;        /* [n_reads] SX_GATE_* */
    int32_t* in_pos;      /* [n_reads] normalizedInputAlignment.pos */
    sx_aln_seg* in_segs;  /* [seg_off[n_reads]] normalizedInputAlignment.path in the slots of the raw one */
} sx_gate_out;

int sx_realign_gates(sx_ctx* ctx, const sx_gate_batch* batch_host, sx_gate_out* out_host);
int sx_realign_gates_dev(sx_ctx* ctx, const sx_gate_batch* batch_dev, sx_gate_out* out_dev);

/* ==========================================================================================
 * K7b  link_alignments   (K7's output -> K1's alignment description; keeps the chain K7 -> K1 -> K6 in device memory)
 *   replaces the per-alignment host work in front of K1: the segment walk of scoreCandidateAlignment
 *   (starling_common/starling_read_align_score.cpp:289-499) with every container look-up resolved --
 *   getMatchingIndelKey :177-224 (which key of cal.getIndels(), or which edge key, a path gap stands for), the insert
 *   sequence each inserted segment is scored against incl. the leading-edge tail rule :334-338 / :394-398, and
 *   IndelBuffer::isCandidateIndel :473-475 (SX_SEGF_NONCANDIDATE) -- i.e. what sx::ReadAlignBatch::addCandidateAlignment
 *   does for host-built batches.
 *
 * Input: the sx_enum_batch K7 read (window keys; reads of a region are consecutive), K7's sx_enum_out and the insert
 * sequences of the window entries.  Output: the alignment part of an sx_align_batch -- alns[] (read = the K7 read
 * index, so the caller's read pools must list the reads in K7's order), segs[] (sx_aln_seg; '=' as MATCH, 'X' and swaps
 * as INSERT + REFSKIP), ins[] -- laid out under K1's staging rule (every region's first segment index a multiple of 8
 * with no-op HARDCLIP pads, its first insert byte a multiple of 16), and aln_begin / seg_begin / ins_begin of regions[]
 * (the caller fills the read / quality / reference fields of the same records).  Alignment order is preserved, so
 * lnp[a] of K1 is the score of K7's alignment a and of K6's alignment a.
 * ======================================================================================== */
typedef struct sx_link_out { /* caller-allocated */
    uint32_t cap_segs, cap_ins;
    uint32_t* totals;     /* [2] segments and insert-pool bytes produced (written even when a capacity is too small) */
    sx_region* regions;   /* [n_regions + 1] in/out, incl. the sentinel */
    sx_aln* alns;         /* [n_alns + 1] n_alns = the enumeration's totals[0] */
    sx_aln_seg* segs;     /* [cap_segs]; leave 16 entries beyond totals[0] for K1's slack (filled with no-op segments where they fit) */
    char* ins;            /* [cap_ins + SX_POOL_SLACK] */
    sx_aln_seg* k6_segs;  /* NULL, or [the enumeration's totals[1]]: K7's segments with K6's kinds (MATCH for '=' / 'X', SX_SEG_DELETE,
                             SX_SEG_SKIP, ...), index for index -- with K7's other arrays this is sx_score_indels_batch's alignment part */
} sx_link_out;

/* key_ins_off[n_keys + 1] / key_ins: the insert sequence of window entry k is key_ins[key_ins_off[k] .. key_ins_off[k+1]).
 * n_alns: the enumeration's totals[0] (host value).  SX_ERR_CAPACITY: totals[] says what is needed.  A path whose gap matches no
 * key of its alignment (the reference's assert(isFound), :222) fails the call with SX_ERR_ARG. */
int sx_link_alignments(sx_ctx* ctx, const sx_enum_batch* batch_host, const sx_enum_out* enum_host, uint32_t n_alns, const uint32_t* key_ins_off_host,
                       const char* key_ins_host, sx_link_out* out_host);
int sx_link_alignments_dev(sx_ctx* ctx, const sx_enum_batch* batch_dev, const sx_enum_out* enum_dev, uint32_t n_alns, const uint32_t* key_ins_off_dev,
                           const char* key_ins_dev, sx_link_out* out_dev);

/* ==========================================================================================
 * K9  choose_realignment   (SURVEY 8a row a2, second half: from the scores to rseg.realignment -- the alignment the pileup uses)
 *   replaces the tail of scoreCandidateAlignments   starling_common/starling_read_align.cpp:1573-1741:
 *     the arg-max with isFirstCandidateAlignmentPreferred :1573-1593 (:1352-1377), the smooth pool :1659-1683 (every alignment within
 *     smoothed_lnp_range of the maximum, and among them the preferred one), finishRealignment :1411-1450 with
 *     getClippedAlignmentFromTopAlignmentPool (starling_read_align_clipper.cpp:340-424: read positions on which the alignments of the
 *     pool disagree are soft-clipped off the ends of the chosen one; soft_clip_alignment :255-338).
 *   Not covered: reads with an exon edge pin (rseg.get_segment_edge_pin(), RNA: :1600-1657) and the retain-optimal-soft-clipping test
 *   (:1700-1737, switched on by the RNA workflow only) -- such reads are reported SX_REALIGN_ST_UNSUPPORTED and stay with the caller.
 *
 * Input: the candidate alignments in K7's output arrays (reference path kinds, set order) with K1's scores, the window (candidacy
 * counts of the preference rule), per read its length.  Output, per read: the realignment as (pos, path segments) -- exactly what K4
 * takes as a read's best alignment -- in a CSR whose slots are reserved from the longest path of the read (+2 for the clips).
 * ======================================================================================== */
#define SX_REALIGN_ST_REALIGNED 0x01u   /* rseg.is_realigned = true, realignment written */
#define SX_REALIGN_ST_UNSUPPORTED 0x02u /* pinned read: left to the caller */
#define SX_REALIGN_ST_LIMIT 0x04u       /* read longer than this build's 1024 bases */
#define SX_REALIGN_ST_BADPATH 0x08u     /* "Can't handle cigar code" / a path that does not cover the read (the reference would throw / assert) */

typedef struct sx_realign_batch {
    uint32_t n_regions, n_reads, n_alns;
    const uint32_t* region_read_off;  /* [n_regions + 1] */
    const uint32_t* region_key_off;   /* [n_regions + 1] */
    const sx_indel_key* keys;         /* window entries (flags: SX_IKF_CANDIDATE) */
    const uint32_t* aln_off;          /* [n_reads + 1]  -- K7's output arrays from here on */
    const int32_t* aln_pos;
    const uint32_t* aln_seg_off;      /* [n_alns + 1] */
    const sx_aln_seg* segs;           /* kind = SX_AP_* */
    const uint32_t* aln_key_off;      /* [n_alns + 1] */
    const uint16_t* aln_keys;
    const uint16_t* read_len;         /* [n_reads] */
    const uint8_t* pin_flags;         /* [n_reads] or NULL: nonzero = the read has an edge pin */
    int32_t is_smoothed_alignments;   /* opt.is_smoothed_alignments, 1 */
    int32_t k4_kinds;                 /* 0: output kinds are SX_AP_* (the reference's path); 1: K4's segment kinds (SX_SEG_*, '=' / 'X' as MATCH) */
    double smoothed_lnp_range;        /* std::log(10.) */
    /* Optional (all three NULL or all three set): rseg.getInputAlignment() of every read, SX_AP_* kinds.  With them the output is
     * read_segment::getBestAlignment() (starling_read_segment.hh:134-138) of EVERY read -- the realignment where one was chosen, the
     * mapper's alignment otherwise (status without SX_REALIGN_ST_REALIGNED) -- i.e. K4's input for the whole batch; a read's slots
     * are then reserved from max(longest candidate path + 2, its input path). */
    const int32_t* raw_pos;           /* [n_reads] */
    const uint32_t* raw_seg_off;      /* [n_reads + 1] */
    const sx_aln_seg* raw_segs;
} sx_realign_batch;

typedef struct sx_realign_out { /* caller-allocated */
    uint32_t cap_segs;
    uint32_t* totals;        /* [1] segment slots reserved (written even when cap_segs is too small: SX_ERR_CAPACITY) */
    uint32_t* seg_off;       /* [n_reads + 1] read r's slots are segs[seg_off[r] .. seg_off[r+1]); the first n_seg[r] hold the path, the rest are
                                zero-length HARD_CLIP pads */
    int32_t* pos;            /* [n_reads] realignment.pos */
    uint16_t* n_seg;         /* [n_reads] */
    uint8_t* status;         /* [n_reads] SX_REALIGN_ST_* (0: a read without candidate alignments) */
    uint32_t* best_aln;      /* [n_reads] smooth_cal_ptr as alignment index (UINT32_MAX: none) */
    sx_aln_seg* segs;        /* [cap_segs] */
} sx_realign_out;

int sx_choose_realignment(sx_ctx* ctx, const sx_realign_batch* batch_host, const double* lnp_host, sx_realign_out* out_host);
int sx_choose_realignment_dev(sx_ctx* ctx, const sx_realign_batch* batch_dev, const double* lnp_dev, sx_realign_out* out_dev);

/* ==========================================================================================
 * process_window   (the READ_BUFFER and POST_ALIGN stages of starling_pos_processor_base::process_pos for a window of positions, with
 *   every intermediate in device memory)
 *   replaces  align_pos                         starling_common/starling_pos_processor_base.cpp:732-773
 *                                               (realignAndScoreRead, starling_read_align.cpp:2025-2127, per buffered read segment that is a
 *                                               tier1 / tier2 mapping)
 *             pileup_pos_reads                  :1107-1123 (pileup_read_segment :1127-1421 per read, in read-buffer order, each read through
 *                                               read_segment::getBestAlignment, starling_read_segment.hh:134-138)
 *             computeSampleDiploidSiteGenotype  applications/starling/starling_pos_processor.cpp:254-267 per position (optional)
 *   as the chain  K7g -> K7a -> K7 -> K7b -> K1 -> K6 + K9 -> K4 -> K2a  on ONE description of the window: the reads in read-buffer order
 *   with the MAPPER's alignments, bases and qualities, the IndelBuffer entries around them, the reference.
 *
 * Input (device pointers; the struct itself is host): the union of what the chain's stages read --
 *   regions of reads (the reads buffered around one realignment window share its IndelBuffer entries: sx_enum_batch's region arrays),
 *   per read the mapper's alignment (SX_AP_* kinds), length, SX_PRF_* flags, MAPQ and the non-candidate entries it is an observation of,
 *   the read / quality / reference pools where K1 keeps them (wide base and reference formats; qualities one byte per base or 4-bit
 *   dictionary codes): `regions[g]` carries seq_off / qual_off / read_begin / ref_off / ref_begin / ref_len of region g (its alignment
 *   fields are filled by the link step: the array is in/out), and `ref` is ONE contig segment -- ref[i] is contig position ref_begin + i,
 *   so regions[g].ref_off == regions[g].ref_begin - ref_begin (a multiple of 16) --, which is also the reference the pile-up reads.
 * Output: per read the gate / search / realignment status and its best alignment (pos + path in K4's kinds), score_indels' records,
 *   the pile-up columns of [report_begin, report_end) and -- with do_site_gl -- one sx_digt_result per position.
 *   Any output pointer may be NULL: the result then stays in the context's own buffers (the next stage still reads it).
 * Reads the search leaves to the caller are reported, never silently dropped: SX_ENUM_ST_EXCEPTION (the reference throws), SX_ENUM_ST_LIMIT
 *   (more than 64 indels / 32 segments / 24 keys in one search; the alignment count itself is bounded like the reference's, by
 *   enum_opts.max_alns_per_read = 5000), SX_REALIGN_ST_UNSUPPORTED (exon edge pins).  Such reads are piled up with the mapper's alignment.
 * ======================================================================================== */
typedef struct sx_window_batch {
    uint32_t n_regions, n_reads, n_keys;
    const uint32_t* region_read_off;   /* [n_regions + 1] */
    const uint32_t* region_key_off;    /* [n_regions + 1] */
    const sx_indel_key* keys;          /* [n_keys] incl. the error-rate fields score_indels reads */
    const sx_key_hap* key_hap;         /* [n_keys] or NULL */
    const uint32_t* key_ins_off;       /* [n_keys + 1] */
    const char* key_ins;
    const int32_t* realign_begin;      /* [n_regions] */
    const int32_t* realign_end;
    const int32_t* raw_pos;            /* [n_reads] rseg.getInputAlignment().pos; the reads are in READ-BUFFER order (ascending
                                          get_alignment_buffer_pos, read index within a position) */
    const uint32_t* raw_seg_off;       /* [n_reads + 1] */
    const sx_aln_seg* raw_segs;        /* SX_AP_* kinds */
    const uint16_t* read_len;          /* [n_reads] */
    const uint8_t* read_flags;         /* [n_reads] SX_PRF_* */
    const uint8_t* mapq;               /* [n_reads] */
    const uint32_t* use_key_off;       /* [n_reads + 1] */
    const uint16_t* use_keys;
    const uint32_t* rec_off;           /* [n_reads + 1] score_indels' output slots per read (sx_score_indels_batch.rec_off) */
    sx_region* regions;                /* [n_regions + 1] in/out */
    const uint8_t* seq4;
    const uint8_t* qual;
    const char* ref;
    uint64_t seq4_bytes, qual_bytes, ref_bytes;
    uint32_t qual_bits;                /* 0 / 8, or 4 with qual_dict */
    uint8_t qual_dict[16];
    int32_t ref_begin;                 /* contig position of ref[0] */
    int32_t report_begin, report_end;  /* the positions piled up (and genotyped) */
    const uint32_t* cand_snv;          /* sx_pileup_reads_batch.cand_snv, or NULL */
    uint32_t n_cand_snv;
    uint32_t max_read_len;             /* >= every read_len (0: 1024) */
    int32_t do_site_gl;                /* run K2a on the columns */
    int32_t is_always_test;            /* K2a's is_always_test (the germline caller genotypes every site: 1) */
    int32_t is_retain_optimal_soft_clipping; /* opt.isRetainOptimalSoftClipping (starling_read_align.cpp:1700-1737; the RNA workflow's
                                          --retain-optimal-soft-clipping): not accelerated -- nonzero is refused with SX_ERR_UNSUPPORTED, like the RNA
                                          het-extension model, rather than answered with the DNA behaviour */
    int32_t reserved_;
    sx_enum_opts enum_opts;
    sx_score_indels_opts score_opts;
    sx_pileup_opts pileup_opts;
} sx_window_batch;

#define SX_WIN_TOTALS 10 /* alignments, their segments, their keys, K1 segments, insert-pool bytes, best-alignment slots, tier1 calls, tier2 calls,
                            variant sites, (reserved) */

/* one call record of the window's site results: a position whose most likely genotype is not the reference's (what leaves the window for
 * the variant writers; the in-memory analogue of a variants.vcf line, gathered across GPUs by sx_gatherv_records) */
typedef struct sx_site_call {
    int32_t pos;
    uint32_t n_calls;        /* depth of the position's tier1 column */
    sx_digt_result gl;
} sx_site_call;

typedef struct sx_window_out { /* device pointers, each may be NULL (capacities count only for non-NULL arrays) */
    uint8_t* gate;               /* [n_reads] SX_GATE_* (sub-mapped reads: 0, align_pos :746) */
    uint8_t* enum_status;        /* [n_reads] SX_ENUM_ST_* */
    uint8_t* realign_status;     /* [n_reads] SX_REALIGN_ST_* */
    int32_t* best_pos;           /* [n_reads] getBestAlignment().pos */
    uint32_t* best_seg_off;      /* [n_reads + 1] */
    uint16_t* best_n_seg;        /* [n_reads] */
    sx_aln_seg* best_segs;       /* [cap_best_segs] K4's kinds */
    uint32_t cap_best_segs;
    sx_read_indel_score* recs;   /* [rec_off[n_reads]] */
    uint32_t* n_rec;             /* [n_reads] */
    sx_pileup_columns cols;      /* each array NULL or caller-allocated with the stated capacities */
    sx_digt_result* site_gl;     /* [report_end - report_begin] */
    uint32_t* totals;            /* [SX_WIN_TOTALS] */
    sx_site_call* variant_sites; /* [cap_variant_sites] the computed sites with genome.max_gt != ref_gt, ascending position (needs do_site_gl);
                                    more than the capacity: SX_ERR_CAPACITY, totals[8] says how many */
    uint32_t cap_variant_sites;
} sx_window_out;

enum { SX_WIN_ST_PREP = 0, SX_WIN_ST_GATES, SX_WIN_ST_KEYS, SX_WIN_ST_ENUMERATE, SX_WIN_ST_LINK, SX_WIN_ST_SCORE, SX_WIN_ST_SCORE_INDELS, SX_WIN_ST_CHOOSE,
       SX_WIN_ST_PILEUP, SX_WIN_ST_SITE_GL, SX_WIN_N_STAGES };

void sx_default_window_opts(sx_window_batch* b); /* fills enum_opts (max_alns_per_read = 5000), score_opts, pileup_opts, is_always_test = 1 */
/* SX_ERR_CAPACITY: a caller-provided output array is too small (totals_host, if given, says what the window produced). */
int sx_process_window_dev(sx_ctx* ctx, const sx_window_batch* batch_dev, sx_window_out* out_dev, uint32_t* totals_host /* [SX_WIN_TOTALS] or NULL */);
/* the same with HOST arrays in and out: every input array is copied to the device, the pass runs, and every non-NULL output array is copied
 * back (capacities as above; totals_host says how much of each was produced).  One sx_ctx per host thread: two threads with a context each
 * overlap one window's transfers with the other's kernels. */
int sx_process_window(sx_ctx* ctx, const sx_window_batch* batch_host, sx_window_out* out_host, uint32_t* totals_host);
/* device time of each stage of the most recent sx_process_window_dev on ctx (CUDA events on the compute stream), ms[SX_WIN_N_STAGES] */
int sx_last_window_timing(const sx_ctx* ctx, float* ms);

/* ==========================================================================================
 * Multi-GPU: regions shard across ranks with no data-path collective; one gather of fixed-size
 * call records at the end (the in-memory analogue of concatIndexVcf,
 * src/python/lib/strelkaSharedWorkflow.py:126-136).  The NCCL communicator is created from an
 * id the caller distributes out of band (torch.distributed / MPI / file).
 * ======================================================================================== */
#define SX_NCCL_ID_BYTES 128
int sx_comm_get_unique_id(void* id_out /*[SX_NCCL_ID_BYTES]*/);
int sx_comm_init(sx_ctx* ctx, const void* id, int rank, int world_size);
/* every rank contributes the SAME `bytes` from local_dev; rank `root` (0 <= root < world_size) receives world_size*bytes in all_dev
 * (non-NULL on the root; ncclGather semantics via grouped send/recv); blocks until complete.  Ranks whose blocks differ in size
 * (n % world_size != 0 under strelka_b200/shard.py's shard_range) use sx_gatherv_records. */
int sx_gather_records(sx_ctx* ctx, const void* local_dev, size_t bytes, void* all_dev, int root);
/* the same exchange enqueued on the context's communication stream behind the work already on its compute stream: returns at once, so
 * the next step's kernels overlap rank 0's receives; sx_comm_wait blocks until the last enqueued gather has completed. */
int sx_gather_records_async(sx_ctx* ctx, const void* local_dev, size_t bytes, void* all_dev, int root);
int sx_comm_wait(sx_ctx* ctx);
/* variable block sizes: the per-rank byte counts are exchanged first, rank p's block lands at offsets_out[p] (= the exclusive prefix
 * sum of the counts; offsets_out[world_size] = total; written on the root, may be NULL).  SX_ERR_CAPACITY on EVERY rank (no rank is
 * left waiting) when the total exceeds all_capacity.  Blocking. */
int sx_gatherv_records(sx_ctx* ctx, const void* local_dev, size_t bytes, void* all_dev, size_t all_capacity, uint64_t* offsets_out, int root);

/* ------------------------------------------------------------------------------------------
 * Instrumentation: device time (ms, CUDA events on the launching stream) and launch count of
 * the kernels run by the most recent entry-point call on ctx.
 * ---------------------------------------------------------------------------------------- */
typedef struct sx_timing {
    float kernel_ms;     /* sum over this call's kernels */
    float h2d_ms, d2h_ms;
    uint32_t launches;   /* kernels launched by this call */
    uint32_t pad;
} sx_timing;
int sx_last_timing(const sx_ctx* ctx, sx_timing* out);
uint64_t sx_total_launches(const sx_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* STRELKA_B200_H */
