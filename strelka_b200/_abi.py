"""ctypes view of include/strelka_b200.h (the C ABI) and the loader of libstrelka_b200.so.

The shared library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is no CPU
fallback: if the library is missing, ``load()`` raises, and without a CUDA device ``sx_create`` fails.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "csrc", "libstrelka_b200.so")

SX_OK = 0
SX_ERR_CUDA, SX_ERR_ARG, SX_ERR_ALIGNMENT, SX_ERR_UNSUPPORTED, SX_ERR_RANGE, SX_ERR_NOMEM, SX_ERR_NCCL = -1, -2, -3, -4, -5, -6, -7
SX_POOL_SLACK = 64
SX_SEG_MATCH, SX_SEG_INSERT, SX_SEG_REFSKIP, SX_SEG_SOFTCLIP, SX_SEG_HARDCLIP = 0, 1, 2, 3, 4
SX_SEGF_NONCANDIDATE = 1
SX_NCCL_ID_BYTES = 128


class SxParams(C.Structure):
    _fields_ = [
        ("bsnp_diploid_theta", C.c_double),
        ("bsnp_ssd_no_mismatch", C.c_double),
        ("bsnp_ssd_one_mismatch", C.c_double),
        ("is_min_vexp", C.c_int32),
        ("is_bsnp_diploid", C.c_int32),
        ("min_vexp", C.c_double),
        ("hetVariantFrequencyExtension", C.c_double),
        ("somatic_snv_rate", C.c_double),
        ("shared_site_error_rate", C.c_double),
        ("shared_site_error_strand_bias_fraction", C.c_double),
        ("ssnv_contam_tolerance", C.c_double),
        ("pipeline_chunks", C.c_int32),
        ("min_read_bp_flank", C.c_int32),
        ("randomBaseMatchProb", C.c_double),
        ("readConfidentSupportThreshold", C.c_double),
    ]


def default_params() -> SxParams:
    """Reference defaults: starling_options (starling_shared.hh:34-39) + configureStrelkaSomaticWorkflow.py.ini."""
    return SxParams(0.001, 0.35, 0.6, 1, 1, 0.25, 0.0, 1e-4, 5e-10, 0.0, 0.15, 0, 5, 0.25, 0.51)


# numpy mirrors of the POD arrays (layout == C structs; checked against sizeof in tests/test_abi.py)
ALN_SEG_DT = np.dtype([("len", "<u2"), ("kind", "u1"), ("flags", "u1")])
ALN_DT = np.dtype([("read", "<u4"), ("ref_pos", "<i4"), ("seg_off", "<u4"), ("ins_off", "<u4")])
ALN8_DT = np.dtype([("read", "<u2"), ("ref_pos", "<i2"), ("seg_off", "<u2"), ("ins_off", "<u2")])  # sx_aln8 (SX_FMT_ALN8)
SX_FMT_ALN8, SX_FMT_SEG2, SX_FMT_BASEQ, SX_FMT_REF4 = 1, 2, 4, 8
REGION_DT = np.dtype(
    [("seq_off", "<u8"), ("qual_off", "<u8"), ("ref_off", "<u8"), ("read_begin", "<u4"), ("aln_begin", "<u4"), ("seg_begin", "<u4"), ("ins_begin", "<u4"),
     ("ref_begin", "<i4"), ("ref_len", "<u4")]
)
GA_RESULT_DT = np.dtype([("score", "<i4"), ("beginPos", "<i4"), ("n_ops", "<u4"), ("status", "<u4")])
DIGT_RS_DT = np.dtype([("ref_pprob", "<f8"), ("max_gt", "<u4"), ("snp_qphred", "<i4"), ("max_gt_qphred", "<i4"), ("pad", "<i4")])
DIGT_RESULT_DT = np.dtype(
    [
        ("genome", DIGT_RS_DT),
        ("poly", DIGT_RS_DT),
        ("strand_bias", "<f8"),
        ("lhood", "<f4", (10,)),
        ("phredLoghood", "<u4", (10,)),
        ("ref_gt", "<u4"),
        ("is_computed", "<u4"),
        ("n_used_calls", "<u4"),
        ("pad", "<u4"),
    ]
)
SITE_CALL_DT = np.dtype([("pos", "<i4"), ("n_calls", "<u4"), ("gl", DIGT_RESULT_DT)])  # sx_site_call, 160 bytes
SSNV_RESULT_DT = np.dtype(
    [
        ("normal_lhood", "<f4", (30,)),
        ("tumor_lhood", "<f4", (30,)),
        ("strandBias", "<f4"),
        ("ref_gt", "<u4"),
        ("is_computed", "<u4"),
        ("snv_tier", "<u4"),
        ("snv_from_ntype_tier", "<u4"),
        ("ntype", "<u4"),
        ("max_gt", "<u4"),
        ("qphred", "<i4"),
        ("from_ntype_qphred", "<i4"),
        ("normal_alt_id", "<u4"),
        ("tumor_alt_id", "<u4"),
        ("nonsomatic_qphred", "<i4"),  # NQSS, callable mode only
    ]
)


INDEL_RESULT_DT = np.dtype([("gt_lhood", "<f8", (15,)), ("support", "<u2", (2, 6)), ("n_gt", "<u4"), ("pad", "<u4")])


class SxIndelBatch(C.Structure):
    _fields_ = [("n_loci", C.c_uint32)] + [(n, C.c_void_p) for n in (
        "read_off", "lnp_off", "allele_off", "ploidy", "allele_del_len", "allele_ins_len", "allele_lnp", "read_length", "non_ambig", "is_fwd")]


# K5b somatic_indel
SX_SINDEL_MAX_ALTS = 16
SX_SINDEL_ST_CAP = 0x100000
SINDEL_READ_DT = np.dtype([("ref", "<f4"), ("indel", "<f4"), ("alt_lnp", "<f4", (2,)), ("read_length", "<u2"), ("non_ambig", "<u2"),
                           ("is_tier1", "u1"), ("n_alt", "u1"), ("alt", "u1", (2,))])
SINDEL_TIER_DT = np.dtype([("normal_lhood", "<f4", (21,)), ("tumor_lhood", "<f4", (21,)), ("qphred", "<i4"), ("from_ntype_qphred", "<i4"),
                           ("ntype", "<u4"), ("max_gt", "<u4"), ("evaluated", "u1"), ("is_overlap", "u1"), ("multi_indel", "u1"), ("pad", "u1")])
SINDEL_RESULT_DT = np.dtype([("tier", SINDEL_TIER_DT, (2,)), ("status", "<u4"), ("is_output", "u1"), ("sindel_tier", "u1"), ("sindel_from_ntype_tier", "u1"),
                             ("is_overlap", "u1"), ("ntype", "<u4"), ("max_gt", "<u4"), ("qphred", "<i4"), ("from_ntype_qphred", "<i4")])


class SxSindelOpts(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("somatic_indel_rate", "bindel_diploid_theta", "indel_contam_tolerance", "shared_indel_error_factor",
                                          "randomBaseMatchProb", "tier2RandomBaseMatchProb")] + [
        ("useTier2Evidence", C.c_int32), ("min_read_bp_flank", C.c_int32 * 2), ("pad", C.c_int32)]


class SxSindelBatch(C.Structure):
    _fields_ = [("n_loci", C.c_uint32), ("pad", C.c_uint32)] + [(n, C.c_void_p) for n in (
        "key", "is_forced_output", "err_idx", "alt_off", "alts", "read_off", "reads")]


# K6b indel_reads
SX_INDEL_READS_ST_DUP_READ = 0x400000


class SxIndelReadsSample(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("n_regions", "n_reads", "n_keys", "pad")] + [(n, C.c_void_p) for n in (
        "region_read_off", "region_key_off", "key_gid", "rec_off", "recs", "n_rec", "read_len", "non_ambig", "read_flags", "read_id")]


class SxIndelLoci(C.Structure):
    _fields_ = [("n_loci", C.c_uint32), ("n_gid", C.c_uint32)] + [(n, C.c_void_p) for n in ("gid", "key", "is_forced_output", "err_idx", "gid_key")]


class SxIndelReadsOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("alt_off", "alts", "read_off", "reads", "status", "totals")] + [("cap_alts", C.c_uint32), ("cap_reads", C.c_uint32)]


# K6g allele_groups
SX_INDEL_MAX_ALLELES = 4


class SxAlleleGroups(C.Structure):
    _fields_ = [("n_groups", C.c_uint32), ("n_gid", C.c_uint32)] + [(n, C.c_void_p) for n in (
        "allele_off", "allele_gid", "contrast_off", "contrast_gid", "ploidy", "gid_key")]


class SxAlleleGroupReadsOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("read_off", "lnp_off", "allele_off", "ploidy", "allele_del_len", "allele_ins_len", "allele_lnp", "read_length", "non_ambig",
                                          "is_fwd", "status", "totals")] + [("cap_reads", C.c_uint32), ("cap_lnp", C.c_uint32)]


def default_sindel_opts() -> SxSindelOpts:
    o = SxSindelOpts()
    load().sx_default_sindel_opts(C.byref(o))
    return o


class SxAlignBatch(C.Structure):
    _fields_ = [
        ("n_regions", C.c_uint32),
        ("n_reads", C.c_uint32),
        ("n_alns", C.c_uint32),
        ("n_segs", C.c_uint32),
        ("regions", C.c_void_p),
        ("read_len", C.c_void_p),
        ("seq4", C.c_void_p),
        ("qual", C.c_void_p),
        ("ref", C.c_void_p),
        ("alns", C.c_void_p),
        ("segs", C.c_void_p),
        ("ins", C.c_void_p),
        ("seq4_bytes", C.c_uint64),
        ("qual_bytes", C.c_uint64),
        ("ref_bytes", C.c_uint64),
        ("ins_bytes", C.c_uint64),
        ("qual_bits", C.c_uint32),
        ("qual_dict", C.c_uint8 * 16),
        ("format", C.c_uint32),
        ("exc_off", C.c_void_p),
        ("exc", C.c_void_p),
    ]


# K4 pileup_reads
SX_SEG_DELETE, SX_SEG_SKIP = 5, 6
SX_PRF_FWD, SX_PRF_TIER1, SX_PRF_TIER1OR2, SX_PRF_PIN_FIRST, SX_PRF_PIN_SECOND, SX_PRF_SKIP = 1, 2, 4, 8, 16, 32
PILEUP_READ_DT = np.dtype([("seq_off", "<u4"), ("qual_off", "<u4"), ("seg_off", "<u4"), ("pos", "<i4"), ("len", "<u2"), ("mapq", "u1"), ("flags", "u1")])


class SxPileupOpts(C.Structure):
    _fields_ = [
        ("isBasecallQualAdjustedForMapq", C.c_int32),
        ("minBasecallErrorPhredProb", C.c_int32),
        ("mismatchDensityFilterFlankSize", C.c_uint32),
        ("mismatchDensityFilterMaxMismatchCount", C.c_uint32),
        ("useTier2Evidence", C.c_int32),
        ("tier2MismatchDensityFilterMaxMismatchCount", C.c_int32),
        ("minDistanceFromReadEdge", C.c_uint32),
        ("reserved_", C.c_uint32),
    ]


class SxPileupReadsBatch(C.Structure):
    _fields_ = [
        ("n_reads", C.c_uint32),
        ("n_segs", C.c_uint32),
        ("reads", C.c_void_p),
        ("seq4", C.c_void_p),
        ("qual", C.c_void_p),
        ("segs", C.c_void_p),
        ("ref", C.c_void_p),
        ("ref_begin", C.c_int32),
        ("ref_len", C.c_uint32),
        ("report_begin", C.c_int32),
        ("report_end", C.c_int32),
        ("cand_snv", C.c_void_p),
        ("n_cand_snv", C.c_uint32),
        ("max_ref_span", C.c_uint32),
        ("max_read_len", C.c_uint32),
        ("reserved_", C.c_uint32),
        ("opts", SxPileupOpts),
        ("buffer_pos", C.c_void_p),
        ("max_pos_shift", C.c_uint32),
        ("qual_bits", C.c_uint32),
        ("qual_dict", C.c_uint8 * 16),
    ]


class SxPileupColumns(C.Structure):
    _fields_ = [
        ("site_off", C.c_void_p),
        ("calls", C.c_void_p),
        ("t2_off", C.c_void_p),
        ("t2_calls", C.c_void_p),
        ("n_spandel", C.c_void_p),
        ("n_submapped", C.c_void_p),
        ("calls_capacity", C.c_uint64),
        ("t2_capacity", C.c_uint64),
    ]


def default_pileup_opts() -> SxPileupOpts:
    """blt_options / starling_base_options defaults + the germline workflow's mismatch density filter (flank 20, max 2)."""
    return SxPileupOpts(1, 17, 20, 2, 0, 10, 0, 0)


# K4m pileup_metrics
SX_PM_MAPQ, SX_PM_GERMLINE, SX_PM_SOMATIC = 1, 2, 3
SX_PM_ST_MQ_OVERFLOW, SX_PM_ST_BASEQ_OVERFLOW, SX_PM_ST_READ_POS_OVERFLOW = 1, 2, 4
PILEUP_METRICS_DT = np.dtype([("mapq_sum_sq", "<f8"), ("read_pos_ranksum", "<f8"), ("mq_ranksum", "<f8"), ("baseq_ranksum", "<f8"), ("raw_pos", "<f8"),
                              ("raw_baseq", "<f8"), ("mean_edge_distance", "<f8"), ("mapq_count", "<u4"), ("mapq_zero", "<u4"), ("n_alt_read_pos", "<u4"),
                              ("median_read_pos", "<u2"), ("median_read_pos_var", "<u2"), ("status", "<u4"), ("pad", "<u4")])  # sx_pileup_metrics_rec
assert PILEUP_METRICS_DT.itemsize == 80


class SxPileupMetricsOpts(C.Structure):
    _fields_ = [("mode", C.c_uint32), ("reserved_", C.c_uint32), ("full_len", C.c_void_p), ("full_off", C.c_void_p)]


# K6 score_indels
SX_INDEL_TYPE_INDEL, SX_INDEL_TYPE_MISMATCH = 0, 1
SX_IKF_CANDIDATE = 1
SX_SIF_FWD, SX_SIF_TIER1, SX_SIF_INCOMPLETE = 1, 2, 4
SX_RIS_SCORED, SX_RIS_SUBOVERLAP = 1, 2
INDEL_KEY_DT = np.dtype([("pos", "<i4"), ("del_len", "<u2"), ("ins_len", "<u2"), ("ins_id", "<u4"), ("type", "u1"), ("flags", "u1"), ("pad", "<u2"),
                         ("ref_to_indel_lnp", "<f8"), ("indel_to_ref_lnp", "<f8")])
READ_INDEL_SCORE_DT = np.dtype([("key", "<u2"), ("flags", "u1"), ("n_alt", "u1"), ("read_pos", "<i2"), ("dist_from_edge", "<i2"), ("ref_lnp", "<f4"),
                                ("indel_lnp", "<f4"), ("alt_key", "<u2", (2,)), ("alt_lnp", "<f4", (2,)), ("pad", "<u4")])
assert INDEL_KEY_DT.itemsize == 32 and READ_INDEL_SCORE_DT.itemsize == 32


class SxScoreIndelsOpts(C.Structure):
    _fields_ = [("max_indel_size", C.c_uint32), ("upstream_oligo_size", C.c_uint32), ("min_read_bp_flank", C.c_int32), ("is_smoothed_alignments", C.c_int32),
                ("smoothed_lnp_range", C.c_double)]


class SxScoreIndelsBatch(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("n_regions", "n_reads", "n_alns", "n_keys")] + [(n, C.c_void_p) for n in (
        "region_read_off", "region_key_off", "keys", "aln_off", "aln_pos", "aln_seg_off", "segs", "aln_key_off", "aln_keys", "read_len", "non_ambig",
        "full_len", "full_off", "read_flags", "rec_off")] + [("opts", SxScoreIndelsOpts)]


class SxScoreIndelsOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("recs", "n_rec", "max_aln", "eval_aln")]


def default_score_indels_opts() -> SxScoreIndelsOpts:
    """starling_base_options defaults (starling_base_shared.hh:108,124,170-171,206)."""
    import math

    return SxScoreIndelsOpts(49, 0, 5, 1, math.log(10.0))


# K7 enumerate_alignments
SX_AP_MATCH, SX_AP_INSERT, SX_AP_DELETE, SX_AP_SKIP, SX_AP_SOFT_CLIP, SX_AP_HARD_CLIP, SX_AP_PAD, SX_AP_SEQ_MATCH, SX_AP_SEQ_MISMATCH = 1, 2, 3, 4, 5, 6, 7, 8, 9
SX_IKF_NOT_DISCOVERED, SX_IKF_FORCED_OUTPUT = 2, 4
SX_ENUM_MAX_SAMPLES = 4
SX_NO_KEY = 0xFFFF
SX_ENUM_ST_ORIGIN_SKIP, SX_ENUM_ST_MAX_TOGGLE, SX_ENUM_ST_EXCEPTION, SX_ENUM_ST_LIMIT = 1, 2, 4, 8
SX_ERR_CAPACITY = -8
SX_ENUM_F_FAST = 1
KEY_HAP_DT = np.dtype([("active_region_id", "<i4"), ("haplotype_id", "i1", (4,)), ("bypass_mask", "u1"), ("pad", "u1", (3,))])
assert KEY_HAP_DT.itemsize == 12


class SxEnumOpts(C.Structure):
    _fields_ = [("max_indel_size", C.c_uint32), ("max_read_indel_toggle", C.c_int32), ("max_candidate_indel_density", C.c_double), ("n_max_toggle", C.c_uint32),
                ("max_toggle", C.c_uint8 * 100), ("is_haplotyping_enabled", C.c_int32), ("n_samples", C.c_uint32), ("sample_id", C.c_uint32),
                ("max_alns_per_read", C.c_uint32), ("flags", C.c_uint32)]


class SxEnumBatch(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("n_regions", "n_reads", "n_keys")] + [(n, C.c_void_p) for n in (
        "region_read_off", "region_key_off", "keys", "key_hap", "realign_begin", "realign_end", "in_pos", "in_seg_off", "in_segs", "in_key_off", "in_keys",
        "use_key_off", "use_keys", "in_lead_key", "in_trail_key", "read_len", "gate")] + [("opts", SxEnumOpts)]


class SxEnumOut(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("cap_alns", "cap_segs", "cap_keys")] + [(n, C.c_void_p) for n in (
        "totals", "aln_off", "status", "aln_pos", "aln_seg_off", "segs", "aln_key_off", "aln_keys", "aln_lead_key", "aln_trail_key")]


class SxLinkOut(C.Structure):
    _fields_ = [("cap_segs", C.c_uint32), ("cap_ins", C.c_uint32)] + [(n, C.c_void_p) for n in ("totals", "regions", "alns", "segs", "ins", "k6_segs")]


class SxPrepOut(C.Structure):
    _fields_ = [("cap_keys", C.c_uint32)] + [(n, C.c_void_p) for n in ("totals", "in_key_off", "in_keys", "in_lead_key", "in_trail_key")]


SX_REALIGN_ST_REALIGNED, SX_REALIGN_ST_UNSUPPORTED, SX_REALIGN_ST_LIMIT, SX_REALIGN_ST_BADPATH = 1, 2, 4, 8


class SxRealignBatch(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("n_regions", "n_reads", "n_alns")] + [(n, C.c_void_p) for n in (
        "region_read_off", "region_key_off", "keys", "aln_off", "aln_pos", "aln_seg_off", "segs", "aln_key_off", "aln_keys", "read_len", "pin_flags")] + [
        ("is_smoothed_alignments", C.c_int32), ("k4_kinds", C.c_int32), ("smoothed_lnp_range", C.c_double),
        ("raw_pos", C.c_void_p), ("raw_seg_off", C.c_void_p), ("raw_segs", C.c_void_p)]


class SxRealignOut(C.Structure):
    _fields_ = [("cap_segs", C.c_uint32)] + [(n, C.c_void_p) for n in ("totals", "seg_off", "pos", "n_seg", "status", "best_aln", "segs")]


SX_GATE_REALIGN, SX_GATE_SOFT_CLIPPED = 1, 2


class SxGateBatch(C.Structure):
    _fields_ = [("n_regions", C.c_uint32), ("n_reads", C.c_uint32)] + [(n, C.c_void_p) for n in (
        "region_read_off", "region_key_off", "keys", "realign_begin", "realign_end", "raw_pos", "seg_off", "raw_segs", "read_len", "pin_flags")] + [
        ("max_indel_size", C.c_uint32)]


class SxWindowBatch(C.Structure):
    _fields_ = ([(n, C.c_uint32) for n in ("n_regions", "n_reads", "n_keys")] + [(n, C.c_void_p) for n in (
        "region_read_off", "region_key_off", "keys", "key_hap", "key_ins_off", "key_ins", "realign_begin", "realign_end", "raw_pos", "raw_seg_off", "raw_segs", "read_len",
        "read_flags", "mapq", "use_key_off", "use_keys", "rec_off", "regions", "seq4", "qual", "ref")] + [
        ("seq4_bytes", C.c_uint64), ("qual_bytes", C.c_uint64), ("ref_bytes", C.c_uint64), ("qual_bits", C.c_uint32), ("qual_dict", C.c_uint8 * 16),
        ("ref_begin", C.c_int32), ("report_begin", C.c_int32), ("report_end", C.c_int32), ("cand_snv", C.c_void_p), ("n_cand_snv", C.c_uint32), ("max_read_len", C.c_uint32),
        ("do_site_gl", C.c_int32), ("is_always_test", C.c_int32), ("is_retain_optimal_soft_clipping", C.c_int32), ("reserved_", C.c_int32), ("enum_opts", SxEnumOpts), ("score_opts", SxScoreIndelsOpts), ("pileup_opts", SxPileupOpts)])


class SxWindowOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("gate", "enum_status", "realign_status", "best_pos", "best_seg_off", "best_n_seg", "best_segs")] + [("cap_best_segs", C.c_uint32)] + [
        (n, C.c_void_p) for n in ("recs", "n_rec")] + [("cols", SxPileupColumns), ("site_gl", C.c_void_p), ("totals", C.c_void_p), ("variant_sites", C.c_void_p),
                                                       ("cap_variant_sites", C.c_uint32)]


SX_WIN_TOTALS, SX_WIN_N_STAGES = 10, 10
SX_WIN_STAGE_NAMES = ("prep", "k7g_gates", "k7a_keys", "k7_enumerate", "k7b_link", "k1_score", "k6_score_indels", "k9_choose", "k4_pileup", "k2a_site_gl")


# somatic window pass
SOMATIC_SITE_CALL_DT = np.dtype([("pos", "<i4"), ("n_calls", "<u4", (2,)), ("pad", "<u4"), ("r", SSNV_RESULT_DT)])  # sx_somatic_site_call, 304 bytes
SOMATIC_INDEL_CALL_DT = np.dtype([("locus", "<u4"), ("pad", "<u4"), ("r", SINDEL_RESULT_DT)])  # sx_somatic_indel_call, 408 bytes


class SxSomaticWindowBatch(C.Structure):
    _fields_ = [("sample", SxWindowBatch * 2), ("key_gid", C.c_void_p * 2), ("read_id", C.c_void_p * 2), ("snv_forced_output", C.c_void_p), ("loci", SxIndelLoci),
                ("sindel_opts", SxSindelOpts), ("err_prob", C.c_void_p), ("n_err", C.c_uint32), ("is_compute_nonsomatic", C.c_uint32)]


class SxSomaticWindowOut(C.Structure):
    _fields_ = [("sample", SxWindowOut * 2)] + [(n, C.c_void_p) for n in ("site_snv", "snv_calls", "indel", "indel_calls", "totals")] + [
        ("cap_snv_calls", C.c_uint32), ("cap_indel_calls", C.c_uint32)]


SX_SWIN_TOTALS, SX_SWIN_N_STAGES = 4, 7
SX_SWIN_STAGE_NAMES = ("normal", "tumor", "k2b_site_snv", "snv_calls", "k6b_link", "k5b_indel", "indel_calls")
SX_WIN_ST_METRICS, SX_SWIN_ST_METRICS = SX_WIN_N_STAGES, SX_SWIN_N_STAGES


class SxGateOut(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("gate", "in_pos", "in_segs")]


def default_enum_opts() -> SxEnumOpts:
    """starling_base_options defaults (starling_base_shared.hh:124,139,145,160) through the library's own sx_default_enum_opts."""
    o = SxEnumOpts()
    load().sx_default_enum_opts(C.byref(o))
    return o


class SxGaScores(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("match", "mismatch", "open", "extend", "offEdge", "insertDelete", "isAllowEdgeInsertion", "isRequireEdgeDeletion")]


class SxGaBatch(C.Structure):
    _fields_ = [
        ("n", C.c_uint32),
        ("query", C.c_void_p),
        ("ref", C.c_void_p),
        ("query_off", C.c_void_p),
        ("ref_off", C.c_void_p),
        ("max_ops", C.c_uint32),
    ]


class SxPileupBatch(C.Structure):
    _fields_ = [
        ("n_sites", C.c_uint32),
        ("site_off", C.c_void_p),
        ("calls", C.c_void_p),
        ("t2_off", C.c_void_p),
        ("t2_calls", C.c_void_p),
        ("ref_base", C.c_void_p),
        ("ploidy", C.c_void_p),
    ]


# K2c site_continuous
SX_CONT_MAX_SAMPLES = 8
SX_CONT_REF_LOCUS = 4
SX_CONT_GT_HOMREF, SX_CONT_GT_HET, SX_CONT_GT_HOM = 0, 1, 2
SX_CONT_ST_QSCORE_TIE = 0x2000000
CONT_LOCUS_DT = np.dtype([("strand_bias", "<f8"), ("pos", "<i4"), ("qual", "<i4"), ("sb_fwd_alt", "<u4"), ("sb_rev_alt", "<u4"), ("sb_fwd_other", "<u4"),
                          ("sb_rev_other", "<u4"), ("alt", "u1"), ("ref", "u1"), ("forced", "u1"), ("pad", "u1", (5,))])
CONT_SAMPLE_DT = np.dtype([("af", "<f8"), ("strand_bias", "<f8")] + [(n, "<u4") for n in (
    "ref_fwd", "ref_rev", "alt_fwd", "alt_rev", "non_confident_fwd", "non_confident_rev", "total_depth", "allele_depth", "used", "unused")] + [
    ("gq", "<i4"), ("status", "<u4"), ("gt", "u1"), ("pad", "u1", (7,))])


class SxContOpts(C.Structure):
    _fields_ = [("min_het_vf", C.c_double), ("max_abs_sample_strand_bias", C.c_double), ("expected_qscore", C.c_int32), ("max_qscore", C.c_int32)]


class SxContBatch(C.Structure):
    _fields_ = [("n_sites", C.c_uint32), ("n_samples", C.c_uint32), ("pos_begin", C.c_int32), ("pad", C.c_uint32), ("forced_output", C.c_void_p),
                ("sample", SxPileupBatch * SX_CONT_MAX_SAMPLES)]


class SxContOut(C.Structure):
    _fields_ = [("loci", C.c_void_p), ("samples", C.c_void_p), ("site_rec_off", C.c_void_p), ("cap_loci", C.c_uint32), ("pad", C.c_uint32)]


class SxTiming(C.Structure):
    _fields_ = [("kernel_ms", C.c_float), ("h2d_ms", C.c_float), ("d2h_ms", C.c_float), ("launches", C.c_uint32), ("pad", C.c_uint32)]


# every symbol include/strelka_b200.h declares: (name, restype, argtypes)
_P = C.c_void_p
SYMBOLS = [
    ("sx_default_params", None, [C.POINTER(SxParams)]),
    ("sx_create", C.c_int, [C.c_int, C.POINTER(SxParams), C.POINTER(_P)]),
    ("sx_destroy", None, [_P]),
    ("sx_set_host_wait_policy", C.c_int, [C.c_int, C.c_int]),
    ("sx_last_error", C.c_char_p, [_P]),
    ("sx_abi_version", C.c_int, []),
    ("sx_host_alloc", _P, [C.c_size_t]),
    ("sx_host_free", None, [_P]),
    ("sx_dev_alloc", _P, [_P, C.c_size_t]),
    ("sx_dev_free", None, [_P, _P]),
    ("sx_memcpy_h2d", C.c_int, [_P, _P, _P, C.c_size_t]),
    ("sx_memcpy_d2h", C.c_int, [_P, _P, _P, C.c_size_t]),
    ("sx_memcpy_d2d", C.c_int, [_P, _P, _P, C.c_size_t]),
    ("sx_timer_mark", C.c_int, [_P, C.c_int]),
    ("sx_stream_join", C.c_int, [_P, _P]),
    ("sx_timer_elapsed_ms", C.c_int, [_P, C.POINTER(C.c_double)]),
    ("sx_synchronize", C.c_int, [_P]),
    ("sx_score_alignments", C.c_int, [_P, C.POINTER(SxAlignBatch), _P]),
    ("sx_score_alignments_dev", C.c_int, [_P, C.POINTER(SxAlignBatch), _P]),
    ("sx_align_batch_cells", C.c_uint64, [C.POINTER(SxAlignBatch)]),
    ("sx_read_max_dev", C.c_int, [_P, C.POINTER(SxAlignBatch), _P, _P, _P]),
    ("sx_ga_active_region_scores", None, [C.POINTER(SxGaScores)]),
    ("sx_global_align", C.c_int, [_P, C.POINTER(SxGaScores), C.POINTER(SxGaBatch), _P, _P]),
    ("sx_global_align_dev", C.c_int, [_P, C.POINTER(SxGaScores), C.POINTER(SxGaBatch), _P, _P]),
    ("sx_site_gl_germline", C.c_int, [_P, C.POINTER(SxPileupBatch), C.c_int, _P]),
    ("sx_site_gl_germline_dev", C.c_int, [_P, C.POINTER(SxPileupBatch), C.c_int, _P]),
    ("sx_dependent_eprob", C.c_int, [_P, C.POINTER(SxPileupBatch), _P, _P]),
    ("sx_site_gl_somatic", C.c_int, [_P, C.POINTER(SxPileupBatch), C.POINTER(SxPileupBatch), _P, _P]),
    ("sx_site_gl_somatic_dev", C.c_int, [_P, C.POINTER(SxPileupBatch), C.POINTER(SxPileupBatch), _P, _P]),
    ("sx_site_gl_somatic_callable", C.c_int, [_P, C.POINTER(SxPileupBatch), C.POINTER(SxPileupBatch), _P, _P]),
    ("sx_site_gl_somatic_callable_dev", C.c_int, [_P, C.POINTER(SxPileupBatch), C.POINTER(SxPileupBatch), _P, _P]),
    ("sx_somatic_callable_regions_dev", C.c_int, [_P, _P, C.c_uint32, C.c_int32, _P, _P, C.c_uint32, C.POINTER(C.c_uint32)]),
    ("sx_default_score_indels_opts", None, [C.POINTER(SxScoreIndelsOpts)]),
    ("sx_score_indels", C.c_int, [_P, C.POINTER(SxScoreIndelsBatch), _P, C.POINTER(SxScoreIndelsOut)]),
    ("sx_score_indels_dev", C.c_int, [_P, C.POINTER(SxScoreIndelsBatch), _P, C.POINTER(SxScoreIndelsOut)]),
    ("sx_default_enum_opts", None, [C.POINTER(SxEnumOpts)]),
    ("sx_enumerate_alignments", C.c_int, [_P, C.POINTER(SxEnumBatch), C.POINTER(SxEnumOut)]),
    ("sx_enumerate_alignments_dev", C.c_int, [_P, C.POINTER(SxEnumBatch), C.POINTER(SxEnumOut)]),
    ("sx_alignment_indels", C.c_int, [_P, C.POINTER(SxEnumBatch), _P, _P, _P, _P, _P, C.POINTER(SxPrepOut)]),
    ("sx_alignment_indels_dev", C.c_int, [_P, C.POINTER(SxEnumBatch), _P, _P, _P, _P, _P, C.POINTER(SxPrepOut)]),
    ("sx_choose_realignment", C.c_int, [_P, C.POINTER(SxRealignBatch), _P, C.POINTER(SxRealignOut)]),
    ("sx_choose_realignment_dev", C.c_int, [_P, C.POINTER(SxRealignBatch), _P, C.POINTER(SxRealignOut)]),
    ("sx_realign_gates", C.c_int, [_P, C.POINTER(SxGateBatch), C.POINTER(SxGateOut)]),
    ("sx_realign_gates_dev", C.c_int, [_P, C.POINTER(SxGateBatch), C.POINTER(SxGateOut)]),
    ("sx_link_alignments", C.c_int, [_P, C.POINTER(SxEnumBatch), C.POINTER(SxEnumOut), C.c_uint32, _P, _P, C.POINTER(SxLinkOut)]),
    ("sx_link_alignments_dev", C.c_int, [_P, C.POINTER(SxEnumBatch), C.POINTER(SxEnumOut), C.c_uint32, _P, _P, C.POINTER(SxLinkOut)]),
    ("sx_indel_gl", C.c_int, [_P, C.POINTER(SxIndelBatch), _P]),
    ("sx_indel_gl_dev", C.c_int, [_P, C.POINTER(SxIndelBatch), _P]),
    ("sx_default_sindel_opts", None, [C.POINTER(SxSindelOpts)]),
    ("sx_somatic_indel", C.c_int, [_P, C.POINTER(SxSindelOpts), C.POINTER(SxSindelBatch), _P, C.c_uint32, _P]),
    ("sx_somatic_indel_dev", C.c_int, [_P, C.POINTER(SxSindelOpts), C.POINTER(SxSindelBatch), _P, C.c_uint32, _P]),
    ("sx_link_indel_reads", C.c_int, [_P, C.POINTER(SxIndelReadsSample), C.POINTER(SxIndelReadsSample), C.POINTER(SxIndelLoci), C.POINTER(SxIndelReadsOut), _P]),
    ("sx_link_indel_reads_dev", C.c_int, [_P, C.POINTER(SxIndelReadsSample), C.POINTER(SxIndelReadsSample), C.POINTER(SxIndelLoci), C.POINTER(SxIndelReadsOut), _P]),
    ("sx_somatic_indel_from_records_dev", C.c_int, [_P, C.POINTER(SxSindelOpts), C.POINTER(SxIndelReadsSample), C.POINTER(SxIndelReadsSample), C.POINTER(SxIndelLoci),
                                                    _P, C.c_uint32, _P]),
    ("sx_link_allele_groups", C.c_int, [_P, C.POINTER(SxIndelReadsSample), C.POINTER(SxAlleleGroups), C.POINTER(SxAlleleGroupReadsOut), _P]),
    ("sx_link_allele_groups_dev", C.c_int, [_P, C.POINTER(SxIndelReadsSample), C.POINTER(SxAlleleGroups), C.POINTER(SxAlleleGroupReadsOut), _P]),
    ("sx_indel_gl_from_records_dev", C.c_int, [_P, C.POINTER(SxIndelReadsSample), C.POINTER(SxAlleleGroups), _P, _P]),
    ("sx_default_pileup_opts", None, [C.POINTER(SxPileupOpts)]),
    ("sx_pileup_reads", C.c_int, [_P, C.POINTER(SxPileupReadsBatch), C.POINTER(SxPileupColumns)]),
    ("sx_pileup_reads_dev", C.c_int, [_P, C.POINTER(SxPileupReadsBatch), C.POINTER(SxPileupColumns)]),
    ("sx_pileup_metrics", C.c_int, [_P, C.POINTER(SxPileupReadsBatch), C.POINTER(SxPileupMetricsOpts), _P]),
    ("sx_pileup_metrics_dev", C.c_int, [_P, C.POINTER(SxPileupReadsBatch), C.POINTER(SxPileupMetricsOpts), _P]),
    ("sx_default_window_opts", None, [C.POINTER(SxWindowBatch)]),
    ("sx_process_window_dev", C.c_int, [_P, C.POINTER(SxWindowBatch), C.POINTER(SxWindowOut), _P]),
    ("sx_process_window", C.c_int, [_P, C.POINTER(SxWindowBatch), C.POINTER(SxWindowOut), _P]),
    ("sx_last_window_timing", C.c_int, [_P, _P]),
    ("sx_process_somatic_window_dev", C.c_int, [_P, C.POINTER(SxSomaticWindowBatch), C.POINTER(SxSomaticWindowOut), _P]),
    ("sx_last_somatic_window_timing", C.c_int, [_P, _P]),
    ("sx_process_window_metrics_dev", C.c_int, [_P, C.POINTER(SxWindowBatch), C.POINTER(SxWindowOut), _P, C.POINTER(SxPileupMetricsOpts), _P]),
    ("sx_last_window_metrics_timing", C.c_int, [_P, _P]),
    ("sx_process_somatic_window_metrics_dev", C.c_int, [_P, C.POINTER(SxSomaticWindowBatch), C.POINTER(SxSomaticWindowOut), _P, C.POINTER(C.c_void_p * 2),
                                                        C.POINTER(C.c_void_p * 2)]),
    ("sx_last_somatic_window_metrics_timing", C.c_int, [_P, _P]),
    ("sx_default_cont_opts", None, [C.POINTER(SxContOpts)]),
    ("sx_site_continuous", C.c_int, [_P, C.POINTER(SxContOpts), C.POINTER(SxContBatch), C.POINTER(SxContOut), _P]),
    ("sx_site_continuous_dev", C.c_int, [_P, C.POINTER(SxContOpts), C.POINTER(SxContBatch), C.POINTER(SxContOut), _P]),
    ("sx_cont_qscore", C.c_int, [_P, C.POINTER(SxContOpts), C.c_uint32, _P, _P, _P, _P]),
    ("sx_cont_qscore_dev", C.c_int, [_P, C.POINTER(SxContOpts), C.c_uint32, _P, _P, _P, _P]),
    ("sx_comm_get_unique_id", C.c_int, [_P]),
    ("sx_comm_init", C.c_int, [_P, _P, C.c_int, C.c_int]),
    ("sx_gather_records", C.c_int, [_P, _P, C.c_size_t, _P, C.c_int]),
    ("sx_gather_records_async", C.c_int, [_P, _P, C.c_size_t, _P, C.c_int]),
    ("sx_comm_wait", C.c_int, [_P]),
    ("sx_gatherv_records", C.c_int, [_P, _P, C.c_size_t, _P, C.c_size_t, _P, C.c_int]),
    ("sx_last_timing", C.c_int, [_P, C.POINTER(SxTiming)]),
    ("sx_total_launches", C.c_uint64, [_P]),
]

_lib = None


def load(path: str | None = None) -> C.CDLL:
    """Load libstrelka_b200.so and bind every declared symbol.  Raises if the library is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise RuntimeError(
            f"{p} not found: the CUDA extension has not been built (run `python -c 'import __graft_entry__ as g; g.build()'`). "
            "strelka_b200 has no CPU fallback."
        )
    lib = C.CDLL(p, mode=C.RTLD_GLOBAL)
    for name, restype, argtypes in SYMBOLS:
        fn = getattr(lib, name)  # AttributeError here == ABI symbol missing
        fn.restype = restype
        fn.argtypes = argtypes
    if path is None:
        _lib = lib
    return lib


def ptr(a: np.ndarray | None) -> int | None:
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data
