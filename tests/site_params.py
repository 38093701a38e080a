"""The parameter points at which the somatic SNV model (K2b) and the indel genotype model (K5) are compared with the reference and the
oracle, shared by the CPU tests (tests/test_site_model_params.py), the frozen reference answers (tests/golden/make_site_params_golden.py)
and the GPU tests (tests/test_gpu_site_model_params.py).  Each point is A.default_params() with the named fields changed.

Every value is one the reference accepts: strelka_option_parser.cpp:161-163 checks somatic_snv_rate, shared_site_error_rate and
shared_site_error_strand_bias_fraction against [0, 1]; ssnv_contam_tolerance is documented as [0, 1] and not checked;
min_read_bp_flank, randomBaseMatchProb and readConfidentSupportThreshold have no command-line check (Tier2Options.hh:30 asserts
randomBaseMatchProb in [0, 1] for the tier2 copy).  No value listed here was left out.

shared_site_error_strand_bias_fraction = 1 does not zero the non-strand error rate by itself: the strand rate is rounded to float before
it is subtracted from the double rate (position_somatic_snv_strand_grid.cpp:49-50), so the difference is the rounding error of the
rate.  At the default rate 5e-10 that is +1.4e-17 (ln = -38.8); at 1e-3 it is -4.7e-11, whose log is NaN; at a rate that is exact in
float (2^-30) it is 0 and the log is -inf.  The three ssebf=1 points cover all three."""
from __future__ import annotations

import hashlib
import os

import numpy as np

import reflib
import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

K2B_POINTS = {
    "default": {},
    "ssebf_0.5": dict(shared_site_error_strand_bias_fraction=0.5),
    "ssebf_1": dict(shared_site_error_strand_bias_fraction=1.0),
    "ssebf_1_exact_rate": dict(shared_site_error_strand_bias_fraction=1.0, shared_site_error_rate=2.0**-30),  # ln(0) = -inf
    "contam_0": dict(ssnv_contam_tolerance=0.0),
    "contam_1": dict(ssnv_contam_tolerance=1.0),
    "snv_rate_1e-6": dict(somatic_snv_rate=1e-6),
    "snv_rate_0.1": dict(somatic_snv_rate=0.1),
    "sse_rate_1e-3": dict(shared_site_error_rate=1e-3),
    "theta_1e-2": dict(bsnp_diploid_theta=1e-2),
    # all of the above at once; the non-strand rate is 1e-3 - float(1e-3) < 0, so ln of it is NaN
    "all": dict(shared_site_error_strand_bias_fraction=1.0, ssnv_contam_tolerance=1.0, somatic_snv_rate=0.1, shared_site_error_rate=1e-3,
                bsnp_diploid_theta=1e-2),
    "all_ssebf_0.5": dict(shared_site_error_strand_bias_fraction=0.5, ssnv_contam_tolerance=1.0, somatic_snv_rate=0.1, shared_site_error_rate=1e-3,
                          bsnp_diploid_theta=1e-2),
}

K5_POINTS = {
    "default": {},
    "flank_0": dict(min_read_bp_flank=0),
    "flank_1": dict(min_read_bp_flank=1),
    "flank_40": dict(min_read_bp_flank=40),  # past half of the short reads' length: base_expect clamps to 0
    "rbm_0.1": dict(randomBaseMatchProb=0.1),
    "rbm_0.5": dict(randomBaseMatchProb=0.5),
    "support_0.5": dict(readConfidentSupportThreshold=0.5),
    "support_0.9": dict(readConfidentSupportThreshold=0.9),
    "all": dict(min_read_bp_flank=40, randomBaseMatchProb=0.5, readConfidentSupportThreshold=0.5),
}

# the point of the large K2b batch, and those of the somatic window pass on a non-default context
K2B_LARGE_POINT = "all_ssebf_0.5"
WINDOW_POINTS = ("ssebf_0.5", "snv_rate_0.1")


def params(overrides: dict) -> A.SxParams:
    p = A.default_params()
    for k, v in overrides.items():
        assert any(k == f[0] for f in A.SxParams._fields_), k
        setattr(p, k, v)
    return p


def k2b(name: str) -> A.SxParams:
    return params(K2B_POINTS[name])


def k5(name: str) -> A.SxParams:
    return params(K5_POINTS[name])


# ---------------------------------------------------------------------------------------------------------------------------------
# the edge batches (tests/specgen.py) every point runs on, and the frozen reference answers of tests/golden/site_params_ref.npz
# ---------------------------------------------------------------------------------------------------------------------------------
K2B_EDGE_SEED, K5_EDGE_SEED = 8100, 8200
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "site_params_ref.npz")
# the fields the reference harness returns (oracle/ref_harness.cpp ref_site_gl_somatic); strandBias is frozen and compared by its bits
K2B_REF_FIELDS = ("ref_gt", "is_computed", "snv_tier", "snv_from_ntype_tier", "ntype", "max_gt", "qphred", "from_ntype_qphred", "normal_alt_id", "tumor_alt_id",
                  "strandBias")

_batches = {}


def k2b_edge_batch():
    """(normal, tumor, forced, kind) of specgen.somatic_edge_sites, tier2 calls on both samples"""
    if "k2b" not in _batches:
        _batches["k2b"] = specgen.somatic_edge_sites(np.random.default_rng(K2B_EDGE_SEED))
    return _batches["k2b"]


def k5_edge_batch() -> B.IndelBatch:
    if "k5" not in _batches:
        _batches["k5"] = B.IndelBatch(specgen.indel_edge_loci(np.random.default_rng(K5_EDGE_SEED)))
    return _batches["k5"]


def inputs_digest() -> str:
    npb, tpb, forced, kind = k2b_edge_batch()
    ib = k5_edge_batch()
    h = hashlib.sha256()
    for a in (npb.site_off, npb.calls, npb.t2_off, npb.t2_calls, npb.ref_base, tpb.site_off, tpb.calls, tpb.t2_off, tpb.t2_calls, forced, kind, ib.read_off,
              ib.allele_off, ib.ploidy, ib.allele_del_len, ib.allele_ins_len, ib.allele_lnp, ib.read_length, ib.non_ambig, ib.is_fwd):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def k2b_fields(out: np.ndarray) -> np.ndarray:
    """the reference harness's fields of sx_ssnv_result records as one int32 array [field, site] (strandBias by its bits)"""
    return np.stack([np.ascontiguousarray(out[f]).view(np.int32) if f == "strandBias" else out[f].astype(np.int32) for f in K2B_REF_FIELDS])


def golden_key(model: str, point: str, mode: str = "") -> str:
    return f"{model}__{point}" + (f"__{mode}" if mode else "")


def _tier2_as_tier1(pb: B.PileupBatch) -> B.PileupBatch:
    """the tier2 view of each site (the tier1 calls that survive it, filter bits cleared, then the unfiltered tier2 calls, in that order)
    as a tier1-only batch"""
    n = pb.n_sites

    def part(off, calls, keep, rank):
        site = np.repeat(np.arange(n), np.diff(off.astype(np.int64)))
        c = calls[: int(off[-1])]
        k = keep(c)
        return site[k], np.full(int(k.sum()), rank), (c[k] & np.uint16(0x0FFF)).astype(np.uint16)

    s1, r1, c1 = part(pb.site_off, pb.calls, lambda c: ((c >> 12) & 1 == 0) | ((c >> 13) & 1 == 1), 0)
    s2, r2, c2 = part(pb.t2_off, pb.t2_calls, lambda c: (c >> 12) & 1 == 0, 1)
    site, rank, calls = np.concatenate([s1, s2]), np.concatenate([r1, r2]), np.concatenate([c1, c2])
    order = np.lexsort((np.arange(site.size), rank, site))
    off = np.concatenate([[0], np.cumsum(np.bincount(site, minlength=n))]).astype(np.uint32)
    return B.PileupBatch(off, calls[order], pb.ref_base, pb.ploidy)


def ntype_unset(p: A.SxParams, npb: B.PileupBatch, tpb: B.PileupBatch) -> np.ndarray:
    """The sites where the reference leaves `ntype` unassigned: a tier whose six posteriors are all NaN (a quality-0 call can make a whole
    term list -inf; ln of a negative non-strand error rate is NaN) never passes `err_som_and_ngt < min_not_somfrom_sum`
    (qscore_calculator.cpp:198-203), and its snv_result_set is a default-initialised local (position_somatic_snv_strand_grid.cpp:265).
    The device and the oracle report 0 there (include/strelka_b200.h, sx_ssnv_result).  Found from the oracle: such a tier has qphred 3070
    (log10 of NaN loses to the floor) and from_ntype_qphred 0; an evaluated tier with any finite posterior has from_ntype_qphred >= 2
    when its qphred is 3070."""
    ones = np.ones(npb.n_sites, np.uint8)

    def unset(r):
        return (r["is_computed"] == 1) & (r["qphred"] == 3070) & (r["from_ntype_qphred"] == 0)

    n1, t1 = specgen.somatic_tier2_view(npb, tpb, "neither")
    m = unset(reflib.ox_somatic(p, n1, t1, ones))
    if npb.t2_off is not None and tpb.t2_off is not None:
        m |= unset(reflib.ox_somatic(p, _tier2_as_tier1(npb), _tier2_as_tier1(tpb), ones))
    return m


def reference_fields(p: A.SxParams, npb: B.PileupBatch, tpb: B.PileupBatch, forced) -> np.ndarray:
    """the reference's answer as k2b_fields, with ntype 0 where the reference leaves it unassigned (ntype_unset): what the device and the
    oracle report there, and what is frozen, since the reference's own value there changes with what ran before it in the process"""
    f = k2b_fields(reflib.ref_somatic(p, npb, tpb, forced))
    f[K2B_REF_FIELDS.index("ntype")][ntype_unset(p, npb, tpb)] = 0
    return f


def compare_fields(got: np.ndarray, want: np.ndarray, what=""):
    """sx_ssnv_result records against reference fields (reference_fields), field by field"""
    g = k2b_fields(got)
    for i, f in enumerate(K2B_REF_FIELDS):
        bad = np.nonzero(g[i] != want[i])[0]
        assert bad.size == 0, (what, f, int(bad[0]), int(g[i][bad[0]]), int(want[i][bad[0]]))
