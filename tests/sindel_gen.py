"""K5b somatic_indel test infrastructure: the seeded synthetic batch generator and the loaders of the two CPU checkers
   oracle/libsindel_oracle.so              -- our scalar restatement (oracle/somatic_indel_oracle.cpp)
   oracle/_ref/libstrelka_ref_sindel.so    -- the reference's own get_somatic_indel behind a C shim (oracle/ref_harness_somatic_indel.cpp)
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from strelka_b200 import _abi as A
from strelka_b200 import batch as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SO = os.path.join(ROOT, "oracle", "libsindel_oracle.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libstrelka_ref_sindel.so")
_P = C.c_void_p
_libs: dict = {}

# locus kinds: (P(read supports the candidate) in the normal, in the tumor)
KINDS = np.array([[0.0, 0.3], [0.5, 0.5], [0.0, 0.0], [0.05, 0.08]])
KIND_P = [0.35, 0.2, 0.3, 0.15]  # somatic, germline, reference, noise


def random_somatic_indel_batch(rng: np.random.Generator, n: int, normal_depth: float = 40.0, tumor_depth: float = 60.0, tier2_frac: float = 0.2,
                               max_alts: int = 4, zero_depth_frac: float = 0.08, short_read_frac: float = 0.05, forced_frac: float = 0.1,
                               flank: int = 5) -> B.SomaticIndelBatch:
    """A seeded batch of n candidate indels.  Per locus: a kind (somatic / germline / reference / noise), a table of 0..max_alts distinct
    alternates within 8 bases of the candidate (so some pairs conflict and some do not), Poisson depths (some loci with none in a sample),
    and per read ref / indel / 0-2 alternate path scores drawn from the kind, 20 % tier2 reads, some reads at or below 2*flank bases."""
    kind = rng.choice(len(KIND_P), n, p=KIND_P)
    nd = rng.poisson(normal_depth, n)
    td = rng.poisson(tumor_depth, n)
    nd[rng.random(n) < zero_depth_frac] = 0
    td[rng.random(n) < zero_depth_frac] = 0
    key = np.zeros(n, A.INDEL_KEY_DT)
    key["pos"] = 1000
    key["del_len"] = rng.integers(0, 6, n)
    key["ins_len"] = rng.integers(0, 6, n)
    key["ins_len"][(key["del_len"] == 0) & (key["ins_len"] == 0)] = 1
    forced = (rng.random(n) < forced_frac).astype(np.uint8)
    err_table = np.array([1e-4, 5e-4, 2e-3, 8e-3, 0.03, 0.1], np.float64)
    err_idx = rng.integers(0, err_table.size, n).astype(np.uint32)

    n_alts = rng.integers(0, max_alts + 1, n)
    alt_off = np.zeros(n + 1, np.uint32)
    alt_off[1:] = np.cumsum(n_alts)
    na_tot = int(alt_off[-1])
    alt_locus = np.repeat(np.arange(n), n_alts)
    alts = np.zeros(na_tot, A.INDEL_KEY_DT)
    # a locus's entries are distinct IndelKeys: distinct (pos, del_len, ins_len), the insert sequence being the same for equal lengths
    # (ins_id 0), so the reference keys them apart exactly as the table does; a repeated triple is drawn again
    redo = np.ones(na_tot, bool)
    while redo.any():
        m = int(redo.sum())
        alts["pos"][redo] = 1000 + rng.integers(-8, 9, m)
        alts["del_len"][redo] = rng.integers(0, 5, m)
        alts["ins_len"][redo] = rng.integers(0, 4, m)
        alts["del_len"][(alts["del_len"] == 0) & (alts["ins_len"] == 0)] = 1
        code = ((alt_locus.astype(np.int64) * 64 + (alts["pos"] - 990)) * 8 + alts["del_len"]) * 8 + alts["ins_len"]
        _, first = np.unique(code, return_index=True)
        redo = np.ones(na_tot, bool)
        redo[first] = False

    depth = np.stack([nd, td], axis=1).ravel()  # normal, tumor, normal, ...
    read_off = np.zeros(2 * n + 1, np.uint32)
    read_off[1:] = np.cumsum(depth)
    R = int(read_off[-1])
    slot = np.repeat(np.arange(2 * n), depth)
    locus, sample = slot // 2, slot % 2
    reads = np.zeros(R, A.SINDEL_READ_DT)
    supports = rng.random(R) < KINDS[kind[locus], sample]
    good, bad = -rng.uniform(0, 2, R), -rng.uniform(4, 25, R)
    reads["indel"] = np.where(supports, good, bad).astype(np.float32)
    reads["ref"] = np.where(supports, bad, good).astype(np.float32)
    rlen = rng.integers(100, 151, R)
    short = rng.random(R) < short_read_frac
    rlen[short] = rng.integers(0, 2 * flank + 2, int(short.sum()))
    reads["read_length"] = rlen
    reads["non_ambig"] = (rlen * rng.uniform(0.5, 1.0, R)).astype(np.uint16)
    reads["is_tier1"] = (rng.random(R) >= tier2_frac).astype(np.uint8)
    la = n_alts[locus]
    k = np.minimum(rng.integers(0, 3, R), la)
    reads["n_alt"] = k
    a0 = rng.integers(0, np.maximum(la, 1))
    a1 = (a0 + 1 + rng.integers(0, np.maximum(la - 1, 1))) % np.maximum(la, 1)
    reads["alt"][:, 0] = np.where(k > 0, a0, 0)
    reads["alt"][:, 1] = np.where(k > 1, a1, 0)
    alt_lnp = -rng.uniform(0, 25, (R, 2))
    alt_support = (k > 0) & (rng.random(R) < 0.15)
    alt_lnp[alt_support, 0] = -rng.uniform(0, 1.5, int(alt_support.sum()))
    alt_lnp[k < 1, 0] = 0
    alt_lnp[k < 2, 1] = 0
    reads["alt_lnp"] = alt_lnp.astype(np.float32)
    return B.SomaticIndelBatch(key, forced, err_idx, err_table, alt_off, alts, read_off, reads)


def oracle() -> C.CDLL:
    if "ox" not in _libs:
        if not os.path.exists(ORACLE_SO):
            subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "somatic_indel.mk", "libsindel_oracle.so"])
        lib = C.CDLL(ORACLE_SO)
        lib.ox_somatic_indel.argtypes = [C.POINTER(A.SxSindelOpts), C.POINTER(A.SxSindelBatch), _P, C.c_uint32, _P]
        _libs["ox"] = lib
    return _libs["ox"]


def have_ref() -> bool:
    return os.path.exists(REF_SO)


def ox_somatic_indel(opts: A.SxSindelOpts, sb: B.SomaticIndelBatch) -> np.ndarray:
    out = np.zeros(max(1, sb.n_loci), A.SINDEL_RESULT_DT)
    rc = oracle().ox_somatic_indel(C.byref(opts), C.byref(sb.c), A.ptr(sb.err_prob), sb.err_prob.size, A.ptr(out))
    assert rc == 0, rc
    return out[: sb.n_loci]


def ref_somatic_indel(opts: A.SxSindelOpts, sb: B.SomaticIndelBatch) -> np.ndarray:
    if "ref" not in _libs:
        lib = C.CDLL(REF_SO)
        lib.ref_somatic_indel.argtypes = [C.POINTER(A.SxSindelOpts), C.POINTER(A.SxSindelBatch), _P, C.c_uint32, _P, C.c_char_p, C.c_int]
        _libs["ref"] = lib
    out = np.zeros(max(1, sb.n_loci), A.SINDEL_RESULT_DT)
    err = C.create_string_buffer(1024)
    rc = _libs["ref"].ref_somatic_indel(C.byref(opts), C.byref(sb.c), A.ptr(sb.err_prob), sb.err_prob.size, A.ptr(out), err, 1024)
    assert rc == 0, err.value.decode()
    return out[: sb.n_loci]


def ref_somatic_indel_seconds(opts: A.SxSindelOpts, sb: B.SomaticIndelBatch) -> float:
    """Host seconds spent inside the reference's get_somatic_indel over the batch (one core; the harness's own object building excluded)."""
    ref_somatic_indel(opts, B.SomaticIndelBatch(sb.key[:0], sb.is_forced_output[:0], sb.err_idx[:0], sb.err_prob, sb.alt_off[:1], sb.alts[:0],
                                                sb.read_off[:1], sb.reads[:0]))  # loads the library
    lib = _libs["ref"]
    lib.ref_somatic_indel_timed.argtypes = [C.POINTER(A.SxSindelOpts), C.POINTER(A.SxSindelBatch), _P, C.c_uint32, _P, C.POINTER(C.c_double), C.c_char_p, C.c_int]
    out = np.zeros(max(1, sb.n_loci), A.SINDEL_RESULT_DT)
    secs = C.c_double(0)
    err = C.create_string_buffer(1024)
    rc = lib.ref_somatic_indel_timed(C.byref(opts), C.byref(sb.c), A.ptr(sb.err_prob), sb.err_prob.size, A.ptr(out), C.byref(secs), err, 1024)
    assert rc == 0, err.value.decode()
    return secs.value


# the parity cases: (seed, n_loci, generator kwargs, opts overrides)
CASES = [
    (0, 500, {}, {}),
    (1, 500, {"normal_depth": 6.0, "tumor_depth": 9.0, "zero_depth_frac": 0.25}, {}),
    (2, 500, {"tier2_frac": 0.5}, {"useTier2Evidence": 0}),
    (3, 500, {}, {"somatic_indel_rate": 3e-4, "bindel_diploid_theta": 2e-3, "indel_contam_tolerance": 0.4, "shared_indel_error_factor": 1.2}),
    (4, 500, {"short_read_frac": 0.4, "flank": 8}, {"min_read_bp_flank": (3, 8), "randomBaseMatchProb": 0.25, "tier2RandomBaseMatchProb": 0.4}),
    (5, 500, {"normal_depth": 20.0, "tumor_depth": 30.0, "forced_frac": 0.4, "max_alts": 8}, {}),
]


def case(i: int):
    seed, n, gk, ok = CASES[i]
    sb = random_somatic_indel_batch(np.random.default_rng(1000 + seed), n, **gk)
    o = A.default_sindel_opts()
    for k_, v in ok.items():
        if k_ == "min_read_bp_flank":
            o.min_read_bp_flank[0], o.min_read_bp_flank[1] = v
        else:
            setattr(o, k_, v)
    return sb, o


def inputs_digest(sb: B.SomaticIndelBatch) -> str:
    import hashlib

    h = hashlib.sha256()
    for a in (sb.key, sb.is_forced_output, sb.err_idx, sb.err_prob, sb.alt_off, sb.alts, sb.read_off, sb.reads):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def compare_to_reference(ox: np.ndarray, ref: np.ndarray, sb: B.SomaticIndelBatch, opts: A.SxSindelOpts) -> None:
    """Our record against the reference harness's: the final call (every defined field) and, for every tier the model evaluated,
    the 2x21 float likelihoods bit for bit and calculate_result_set_grid's result (qphred only where the multi-indel filter did not
    reject the tier)."""
    assert np.array_equal(ox["is_output"], ref["is_output"]), np.nonzero(ox["is_output"] != ref["is_output"])[0][:10]
    out = ox["is_output"] == 1
    for f in ("sindel_tier", "sindel_from_ntype_tier", "is_overlap", "max_gt", "qphred"):
        assert np.array_equal(ox[f][out], ref[f][out]), f
    defined = out & ~((sb.is_forced_output == 1) & (opts.useTier2Evidence == 0))
    for f in ("ntype", "from_ntype_qphred"):
        assert np.array_equal(ox[f][defined], ref[f][defined]), f
    for t in range(2):
        ev = ox["tier"][:, t]["evaluated"] == 1
        a, b = ox["tier"][:, t][ev], ref["tier"][:, t][ev]
        for f in ("normal_lhood", "tumor_lhood"):
            assert np.array_equal(a[f].view(np.uint32), b[f].view(np.uint32)), (t, f)
        for f in ("ntype", "max_gt", "from_ntype_qphred"):
            assert np.array_equal(a[f], b[f]), (t, f)
        kept = a["multi_indel"] == 0
        assert np.array_equal(a["qphred"][kept], b["qphred"][kept]), (t, "qphred")
        assert np.all(a["qphred"][~kept] == 0)
