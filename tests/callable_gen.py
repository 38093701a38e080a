"""K2b's callable mode (isComputeNonSomatic) and the somatic callable regions, for the CPU tests, the frozen reference answers and the GPU tests:
   oracle/somatic_callable_oracle.cpp        -- the callable-mode restatement (forced K2b of liboracle.so + the non-somatic posterior)
   tests/cpp/k2b_nonsomatic_host.cpp         -- the kernel's own body (strelka_b200/csrc/k2b_nonsomatic.cuh) compiled with g++
   oracle/ref_harness_somatic_callable.cpp   -- the reference's position_somatic_snv_call(..., true, sgt) and SomaticCallableProcessor
The cases are specgen.somatic_edge_sites in each tier2 configuration (specgen.SOMATIC_TIER2_MODES) at the default parameters, and at every K2b point of
tests/site_params.py with tier2 calls on both samples.  NQSS reads only the tier1 likelihoods, which no parameter point and no tier2 configuration
changes: every case gives the same NQSS on the same sites, so the non-somatic posterior's coverage is that of the one 1320-site edge batch.  The
cases differ in the fields that decide the records and the callable track through QSS (qphred, the tiers, the tier2 copy)."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

import site_params as SP
import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SO = os.path.join(ROOT, "oracle", "libsomatic_callable_oracle.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libstrelka_ref_somatic_callable.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "somatic_callable_ref.npz")
CHROM, POS_BEGIN = "chr1", 1000
FIELDS = SP.K2B_REF_FIELDS + ("nonsomatic_qphred",)
_P = C.c_void_p
_libs: dict = {}


def cases():
    """[(name, params, normal, tumor, forced)]"""
    npb, tpb, forced, _ = SP.k2b_edge_batch()
    out = []
    for mode in specgen.SOMATIC_TIER2_MODES:
        n, t = specgen.somatic_tier2_view(npb, tpb, mode)
        out.append((f"default__{mode}", SP.k2b("default"), n, t, forced))
    for point in SP.K2B_POINTS:
        if point != "default":
            out.append((f"{point}__both", SP.k2b(point), npb, tpb, forced))
    return out


def inputs_digest() -> str:
    h = hashlib.sha256(SP.inputs_digest().encode())
    for name, p, _, _, _ in cases():
        h.update(name.encode())
        h.update(bytes(p))
    return h.hexdigest()


def oracle() -> C.CDLL:
    if "ox" not in _libs:
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "somatic_callable.mk", "libsomatic_callable_oracle.so"])
        lib = C.CDLL(ORACLE_SO)
        lib.ox_site_gl_somatic_callable.argtypes = [C.POINTER(A.SxParams), C.POINTER(A.SxPileupBatch), C.POINTER(A.SxPileupBatch), _P, _P]
        _libs["ox"] = lib
    return _libs["ox"]


def host_body() -> C.CDLL:
    if "core" not in _libs:
        _libs["dir"] = tempfile.TemporaryDirectory()
        so = os.path.join(_libs["dir"].name, "libk2b_nonsomatic_host.so")
        subprocess.check_call(["g++", "-std=gnu++17", "-O2", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", "-I" + os.path.join(ROOT, "include"),
                               "-I" + os.path.join(ROOT, "strelka_b200", "csrc"), os.path.join(ROOT, "tests", "cpp", "k2b_nonsomatic_host.cpp"), "-o", so])
        lib = C.CDLL(so)
        lib.k2bn_host_qphred.argtypes = [_P, C.c_uint64, _P]
        lib.k2bn_host_outcomes.argtypes = [_P, C.c_uint64, _P]
        _libs["core"] = lib
    return _libs["core"]


def have_ref() -> bool:
    return os.path.exists(REF_SO)


def ref() -> C.CDLL:
    if "ref" not in _libs:
        lib = C.CDLL(REF_SO)
        lib.ref_site_gl_somatic_callable.argtypes = [C.POINTER(A.SxParams), C.POINTER(A.SxPileupBatch), C.POINTER(A.SxPileupBatch), _P, C.c_char_p, C.c_int32,
                                                     _P, _P, C.c_uint64, C.POINTER(C.c_uint64), C.c_char_p, C.c_int]
        _libs["ref"] = lib
    return _libs["ref"]


def ox_callable(p: A.SxParams, npb: B.PileupBatch, tpb: B.PileupBatch, forced=None) -> np.ndarray:
    out = np.zeros(npb.n_sites, A.SSNV_RESULT_DT)
    f = None if forced is None else np.ascontiguousarray(forced, np.uint8)
    assert oracle().ox_site_gl_somatic_callable(C.byref(p), C.byref(npb.c), C.byref(tpb.c), A.ptr(f), out.ctypes.data) == 0
    return out


def tier1_records(p: A.SxParams, npb: B.PileupBatch, tpb: B.PileupBatch) -> np.ndarray:
    """forced K2b records of the tier1 view alone: the likelihoods the non-somatic posterior reads"""
    n1, t1 = specgen.somatic_tier2_view(npb, tpb, "neither")
    import reflib

    return reflib.ox_somatic(p, n1, t1, np.ones(npb.n_sites, np.uint8))


def host_nonsomatic(tier1: np.ndarray) -> np.ndarray:
    t = np.ascontiguousarray(tier1)
    out = np.zeros(t.size, np.int32)
    host_body().k2bn_host_qphred(t.ctypes.data, t.size, out.ctypes.data)
    return out


def host_outcomes(tier1: np.ndarray) -> np.ndarray:
    t = np.ascontiguousarray(tier1)
    out = np.zeros(t.size, np.uint32)
    host_body().k2bn_host_outcomes(t.ctypes.data, t.size, out.ctypes.data)
    return out


def ref_callable(p: A.SxParams, npb: B.PileupBatch, tpb: B.PileupBatch, forced=None, chrom: str = CHROM, pos_begin: int = POS_BEGIN):
    """the reference's (records, BED text)"""
    out = np.zeros(npb.n_sites, A.SSNV_RESULT_DT)
    f = None if forced is None else np.ascontiguousarray(forced, np.uint8)
    cap = 64 * npb.n_sites + 64
    bed = C.create_string_buffer(cap)
    n = C.c_uint64(0)
    err = C.create_string_buffer(1024)
    rc = ref().ref_site_gl_somatic_callable(C.byref(p), C.byref(npb.c), C.byref(tpb.c), A.ptr(f), chrom.encode(), pos_begin, out.ctypes.data, bed, cap,
                                            C.byref(n), err, 1024)
    assert rc == 0, (rc, err.value)
    return out, bed.value.decode()


def fields(out: np.ndarray) -> np.ndarray:
    """the reference harness's fields as one int32 array [field, site] (strandBias by its bits)"""
    return np.stack([np.ascontiguousarray(out[f]).view(np.int32) if f == "strandBias" else out[f].astype(np.int32) for f in FIELDS])


def reference_fields(p: A.SxParams, npb: B.PileupBatch, tpb: B.PileupBatch, forced):
    """(fields, BED text) of the reference, with ntype 0 where the reference leaves it unassigned (site_params.ntype_unset)"""
    r, bed = ref_callable(p, npb, tpb, forced)
    f = fields(r)
    f[FIELDS.index("ntype")][SP.ntype_unset(p, npb, tpb)] = 0
    return f, bed


def compare_fields(got: np.ndarray, want: np.ndarray, what=""):
    g = fields(got)
    for i, f in enumerate(FIELDS):
        bad = np.nonzero(g[i] != want[i])[0]
        assert bad.size == 0, (what, f, int(bad[0]), int(g[i][bad[0]]), int(want[i][bad[0]]))


def bed_text(begin: np.ndarray, end: np.ndarray, chrom: str = CHROM) -> str:
    return "".join(f"{chrom}\t{b}\t{e}\n" for b, e in zip(begin.tolist(), end.tolist()))


def host_bed(out: np.ndarray, pos_begin: int = POS_BEGIN, chrom: str = CHROM) -> str:
    return bed_text(*B.somatic_callable_regions(out, pos_begin), chrom=chrom)


def golden() -> dict:
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def synthetic_records(rng: np.random.Generator, n: int, p_callable: float) -> np.ndarray:
    """sx_ssnv_result records whose QSS and NQSS straddle the threshold of 15, callable with probability about p_callable"""
    r = np.zeros(n, A.SSNV_RESULT_DT)
    c = rng.random(n) < p_callable
    which = rng.integers(0, 3, n)  # callable by QSS, by NQSS, by both
    lo = lambda: rng.integers(0, 15, n)  # noqa: E731
    hi = lambda: rng.integers(15, 200, n)  # noqa: E731
    r["qphred"] = np.where(c & (which != 1), hi(), lo())
    r["nonsomatic_qphred"] = np.where(c & (which != 0), hi(), lo())
    r["is_computed"] = 1
    return r


# ---- the somatic window pass in callable mode: a digest of its NQSS, QSS and callable regions, frozen from the reference
WINDOW_GOLDEN = os.path.join(ROOT, "tests", "golden", "somatic_callable_window_digests.json")


def window_digest(qphred: np.ndarray, nonsomatic_qphred: np.ndarray, begin: np.ndarray, end: np.ndarray) -> str:
    h = hashlib.sha256()
    for a in (np.asarray(qphred, np.int32), np.asarray(nonsomatic_qphred, np.int32), np.asarray(begin, np.int32), np.asarray(end, np.int32)):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def bed_intervals(bed: str):
    f = [ln.split("\t") for ln in bed.splitlines()]
    return np.array([int(x[1]) for x in f], np.int32), np.array([int(x[2]) for x in f], np.int32)


def reference_window_digest(p: A.SxParams, pb, forced, pos_begin: int) -> str:
    """the reference's position_somatic_snv_call(..., true, sgt) and SomaticCallableProcessor on a window's two column sets"""
    r, bed = ref_callable(p, pb[0], pb[1], forced, pos_begin=pos_begin)
    return window_digest(r["qphred"], r["nonsomatic_qphred"], *bed_intervals(bed))
