"""K2c site_continuous test support: seeded multi-sample columns that reach every branch of the model, and the three implementations the
tests compare with the device --
   oracle/continuous_oracle.cpp     -- the scalar restatement of the reference's loops (libcontinuous_oracle.so)
   tests/cpp/k2c_core_host.cpp      -- the kernels' own body (strelka_b200/csrc/k2c_core.cuh) compiled with g++
   oracle/_ref/libstrelka_ref_continuous.so -- the reference's getAlleleSequencingErrorQscore and strandBias (where built)
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200 import batch as B  # noqa: E402

ORACLE_SO = os.path.join(ROOT, "oracle", "libcontinuous_oracle.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libstrelka_ref_continuous.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "continuous_ref.npz")
GRID_N = 16384   # the GQ grid covers every total depth up to this
# |K2c - reference| of strandBias (the reference evaluates Boost's binomial pdf in x87 long double, K2c in double): largest measured on the
# frozen answers 1.0e-12; pinned with a thousandfold margin, still far below the 0.05 step of the printed SB / SNVSB
SB_BOUND = 1e-9
_libs: dict = {}
_RUN_ARGS = [C.POINTER(A.SxContOpts), C.c_double, C.POINTER(A.SxContBatch), C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32]


def oracle() -> C.CDLL:
    if "ox" not in _libs:
        subprocess.check_call(["make", "-s", "-C", os.path.join(ROOT, "oracle"), "-f", "continuous.mk", "libcontinuous_oracle.so"])
        lib = C.CDLL(ORACLE_SO)
        lib.ocont_run.argtypes = _RUN_ARGS
        lib.ocont_run.restype = C.c_uint32
        _libs["ox"] = lib
    return _libs["ox"]


def host_body() -> C.CDLL:
    if "core" not in _libs:
        _libs["dir"] = tempfile.TemporaryDirectory()
        so = os.path.join(_libs["dir"].name, "libk2c_core_host.so")
        subprocess.check_call(["g++", "-std=gnu++17", "-O2", "-fPIC", "-shared", "-Wall", "-ffp-contract=off", "-I" + os.path.join(ROOT, "include"),
                               "-I" + os.path.join(ROOT, "strelka_b200", "csrc"), os.path.join(ROOT, "tests", "cpp", "k2c_core_host.cpp"), "-o", so])
        lib = C.CDLL(so)
        lib.k2ccore_run.argtypes = _RUN_ARGS
        lib.k2ccore_run.restype = C.c_uint32
        lib.k2ccore_qscore.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_double, C.c_int32, C.c_void_p, C.c_void_p]
        lib.k2ccore_strand_bias.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        _libs["core"] = lib
    return _libs["core"]


def have_ref() -> bool:
    return os.path.exists(REF_SO)


def ref() -> C.CDLL:
    if "ref" not in _libs:
        lib = C.CDLL(REF_SO)
        lib.refc_qscore.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_void_p]
        lib.refc_strand_bias.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p]
        _libs["ref"] = lib
    return _libs["ref"]


def err_rate(opts: A.SxContOpts) -> float:
    return math.pow(10.0, -opts.expected_qscore / 10.0)


def default_opts() -> A.SxContOpts:
    return A.SxContOpts(0.01, 99.0, 17, 40)


def _run(fn, b: B.ContBatch, opts: A.SxContOpts, cap=None) -> B.ContOut:
    out = B.ContOut(b.n_sites, b.n_samples, B.cont_cap(b) if cap is None else cap)
    out.totals[0] = fn(C.byref(opts), err_rate(opts), C.byref(b.c), A.ptr(out.loci), A.ptr(out.samples), A.ptr(out.site_rec_off), out.cap_loci)
    return out


def ox_run(b, opts, cap=None) -> B.ContOut:
    return _run(oracle().ocont_run, b, opts, cap)


def core_run(b, opts, cap=None) -> B.ContOut:
    return _run(host_body().k2ccore_run, b, opts, cap)


def core_qscore(a, n, opts=None):
    opts = opts or default_opts()
    a, n = np.ascontiguousarray(a, np.uint32), np.ascontiguousarray(n, np.uint32)
    gq, st = np.zeros(a.size, np.int32), np.zeros(a.size, np.uint32)
    host_body().k2ccore_qscore(a.ctypes.data, n.ctypes.data, a.size, err_rate(opts), opts.max_qscore, gq.ctypes.data, st.ctypes.data)
    return gq, st


def core_strand_bias(counts: np.ndarray) -> np.ndarray:
    counts = np.ascontiguousarray(counts, np.uint32).reshape(-1, 4)
    out = np.zeros(len(counts))
    host_body().k2ccore_strand_bias(counts.ctypes.data, len(counts), out.ctypes.data)
    return out


def ref_qscore(a, n, expected_qscore=17, max_qscore=40):
    a, n = np.ascontiguousarray(a, np.uint32), np.ascontiguousarray(n, np.uint32)
    out = np.zeros(a.size, np.int32)
    ref().refc_qscore(a.ctypes.data, n.ctypes.data, a.size, expected_qscore, max_qscore, out.ctypes.data)
    return out


def ref_strand_bias(counts: np.ndarray) -> np.ndarray:
    counts = np.ascontiguousarray(counts, np.uint32).reshape(-1, 4)
    out = np.zeros(len(counts))
    ref().refc_strand_bias(counts.ctypes.data, len(counts), out.ctypes.data)
    return out


# ---- the GQ grid: per n <= GRID_N, the first a whose GQ reaches each of 1..40 (0xffff where no a <= n does)
def grid_pairs():
    """every (a, n) with n <= GRID_N and a <= min(n, L + 10 sqrt(L) + 40), L = n * 10^-1.7: past the first a at GQ 40 by more than a few"""
    ns, As = [], []
    for n in range(GRID_N + 1):
        lam = n * 10 ** -1.7
        top = min(n, int(lam + 10 * math.sqrt(lam) + 40))
        ns.append(np.full(top + 1, n, np.uint32))
        As.append(np.arange(top + 1, dtype=np.uint32))
    return np.concatenate(As), np.concatenate(ns)


def grid_thresholds(a, n, gq):
    """(first[n, q-1] = the first a with GQ >= q, 0xffff if none; the top a evaluated per n); asserts GQ ascends in a"""
    first = np.full((GRID_N + 1, 40), 0xFFFF, np.uint16)
    top = np.zeros(GRID_N + 1, np.uint32)
    starts = np.flatnonzero(np.r_[True, n[1:] != n[:-1]])
    ends = np.r_[starts[1:], len(n)]
    for s, e in zip(starts, ends):
        g = gq[s:e]
        assert np.all(np.diff(g) >= 0), f"GQ not ascending in a at n={n[s]}"
        nn = int(n[s])
        top[nn] = a[e - 1]
        for q in range(1, 41):
            k = np.searchsorted(g, q)
            if k < len(g):
                first[nn, q - 1] = a[s + k]
    return first, top


def gq_from_thresholds(first, a, n):
    f = first[n].astype(np.int64)
    return (f <= a[:, None].astype(np.int64)).sum(axis=1).astype(np.int32)


def sampled_large_pairs(seed=7, count=20000):
    """pairs past the grid's top a (where GQ is 40), and deeper than the grid"""
    rng = np.random.default_rng(seed)
    n = rng.integers(2000, 200000, count).astype(np.uint32)
    lam = n * 10 ** -1.7
    lo = np.minimum(n, (lam + 10 * np.sqrt(lam) + 41).astype(np.uint32))
    a = (lo + (rng.random(count) * (n - lo + 1)).astype(np.uint32)).clip(max=n).astype(np.uint32)
    keep = a > lam + 10 * np.sqrt(lam) + 40
    return a[keep], n[keep]


def strand_bias_cases(seed=3) -> np.ndarray:
    """seeded (fwdAlt, revAlt, fwdOther, revOther): zero totals, a = n on one or both strands, very unbalanced strands, deep columns"""
    rng = np.random.default_rng(seed)
    rows = [[0, 0, 0, 0], [1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1], [5, 5, 0, 0], [5, 0, 0, 5], [0, 5, 5, 0], [3000, 0, 0, 3000],
            [3000, 3000, 0, 0], [1, 1, 3000, 3000], [2000, 0, 0, 0], [0, 0, 2000, 2000], [1, 0, 9999, 0], [1, 1, 1, 1]]
    for _ in range(3000):
        kind = int(rng.integers(0, 5))
        depth = int(rng.choice([5, 30, 300, 3000, 8000]))
        f = int(rng.binomial(depth, rng.choice([0.5, 0.1, 0.01, 0.0, 1.0])))
        r = depth - f
        af_f = float(rng.choice([0.0, 0.005, 0.02, 0.3, 0.5, 1.0])) if kind else float(rng.random())
        af_r = af_f if kind in (0, 1) else float(rng.choice([0.0, 0.005, 0.02, 0.5, 1.0]))
        fa, ra = int(rng.binomial(f, af_f)), int(rng.binomial(r, af_r))
        rows.append([fa, ra, f - fa, r - ra])
    return np.array(rows, np.uint32)


# ---- seeded columns
BASES = "ACGT"


def _calls(rng, n, probs, fwd_frac=0.5, filt_frac=0.03, any_frac=0.01):
    base = rng.choice(4, size=n, p=probs)
    base = np.where(rng.random(n) < any_frac, 4, base)
    fwd = rng.random(n) < fwd_frac
    filt = rng.random(n) < filt_frac
    q = rng.integers(0, 64, n)
    return list(B.pack_call(q, base, fwd, rng.random(n) < 0.1, filt, filt & (rng.random(n) < 0.5)))


KINDS = ("empty", "ordinary", "n_ref", "only_any", "only_filtered", "forced_empty", "vf_exact", "ref_fallback", "multi_alt", "count_ties", "deep",
         "one_strand", "forced_n_ref")


def site_columns(rng, kind: str, S: int):
    """-> (per-sample call lists, ref base, forced)"""
    ref = BASES[int(rng.integers(0, 4))]
    r = BASES.index(ref)
    forced = bool(rng.random() < 0.15)
    cols = []
    for s in range(S):
        if kind == "empty":
            cols.append([])
            continue
        if kind == "forced_empty":
            forced = True
            cols.append([])
            continue
        p = np.full(4, 0.002)
        p[r] = 1.0
        if kind == "ordinary":
            p[(r + 1) % 4] = float(rng.choice([0.0, 0.005, 0.05, 0.3, 1.0]))
        elif kind == "multi_alt":
            p[(r + 1) % 4], p[(r + 2) % 4], p[(r + 3) % 4] = 0.3, 0.2, 0.1
        elif kind == "count_ties":
            p[:] = 1.0
        p = p / p.sum()
        n = int(rng.integers(1, 60))
        if kind == "deep":
            n = int(rng.integers(3000, 7500))
            p = np.full(4, 0.001)
            p[r] = 1.0
            p[(r + 2) % 4] = float(rng.choice([0.005, 0.01, 0.3]))
            p /= p.sum()
        if kind == "only_any":
            cols.append(_calls(rng, n, p, any_frac=1.0, filt_frac=0.0))
        elif kind == "only_filtered":
            cols.append(_calls(rng, n, p, filt_frac=1.0))
        elif kind == "vf_exact":
            # 100 non-ANY cleaned calls with exactly 1 or 99 alt calls: AF at min_het_vf and at 1 - min_het_vf
            k = int(rng.choice([1, 99, 50, 0]))
            base = np.array([(r + 1) % 4] * k + [r] * (100 - k))
            fwd = rng.random(100) < 0.5
            cols.append(list(B.pack_call(rng.integers(0, 64, 100), base, fwd, 0, 0, 0)) + _calls(rng, 5, p, any_frac=1.0, filt_frac=0.5))
        elif kind == "ref_fallback":
            cols.append(list(B.pack_call(rng.integers(0, 64, n), np.full(n, r), rng.random(n) < 0.5, 0, rng.random(n) < 0.1, 0)))
            forced = False
        elif kind == "one_strand":
            cols.append(_calls(rng, n, p, fwd_frac=float(rng.choice([0.0, 1.0]))))
        elif kind == "count_ties":
            m = int(rng.integers(1, 8))
            base = np.repeat(np.arange(4), m)
            cols.append(list(B.pack_call(rng.integers(0, 64, 4 * m), base, rng.random(4 * m) < 0.5, 0, 0, 0)))
        else:
            cols.append(_calls(rng, n, p))
    if kind in ("n_ref", "forced_n_ref"):
        ref = "N"
        forced = kind == "forced_n_ref"
    return cols, ref, forced


def case(seed: int, S: int, n_sites: int = 400, kinds=KINDS, pos_begin: int = 1000) -> B.ContBatch:
    rng = np.random.default_rng(seed)
    per_sample = [[] for _ in range(S)]
    refs, forced = [], []
    for _ in range(n_sites):
        cols, rb, f = site_columns(rng, kinds[int(rng.integers(0, len(kinds)))], S)
        for s in range(S):
            per_sample[s].append(cols[s])
        refs.append(rb)
        forced.append(f)
    samples = [B.PileupBatch.from_sites(per_sample[s], "".join(refs)) for s in range(S)]
    return B.ContBatch(samples, pos_begin, np.array(forced, np.uint8) if any(forced) else None)


def same(a: B.ContOut, b: B.ContOut) -> None:
    n = int(a.totals[0])
    assert n == int(b.totals[0])
    assert np.array_equal(a.site_rec_off, b.site_rec_off)
    assert a.loci[:n].tobytes() == b.loci[:n].tobytes(), "records differ"
    assert a.samples[: n * a.n_samples].tobytes() == b.samples[: n * b.n_samples].tobytes(), "sample entries differ"
