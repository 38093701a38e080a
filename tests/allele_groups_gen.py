"""K6g allele_groups test infrastructure: seeded one-sample cases with allele groups, and the loaders of the CPU checkers
   oracle/liballele_groups_oracle.so   -- the scalar restatement on std::map containers (oracle/allele_groups_oracle.cpp)
   tests/cpp/k6g_core_host.cpp         -- the kernels' own body (strelka_b200/csrc/k6g_core.cuh) compiled with g++

A case's sample is the tumor sample of indel_reads_gen.synthetic_case (K6-shaped records drawn directly: tier-2 reads, suboverlap marks,
read ids permuted against read order, ids indexed differently by overlapping regions).  Its groups are drawn from ids that share windows, so
that reads cover several alleles of a group, some alleles of it or none of them, and contrast alleles are present or absent per read."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

import indel_reads_gen as G
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

ROOT = G.ROOT
ORACLE_SO = os.path.join(ROOT, "oracle", "liballele_groups_oracle.so")
_libs: dict = {}
_ARGS = [C.POINTER(A.SxIndelReadsSample), C.POINTER(A.SxAlleleGroups), C.POINTER(A.SxAlleleGroupReadsOut)]


def oracle() -> C.CDLL:
    if "ox" not in _libs:
        if not os.path.exists(ORACLE_SO):
            subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "allele_groups.mk", "liballele_groups_oracle.so"])
        lib = C.CDLL(ORACLE_SO)
        lib.ox_link_allele_groups.argtypes = _ARGS
        _libs["ox"] = lib
    return _libs["ox"]


def host_body() -> C.CDLL:
    if "core" not in _libs:
        _libs["dir"] = tempfile.TemporaryDirectory()
        so = os.path.join(_libs["dir"].name, "libk6gcore.so")
        subprocess.check_call(["g++", "-std=c++14", "-O2", "-fPIC", "-shared", "-Wall", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "strelka_b200", "csrc"),
                               os.path.join(ROOT, "tests", "cpp", "k6g_core_host.cpp"), "-o", so])
        lib = C.CDLL(so)
        lib.k6gcore_run.argtypes = _ARGS + [C.c_uint32]
        _libs["core"] = lib
    return _libs["core"]


def _run(fn, sample, groups, cap_reads, cap_lnp, *extra):
    cr, cl = B.allele_group_caps(sample, groups)
    out = B.AlleleGroupReadsOut(groups.n_groups, int(groups.allele_off[-1]), cr if cap_reads is None else cap_reads, cl if cap_lnp is None else cap_lnp)
    return fn(C.byref(sample.c), C.byref(groups.c), C.byref(out.c), *extra), out


def ox_link(sample, groups, cap_reads=None, cap_lnp=None):
    """(rc, AlleleGroupReadsOut) of the oracle."""
    return _run(oracle().ox_link_allele_groups, sample, groups, cap_reads, cap_lnp)


def core_link(sample, groups, cap_reads=None, cap_lnp=None, smem_sort=G.SMEM_SORT):
    """(rc, AlleleGroupReadsOut) of the host-compiled kernel body."""
    return _run(host_body().k6gcore_run, sample, groups, cap_reads, cap_lnp, smem_sort)


def same(a: B.AlleleGroupReadsOut, b: B.AlleleGroupReadsOut) -> None:
    """Every output array, byte for byte."""
    for x, y, name in zip(a.trimmed(), b.trimmed(), B.AlleleGroupReadsOut.ARRAYS):
        assert x.tobytes() == y.tobytes(), name


def ids_by_window(sample):
    """The window id lists of the sample's regions (ids that reads of one region can cover together)."""
    return [sample.key_gid[int(sample.region_key_off[g]) : int(sample.region_key_off[g + 1])] for g in range(sample.n_regions)]


def random_groups(rng, sample, n_gid, gid_key, n_groups, max_contrast=5, orphan_frac=0.05):
    """Groups of 1..4 alleles drawn from one region's window (so reads cover several of them), contrasts from the same window or anywhere,
    ploidy 1 or 2; a few groups name an id no read has (the last ids of synthetic_case are in no window)."""
    wins = [w for w in ids_by_window(sample) if w.size]
    alleles, contrasts = [], []
    for _ in range(n_groups):
        w = wins[rng.integers(len(wins))]
        a = int(rng.integers(1, A.SX_INDEL_MAX_ALLELES + 1))
        pick = rng.choice(w, size=min(a, w.size), replace=False).tolist()
        if rng.random() < orphan_frac:
            pick[int(rng.integers(len(pick)))] = n_gid - 1 - int(rng.integers(2))
        c = int(rng.integers(0, max_contrast + 1)) if rng.random() < 0.7 else 0
        pool = np.concatenate([w, rng.integers(0, n_gid, 3).astype(np.uint32)])
        alleles.append(pick)
        contrasts.append([int(x) for x in rng.choice(pool, size=c)] if c else [])
    return B.AlleleGroups.from_lists(alleles, contrasts, rng.integers(1, 3, n_groups), gid_key)


# seed, synthetic_case kwargs, group count
CASES = [
    (0, {}, 400),
    (1, {"permute_ids": False, "depth": 3.0, "max_width": 4}, 300),
    (2, {"special": [(40, 4, 400)], "max_width": 5}, 500),        # one 4-wide window under many reads: groups of 4 alleles with support
    (3, {"special": [(100, 2, 2600)], "depth": 5.0}, 300),        # a narrow one: lists deeper than the shared-memory sort
    (4, {"dup": True, "tier2_frac": 0.6}, 400),
    (5, {"sub_frac": 0.9, "n_regions": 20}, 200),
    (6, {"special": [(10, 3, 1500), (200, 4, 300)], "dup": True, "max_width": 12}, 600),
]


def case(i: int):
    """(sample, groups)"""
    seed, kw, n_groups = CASES[i]
    _, tumor, loci = G.synthetic_case(seed, **kw)
    rng = np.random.default_rng(7100 + seed)
    groups = random_groups(rng, tumor, loci.n_gid, loci.gid_key, n_groups)
    if kw.get("special"):  # groups on the special windows themselves
        extra = [list(range(s0, s0 + min(w, 4))) for s0, w, _ in kw["special"]]
        al = [groups.group(g)[0] for g in range(groups.n_groups)] + extra + [e[:1] for e in extra]
        co = [groups.group(g)[1] for g in range(groups.n_groups)] + [[]] * len(extra) + [e[1:] for e in extra]
        pl = np.concatenate([groups.ploidy, np.full(2 * len(extra), 2, np.uint8)])
        groups = B.AlleleGroups.from_lists(al, co, pl, loci.gid_key)
    return tumor, groups


# ------------------------------------------------------------------------------------------------------------------
# the reference: score_indels into one IndelBuffer, then its own allele-group functions (oracle/ref_harness_germline_indel.cpp)
# ------------------------------------------------------------------------------------------------------------------
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libstrelka_ref_germline_indel.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "germline_indel_ref.npz")
REF_KEYS = ("read_off", "read_id", "lnp_off", "ext_lnp", "read_length", "non_ambig", "is_fwd", "out")


def have_ref() -> bool:
    return os.path.exists(REF_SO)


class _RefSample(C.Structure):
    _fields_ = [("b", C.POINTER(A.SxScoreIndelsBatch))] + [(n, C.c_void_p) for n in ("lnp", "ins_pool", "ins_off", "read_id")]


class _RefReads(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("read_off", "read_id", "lnp_off", "ext_lnp", "read_length", "non_ambig", "is_fwd")] + [("cap_reads", C.c_uint32),
                                                                                                                                  ("cap_lnp", C.c_uint32)]


def params_of(batch) -> A.SxParams:
    """the caller's options for one sample: the K6 batch's flank is the sample's min_read_bp_flank, which K5 reads too"""
    p = A.default_params()
    p.min_read_bp_flank = batch.opts.min_read_bp_flank
    return p


def ref_chain(batch, lnp, read_id, loci, groups):
    """The reference's own score_indels for one sample into ONE IndelBuffer, then per group getAlleleGroupSupportingReadIds,
    getAlleleLogLhoodFromRead on the extended group, and getVariantAlleleGroupGenotypeLhoodsForSample.  Returns a dict of REF_KEYS."""
    if "ref" not in _libs:
        _libs["ref"] = C.CDLL(REF_SO)
    sample = _RefSample(C.pointer(batch.c), A.ptr(lnp), A.ptr(batch.ins_pool), A.ptr(batch.ins_off), A.ptr(read_id))
    pool = np.frombuffer("".join(loci.ins).encode() + b"\0", np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(x) for x in loci.ins])]).astype(np.uint32)
    n, cap = groups.n_groups, batch.n_rec_slots + 1
    width = 1 + A.SX_INDEL_MAX_ALLELES + int(np.diff(groups.contrast_off.astype(np.int64)).max(initial=0))
    r = dict(read_off=np.zeros(n + 1, np.uint32), read_id=np.zeros(cap, np.uint32), lnp_off=np.zeros(n + 1, np.uint32), ext_lnp=np.zeros(cap * width, np.float64),
             read_length=np.zeros(cap, np.uint16), non_ambig=np.zeros(cap, np.uint16), is_fwd=np.zeros(cap, np.uint8))
    reads = _RefReads(*(A.ptr(r[k]) for k in REF_KEYS[:-1]), cap, cap * width)
    out = np.zeros(max(1, n), A.INDEL_RESULT_DT)
    err = C.create_string_buffer(1024)
    fn = _libs["ref"].ref_germline_indel_chain
    fn.argtypes = [C.POINTER(A.SxParams), C.POINTER(_RefSample), C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(A.SxAlleleGroups), C.c_void_p,
                   C.POINTER(_RefReads), C.c_char_p, C.c_int]
    p = params_of(batch)
    rc = fn(C.byref(p), C.byref(sample), A.ptr(loci.gid_key), A.ptr(pool), A.ptr(off), loci.n_gid, C.byref(groups.c), A.ptr(out), C.byref(reads), err, 1024)
    assert rc == 0, err.value.decode()
    nr, nl = int(r["read_off"][-1]), int(r["lnp_off"][-1])
    for k in ("read_id", "read_length", "non_ambig", "is_fwd"):
        r[k] = r[k][:nr]
    r["ext_lnp"] = r["ext_lnp"][:nl]
    r["out"] = out[:n]
    return r


def inputs_digest(batch, lnp, read_id, loci, groups) -> str:
    import hashlib

    h = hashlib.sha256()
    for a in (batch.region_read_off, batch.region_key_off, batch.keys, batch.aln_off, batch.aln_pos, batch.aln_seg_off, batch.segs, batch.aln_key_off, batch.aln_keys,
              batch.read_len, batch.non_ambig, batch.read_flags, batch.rec_off, lnp, read_id, loci.gid_key, groups.allele_off, groups.allele_gid, groups.contrast_off,
              groups.contrast_gid, groups.ploidy):
        h.update(np.ascontiguousarray(a).tobytes())
    h.update(np.int32(batch.opts.min_read_bp_flank).tobytes())
    h.update("|".join(loci.ins).encode())
    return h.hexdigest()


def frozen_ref_chain(key: str, digest: str) -> dict:
    """What ref_chain returned for case `key` when tests/golden/make_germline_indel_golden.py froze it."""
    g = np.load(GOLDEN)
    assert str(g[f"inputs{key}"]) == digest, "the generator no longer makes the inputs the answers were frozen for"
    r = {k: g[f"{k}{key}"] for k in REF_KEYS}
    r["out"] = np.frombuffer(r["out"].tobytes(), A.INDEL_RESULT_DT)
    return r


def fold(ext_lnp, A_: int):
    """the contrast fold of getVariantAlleleGroupGenotypeLhoodsForSample (AlleleGroupGenotype.cpp:225-238) on one read's extended vector"""
    v = list(ext_lnp)
    for i in range(A_ + 1, len(v)):
        if v[i] > v[0]:
            v[0] = v[i]
    return v[: A_ + 1]


def same_as_reference(linked: B.AlleleGroupReadsOut, groups, ref: dict, out) -> None:
    """The link's output against the reference's: per group the supporting-read count, per read (in ascending read id) the exemplar's fields
    and the allele log-likelihoods after the contrast fold, bit for bit; K5's results on the link's batch (`out`) against the reference's
    genotype likelihoods and supporting-read counts, whole records."""
    assert not linked.status[: groups.n_groups].any()
    assert np.array_equal(linked.read_off, ref["read_off"])
    assert np.all(np.diff(ref["read_id"].astype(np.int64))[np.diff(np.searchsorted(ref["read_off"][1:], np.arange(ref["read_id"].size), side="right")) == 0] > 0)
    n = int(linked.totals[0])
    for k in ("read_length", "non_ambig", "is_fwd"):
        assert getattr(linked, k)[:n].tobytes() == ref[k].tobytes(), k
    A_ = np.diff(groups.allele_off.astype(np.int64))
    want = []
    for g in range(groups.n_groups):
        w = int(ref["lnp_off"][g + 1] - ref["lnp_off"][g]) // max(1, int(ref["read_off"][g + 1] - ref["read_off"][g])) if ref["read_off"][g + 1] > ref["read_off"][g] else 0
        for i in range(int(ref["read_off"][g + 1] - ref["read_off"][g])):
            v = ref["ext_lnp"][int(ref["lnp_off"][g]) + i * w : int(ref["lnp_off"][g]) + (i + 1) * w]
            want.extend(fold(v, int(A_[g])))
    want = np.array(want, np.float64)
    assert np.array_equal(want.astype(np.float32).astype(np.float64), want)  # every value is a ReadPathScores float
    assert linked.allele_lnp[: int(linked.totals[1])].tobytes() == want.astype(np.float32).tobytes()
    assert out.tobytes() == ref["out"].tobytes()
