"""K4m (pile-up scoring metrics) on the CPU: the numpy host builder (batch.pileup_metrics) against the per-site statistics of
strelka_b200/csrc/k4m_core.cuh compiled with g++, bit for bit, on the same observations; and the cases reach every branch."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import pileup_metrics_gen as G
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_lib = None


def core():
    global _lib
    if _lib is None:
        so = os.path.join(tempfile.mkdtemp(prefix="k4mcore"), "libk4mcore.so")
        subprocess.check_call(["g++", "-std=c++14", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "include"),
                               "-I" + os.path.join(ROOT, "strelka_b200", "csrc"), os.path.join(ROOT, "tests", "cpp", "k4m_core_host.cpp"), "-o", so])
        _lib = C.CDLL(so)
        _lib.k4m_host_sites.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p]
        _lib.k4m_host_pack.restype = C.c_uint64
        _lib.k4m_host_pack.argtypes = [C.c_uint32] * 9
        _lib.k4m_host_edge_distance.restype = C.c_uint32
        _lib.k4m_host_edge_distance.argtypes = [C.c_uint32] * 3
    return _lib


def core_sites(obs, mode):
    lib = core()
    off = np.zeros(len(obs) + 1, np.uint32)
    off[1:] = np.cumsum([len(o) for o in obs])
    words = np.array([lib.k4m_host_pack(*(int(x) for x in t)) for o in obs for t in o] + [0], np.uint64)
    out = np.zeros(len(obs), A.PILEUP_METRICS_DT)
    lib.k4m_host_sites(words.ctypes.data, off.ctypes.data, len(obs), mode, out.ctypes.data)
    return out


def same_bits(a, b):
    return a.tobytes() == b.tobytes()


CASES = [(name, seed) for name in G.OPTION_SETS for seed in (1, 2)]


@pytest.mark.parametrize("mode", G.MODES)
@pytest.mark.parametrize("name,seed", CASES)
def test_builder_equals_core(name, seed, mode):
    pb = G.random_batch(seed, G.OPTION_SETS[name], n_reads=150, qual_dict=seed == 2)
    obs = []
    want = B.pileup_metrics(pb, mode, observations=obs)
    assert same_bits(core_sites(obs, mode), want)
    assert want["mapq_count"].sum() > 0


@pytest.mark.parametrize("mode", G.MODES)
def test_edge_batch(mode):
    pb = G.edge_batch()
    obs = []
    want = B.pileup_metrics(pb, mode, observations=obs)
    assert same_bits(core_sites(obs, mode), want)
    if mode == A.SX_PM_SOMATIC:
        sizes = set(want["n_alt_read_pos"].tolist())
        assert {0, 1, 2, 3}.issubset(sizes) and any(s >= 4 and s % 2 == 0 for s in sizes) and any(s >= 5 and s % 2 == 1 for s in sizes)
        assert (want["median_read_pos_var"] > 0).any()


def test_full_read_edge_distance():
    pb = G.random_batch(3, n_reads=120)
    fl, fo = G.full_read_arrays(pb, 3)
    obs = []
    want = B.pileup_metrics(pb, A.SX_PM_GERMLINE, fl, fo, observations=obs)
    assert same_bits(core_sites(obs, A.SX_PM_GERMLINE), want)
    assert not same_bits(want, B.pileup_metrics(pb, A.SX_PM_GERMLINE))
    lib = core()
    assert [lib.k4m_host_edge_distance(p, o, n) for p, o, n in ((0, 0, 10), (9, 0, 10), (5, 0, 10), (30, 0, 100), (3, 2, 4), (4, 0, 4))] == [0, 0, 4, 20, 5, 4]  # (the last two: the unsigned wrap of a segment past the full read)


def test_deep_site_and_overflow():
    pb = G.deep_batch(1200)
    obs = []
    want = B.pileup_metrics(pb, A.SX_PM_GERMLINE, observations=obs)
    assert want["mapq_count"].max() > 512
    assert same_bits(core_sites(obs, A.SX_PM_GERMLINE), want)
    pb = G.overflow_batch()
    obs = []
    want = B.pileup_metrics(pb, A.SX_PM_GERMLINE, observations=obs)
    assert want["status"][5] & A.SX_PM_ST_MQ_OVERFLOW and want["mq_ranksum"][5] == 0.0
    assert same_bits(core_sites(obs, A.SX_PM_GERMLINE), want)


@pytest.mark.parametrize("mode", G.MODES)
def test_reference_goldens(mode):
    """the numpy builder and the g++ core equal the reference's own pileup_read_segment with the metrics on (frozen in
    tests/golden/pileup_metrics_ref.npz; and the live harness where oracle/_ref is built), bit for bit"""
    gold = G.golden()
    n = 0
    for key, pb, m in G.golden_cases():
        if m != mode:
            continue
        obs = []
        got = B.pileup_metrics(pb, mode, observations=obs)
        assert same_bits(got, gold[key]), key
        assert same_bits(core_sites(obs, mode), gold[key]), key
        if G.have_ref():
            assert same_bits(G.ref_metrics(pb, mode), gold[key]), key
        n += 1
    assert n == 2 * len(G.OPTION_SETS) + 2


@pytest.mark.parametrize("name", sorted(G.OPTION_SETS))
def test_somatic_filter_matches_k4(name):
    """the somatic-eligible bases are K4's tier1 calls with current_call_filter clear: per position, the alt list's length is the number of
    non-reference tier1 base_call words of the (reference-pinned) K4 oracle with bit 12 clear"""
    import reflib

    pb = G.random_batch(4, G.OPTION_SETS[name])
    site_off, calls = reflib.ox_pileup_reads(pb)[:2]
    ref = bytes(pb.ref[: int(pb.c.ref_len)])
    rb = int(pb.c.report_begin) - int(pb.c.ref_begin)
    want = np.zeros(pb.n_sites, np.uint32)
    for s in range(pb.n_sites):
        for c in calls[int(site_off[s]) : int(site_off[s + 1])].tolist():
            if not (c >> 12) & 1 and "ACGTN"[(c >> 6) & 15] != chr(ref[rb + s]):
                want[s] += 1
    got = B.pileup_metrics(pb, A.SX_PM_SOMATIC)["n_alt_read_pos"]
    assert np.array_equal(got, want) and want.sum() > 0


def test_branches_reached():
    """the cases reach: sub-mapped and tier-2 reads, filtered calls, MAPQ 0 and 255, reverse strand, the var < 1e-4 branch, single-category
    and empty positions, rank ties"""
    pb = G.random_batch(1, G.OPTION_SETS["default"], n_reads=150)
    obs = []
    germ = B.pileup_metrics(pb, A.SX_PM_GERMLINE, observations=obs)
    flat = np.array([t for o in obs for t in o], np.int64)
    assert (flat[:, 3] == 1).any() and (flat[:, 0] == 0).any() and (flat[:, 0] == 255).any()
    assert (flat[:, 6] != flat[:, 7]).any()  # reverse-strand cycles
    som = B.pileup_metrics(pb, A.SX_PM_SOMATIC, observations=(o2 := []))
    flat2 = np.array([t for o in o2 for t in o], np.int64)
    assert (flat2[:, 4] == 0).any() and (flat2[:, 4] == 1).any()  # filtered and kept calls
    tiers = pb.reads["flags"][: pb.n_reads]
    assert ((tiers & A.SX_PRF_TIER1OR2) != 0).any() and ((tiers & A.SX_PRF_TIER1) == 0).any()
    assert (B.pileup_metrics(G.edge_batch(), A.SX_PM_GERMLINE)["mapq_count"] == 0).any()  # empty positions
    # ambiguous-end trimming on both strands, soft clips at both ends, reads across both report edges
    rb, re = int(pb.c.report_begin), int(pb.c.report_end)
    trimmed, clipped, edges = set(), False, set()
    for r in range(pb.n_reads):
        rd = pb.reads[r]
        n, so, fwd = int(rd["len"]), int(rd["seq_off"]), bool(int(rd["flags"]) & A.SX_PRF_FWD)
        end = n - 1 if fwd else 0
        if (int(pb.seq4[so + (end >> 1)]) >> (4 if end % 2 == 0 else 0)) & 15 == 15:
            trimmed.add(fwd)
        kinds = [int(x["kind"]) for x in pb.segs[int(rd["seg_off"]) : int(pb.reads[r + 1]["seg_off"])] if int(x["kind"]) != A.SX_SEG_HARDCLIP]
        clipped |= kinds[0] == A.SX_SEG_SOFTCLIP and kinds[-1] == A.SX_SEG_SOFTCLIP
        span = sum(int(x["len"]) for x in pb.segs[int(rd["seg_off"]) : int(pb.reads[r + 1]["seg_off"])] if int(x["kind"]) in (0, 5, 6))
        for e in (rb, re):
            if int(rd["pos"]) < e < int(rd["pos"]) + span:
                edges.add(e)
    assert trimmed == {True, False} and clipped and edges == {rb, re}
    # 'N' calls at 'N' reference positions count as reference
    eb = G.edge_batch()
    eobs = []
    B.pileup_metrics(eb, A.SX_PM_GERMLINE, observations=eobs)
    ref = bytes(eb.ref[: int(eb.c.ref_len)])
    n_sites = [s for s in range(eb.n_sites) if chr(ref[int(eb.c.report_begin) + s]) == "N"]
    assert n_sites and any(t[2] for s in n_sites for t in eobs[s])
    # a single-category position (all reference: var < 1e-4 -> 0), a two-category one whose values are all tied (z = 0), rank sums otherwise
    cats = [(s, {bool(t[2]) for t in o}, {t[0] for t in o}) for s, o in enumerate(obs) if o]
    assert any(c == {True} and germ["mq_ranksum"][s] == 0.0 for s, c, _ in cats)
    egerm = B.pileup_metrics(eb, A.SX_PM_GERMLINE)
    ecats = [(s, {bool(t[2]) for t in o}, {t[0] for t in o}) for s, o in enumerate(eobs) if o]
    assert any(c == {True, False} and len(v) == 1 and egerm["mq_ranksum"][s] == 0.0 for s, c, v in ecats)
    assert (germ["mq_ranksum"] != 0.0).any()
