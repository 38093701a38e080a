"""K6b indel_reads test infrastructure: seeded two-sample cases and the loaders of the CPU checkers
   oracle/libindel_reads_oracle.so   -- the scalar restatement on std::map containers (oracle/indel_reads_oracle.cpp)
   tests/cpp/k6b_core_host.cpp       -- the kernels' own body (strelka_b200/csrc/k6b_core.cuh) compiled with g++

Two kinds of case.  `synthetic_case` draws K6-shaped records directly, so that every shape the link must handle is there by construction
(see SYNTH_CASES).  `k6_case` runs the K6 generator of tests/specgen.py for two samples that share windows -- the tumor's copy of every
other window carries one more leading entry, so the same IndelKey has different window indices in the two samples -- and is what the
chain tests score with K6 and call with K5b."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile
from types import SimpleNamespace

import numpy as np

import reflib
import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SO = os.path.join(ROOT, "oracle", "libindel_reads_oracle.so")
SMEM_SORT = 512  # K6B_SMEM_SORT of k6b_indel_reads.cu
_libs: dict = {}
_ARGS = [C.POINTER(A.SxIndelReadsSample), C.POINTER(A.SxIndelReadsSample), C.POINTER(A.SxIndelLoci), C.POINTER(A.SxIndelReadsOut)]


def oracle() -> C.CDLL:
    if "ox" not in _libs:
        if not os.path.exists(ORACLE_SO):
            subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-f", "indel_reads.mk", "libindel_reads_oracle.so"])
        lib = C.CDLL(ORACLE_SO)
        lib.ox_link_indel_reads.argtypes = _ARGS
        _libs["ox"] = lib
    return _libs["ox"]


def host_body() -> C.CDLL:
    if "core" not in _libs:
        _libs["dir"] = tempfile.TemporaryDirectory()
        so = os.path.join(_libs["dir"].name, "libk6bcore.so")
        subprocess.check_call(["g++", "-std=c++14", "-O2", "-fPIC", "-shared", "-Wall", "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "strelka_b200", "csrc"),
                               os.path.join(ROOT, "tests", "cpp", "k6b_core_host.cpp"), "-o", so])
        lib = C.CDLL(so)
        lib.k6bcore_run.argtypes = _ARGS + [C.c_uint32]
        _libs["core"] = lib
    return _libs["core"]


def caps(normal, tumor, loci):
    cap_reads = int(normal.n_rec[: normal.n_reads].sum()) + int(tumor.n_rec[: tumor.n_reads].sum())
    return cap_reads, min(2 * cap_reads, A.SX_SINDEL_MAX_ALTS * loci.n_loci)


def _run(fn, normal, tumor, loci, cap_reads, cap_alts, *extra):
    cr, ca = caps(normal, tumor, loci)
    out = B.IndelReadsOut(loci.n_loci, cr if cap_reads is None else cap_reads, ca if cap_alts is None else cap_alts)
    return fn(C.byref(normal.c), C.byref(tumor.c), C.byref(loci.c), C.byref(out.c), *extra), out


def ox_link(normal, tumor, loci, cap_reads=None, cap_alts=None):
    """(rc, IndelReadsOut) of the oracle."""
    return _run(oracle().ox_link_indel_reads, normal, tumor, loci, cap_reads, cap_alts)


def core_link(normal, tumor, loci, cap_reads=None, cap_alts=None, smem_sort=SMEM_SORT):
    """(rc, IndelReadsOut) of the host-compiled kernel body."""
    return _run(host_body().k6bcore_run, normal, tumor, loci, cap_reads, cap_alts, smem_sort)


def same(a: B.IndelReadsOut, b: B.IndelReadsOut) -> None:
    """Every output array, byte for byte."""
    for x, y, name in zip(a.trimmed(), b.trimmed(), ("alt_off", "alts", "read_off", "reads", "status", "totals")):
        assert x.tobytes() == y.tobytes(), name


# ------------------------------------------------------------------------------------------------------------------
# synthetic records
# ------------------------------------------------------------------------------------------------------------------
def _synthetic_sample(rng, n_gid, n_regions, depth, max_width, special, permute_ids, tier2_frac, sub_frac):
    """One sample: regions whose windows are thinned id ranges (overlapping regions index a shared id differently), reads with 0..4 records
    on distinct window entries and 0..2 alternates each.  special = [(first id, width, reads)]: regions added as given (a narrow one with
    many reads makes a deep locus, a wide one a locus with many alternates)."""
    width = rng.integers(1, max_width + 1, n_regions)
    start = rng.integers(0, max(1, n_gid - max_width), n_regions)
    n_reads_of = rng.poisson(depth, n_regions)
    for s0, w, nr in special:
        start, width, n_reads_of = np.append(start, s0), np.append(width, w), np.append(n_reads_of, nr)
    n_regions = start.size
    ids = np.concatenate([np.arange(s, s + w) for s, w in zip(start, width)]).astype(np.uint32)
    first = np.concatenate([[0], np.cumsum(width)[:-1]])
    keep = rng.random(ids.size) < 0.85
    keep[first] = True
    keep[np.repeat(np.arange(n_regions) >= n_regions - len(special), width)] = True
    key_gid = ids[keep]
    n_win = np.add.reduceat(keep.astype(np.int64), first)
    region_key_off = np.concatenate([[0], np.cumsum(n_win)]).astype(np.uint32)
    region_read_off = np.concatenate([[0], np.cumsum(n_reads_of)]).astype(np.uint32)
    n = int(region_read_off[-1])
    region = np.repeat(np.arange(n_regions), n_reads_of)
    w = n_win[region]
    rec_off = np.concatenate([[0], np.cumsum(w)]).astype(np.uint32)
    n_rec = np.minimum(rng.integers(0, 5, n), w)
    n_rec[rng.random(n) < 0.1] = 0
    slots = int(rec_off[-1])
    recs = np.zeros(slots + 1, A.READ_INDEL_SCORE_DT)
    recs["flags"] = A.SX_RIS_SCORED  # what a slot past n_rec says must not matter: it would be an entry of window index 0
    recs["ref_lnp"] = -1.0
    read_of = np.repeat(np.arange(n), n_rec)
    j = np.arange(read_of.size) - np.repeat(np.cumsum(n_rec) - n_rec, n_rec)
    at = rec_off[read_of].astype(np.int64) + j
    wr = w[read_of]
    key = (np.repeat(rng.integers(0, 1 << 30, n), n_rec) + j) % wr
    m = read_of.size
    n_alt = np.minimum(rng.integers(0, 3, m), wr - 1)
    d0 = 1 + rng.integers(0, 1 << 30, m) % np.maximum(wr - 1, 1)
    d1 = 1 + (d0 - 1 + 1 + rng.integers(0, 1 << 30, m) % np.maximum(wr - 2, 1)) % np.maximum(wr - 1, 1)
    r = recs[at]
    r["key"], r["n_alt"] = key, n_alt
    r["flags"] = np.where(rng.random(m) < sub_frac, A.SX_RIS_SUBOVERLAP, A.SX_RIS_SCORED)
    r["read_pos"], r["dist_from_edge"] = rng.integers(0, 150, m), rng.integers(0, 75, m)
    r["ref_lnp"], r["indel_lnp"] = -rng.uniform(0, 25, m), -rng.uniform(0, 25, m)
    r["alt_key"][:, 0] = np.where(n_alt > 0, (key + d0) % wr, 0)
    r["alt_key"][:, 1] = np.where(n_alt > 1, (key + d1) % wr, 0)
    r["alt_lnp"][:, 0] = np.where(n_alt > 0, -rng.uniform(0, 25, m), 0)
    r["alt_lnp"][:, 1] = np.where(n_alt > 1, -rng.uniform(0, 25, m), 0)
    recs[at] = r
    sub_only = rng.random(n) < 0.05  # reads that only mark suboverlap
    recs["flags"][at[sub_only[read_of]]] = A.SX_RIS_SUBOVERLAP
    read_len = rng.integers(30, 151, n + 1).astype(np.uint16)
    sb = SimpleNamespace(n_regions=n_regions, n_reads=n, n_keys=int(key_gid.size), region_read_off=region_read_off, region_key_off=region_key_off, rec_off=rec_off,
                         read_len=read_len, non_ambig=(read_len - rng.integers(0, 3, n + 1)).astype(np.uint16),
                         read_flags=(A.SX_SIF_FWD * rng.integers(0, 2, n + 1) + A.SX_SIF_TIER1 * (rng.random(n + 1) >= tier2_frac)).astype(np.uint8))
    read_id = (1000 + rng.permutation(n + 1)).astype(np.uint32) if permute_ids else None
    return B.IndelReadsSample(sb, recs, np.append(n_rec, 0).astype(np.uint32), key_gid, read_id)


def entries_of(s: B.IndelReadsSample):
    """(id, read index) of every SX_RIS_SCORED record in use, in read order."""
    n_rec = s.n_rec[: s.n_reads].astype(np.int64)
    read_of = np.repeat(np.arange(s.n_reads), n_rec)
    at = s.rec_off[read_of].astype(np.int64) + np.arange(read_of.size) - np.repeat(np.cumsum(n_rec) - n_rec, n_rec)
    region = np.repeat(np.arange(s.n_regions), np.diff(s.region_read_off.astype(np.int64)))
    scored = (s.recs["flags"][at] & A.SX_RIS_SCORED) != 0
    gid = s.key_gid[s.region_key_off[region[read_of]].astype(np.int64) + s.recs["key"][at]]
    return gid[scored], read_of[scored]


def synthetic_case(seed: int, n_gid: int = 300, n_regions: int = 60, depth: float = 8.0, max_width: int = 7, special=(), permute_ids: bool = True,
                   tier2_frac: float = 0.2, sub_frac: float = 0.15, locus_frac: float = 0.6, dup: bool = False):
    """(normal, tumor, loci).  The last 4 ids are in no window: those among the loci are candidates without a read (forced output)."""
    rng = np.random.default_rng(9000 + seed)
    in_windows = n_gid - 4
    normal = _synthetic_sample(rng, in_windows, n_regions, depth, max_width, special, permute_ids, tier2_frac, sub_frac)
    tumor = _synthetic_sample(rng, in_windows, n_regions + 3, depth * 1.5, max_width, special, permute_ids, tier2_frac, sub_frac)
    gid_key = np.zeros(n_gid, A.INDEL_KEY_DT)
    gid_key["pos"] = 1000 + np.arange(n_gid) // 3  # three ids a position ...
    gid_key["del_len"] = rng.integers(0, 4, n_gid)
    gid_key["ins_len"] = 2  # ... of equal insert length: what keeps them apart is the insert sequence (ins_id) and the delete length
    gid_key["ins_id"] = 1 + np.arange(n_gid) % 3
    gid_key["ref_to_indel_lnp"], gid_key["indel_to_ref_lnp"] = -rng.uniform(8, 12, n_gid), -rng.uniform(8, 12, n_gid)
    chosen = rng.random(n_gid) < locus_frac
    chosen[-4:] = [True, False, True, True]
    for s0, w, _ in special:
        chosen[s0 : s0 + w] = True
    gid = np.nonzero(chosen)[0].astype(np.uint32)
    forced = (rng.random(gid.size) < 0.1).astype(np.uint8)
    forced[gid >= in_windows] = 1
    err_prob = np.array([1e-4, 5e-4, 2e-3, 8e-3, 0.03, 0.1])
    loci = B.IndelLoci(gid, gid_key[gid], forced, rng.integers(0, err_prob.size, gid.size), gid_key, err_prob)
    if dup:  # two reads of one tumor list under one id
        g, r = entries_of(tumor)
        listed = np.isin(g, gid)
        u, first, count = np.unique(g[listed], return_index=True, return_counts=True)
        twice = np.nonzero(count >= 2)[0][0]
        r1 = r[listed][first[twice]]
        r2 = r[listed][np.nonzero(g[listed] == u[twice])[0][1]]
        tumor.read_id[r2] = tumor.read_id[r1]
    return normal, tumor, loci


# seed, kwargs.  special regions: (first id, width, reads)
SYNTH_CASES = [
    (0, {}),
    (1, {"permute_ids": False, "depth": 3.0, "locus_frac": 0.3}),
    (2, {"special": [(40, 30, 400)]}),              # a wide window under many reads: loci with more than 16 alternates
    (3, {"special": [(100, 2, 2600)], "depth": 5.0}),  # a narrow one: loci deeper than the shared-memory sort
    (4, {"dup": True, "tier2_frac": 0.6}),
    (5, {"sub_frac": 0.9, "n_regions": 20}),
    (6, {"special": [(10, 3, 1500), (200, 24, 300)], "dup": True, "max_width": 12}),
]


def synth(i: int):
    seed, kw = SYNTH_CASES[i]
    return synthetic_case(seed, **kw)


# ------------------------------------------------------------------------------------------------------------------
# K6-scored records
# ------------------------------------------------------------------------------------------------------------------
def k6_case(seed: int, n_regions: int = 16):
    """Two K6 batches over shared windows, with the scores K1 would give: (batches, lnps, key_gid, read_id, loci), each of the first four a
    [normal, tumor] pair.  The generator's regions are moved 10 kb apart, so that one IndelBuffer can hold all of them; each region's reads
    are dealt to the samples, and within a sample to two regions: one on the generator's window, one on the same window behind one more
    leading entry -- so one IndelKey is reached under different window indices from several regions of both samples.  Ids are the rank in
    IndelKey order, as the IndelBuffer's iteration index would be.  The normal sample is scored at the somatic caller's normal flank."""
    rng = np.random.default_rng(9500 + seed)
    regions, lnp = specgen.random_score_indels_regions(rng, n_regions, reads_per_region=(4, 14))
    parts = ([], []), ([], [])  # per sample: regions, lnp
    a = 0
    for g, (win, reads) in enumerate(regions):
        shift = 10000 * (g + 1) - min(k.pos for k in win)
        for k in win:
            k.pos += shift
        wide = [B.WindowKeySpec(min(k.pos for k in win) - 400, del_len=1)] + list(win)
        split = [[[], []], [[], []]]  # [sample][window kind] -> (read, lnp)
        for r in reads:
            r.alns = [(p + shift, path, kidx) for p, path, kidx in r.alns]
            split[int(rng.random() < 0.6)][int(rng.random() < 0.4)].append((r, lnp[a : a + len(r.alns)]))
            a += len(r.alns)
        for s in range(2):
            moved = [B.ScoredReadSpec(r.length, [(p, path, [i + 1 for i in kidx]) for p, path, kidx in r.alns], r.fwd, r.tier1, r.non_ambig, r.incomplete)
                     for r, _ in split[s][1]]
            parts[s][0].extend([(win, [r for r, _ in split[s][0]]), (wide, moved)])
            parts[s][1].extend(x for kind in range(2) for _, l in split[s][kind] for x in l)
    so = A.default_sindel_opts()
    batches = []
    for s in range(2):
        o = A.default_score_indels_opts()
        o.min_read_bp_flank = so.min_read_bp_flank[s]
        batches.append(B.ScoreIndelsBatch(parts[s][0], o))
    lnps = [np.array(parts[s][1] + [0.0]) for s in range(2)]
    specs = {k.order(): k for s in range(2) for w, _ in parts[s][0] for k in w}
    order = sorted(specs)
    rank = {o: i for i, o in enumerate(order)}
    key_gid = [np.array([rank[k.order()] for w, _ in parts[s][0] for k in w], np.uint32) for s in range(2)]
    gid_key = np.zeros(len(order), A.INDEL_KEY_DT)
    for i, o in enumerate(order):
        k = specs[o]
        gid_key[i]["pos"], gid_key[i]["del_len"], gid_key[i]["ins_len"], gid_key[i]["ins_id"] = k.pos, k.del_len, len(k.ins), i + 1 if k.ins else 0
        gid_key[i]["type"] = A.SX_INDEL_TYPE_MISMATCH if k.mismatch else A.SX_INDEL_TYPE_INDEL
    gid = np.nonzero(gid_key["type"] == A.SX_INDEL_TYPE_INDEL)[0].astype(np.uint32)
    err_prob = np.array([1e-4, 5e-4, 2e-3, 8e-3, 0.03, 0.1])
    loci = B.IndelLoci(gid, gid_key[gid], (rng.random(gid.size) < 0.3).astype(np.uint8), rng.integers(0, err_prob.size, gid.size), gid_key, err_prob)
    loci.ins = [specs[o].ins for o in order]  # test-only: the insert sequences behind the ids (the reference harness rebuilds IndelKeys)
    read_id = [(5 + rng.permutation(b.n_reads + 1)).astype(np.uint32) for b in batches]
    return batches, lnps, key_gid, read_id, loci


def ox_k6_sample(sb: B.ScoreIndelsBatch, lnp, key_gid, read_id) -> B.IndelReadsSample:
    """The K6 oracle's records of one sample, in their slots, as the link's input."""
    out = B.ScoreIndelsOut(sb)
    lib = reflib.oracle()
    lib.ox_score_indels.argtypes = [C.POINTER(A.SxScoreIndelsBatch)] + [C.c_void_p] * 5
    rc = lib.ox_score_indels(C.byref(sb.c), A.ptr(lnp), A.ptr(out.recs), A.ptr(out.n_rec), A.ptr(out.max_aln), A.ptr(out.eval_aln))
    assert rc == 0, rc
    return B.IndelReadsSample(sb, out.recs, out.n_rec, key_gid, read_id)


K6_CASES = 8
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libstrelka_ref_indel_reads.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "indel_reads_ref.npz")


def have_ref() -> bool:
    return os.path.exists(REF_SO)


class _RefSample(C.Structure):
    _fields_ = [("b", C.POINTER(A.SxScoreIndelsBatch))] + [(n, C.c_void_p) for n in ("lnp", "ins_pool", "ins_off", "read_id")]


class _RefMaps(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("read_off", "reads", "entry_id", "alt_off", "alt_gid")] + [("cap_reads", C.c_uint32), ("cap_alts", C.c_uint32)]


def ref_chain(batches, lnps, read_id, loci, opts):
    """The reference's own score_indels for both samples into ONE IndelBuffer, then its get_somatic_indel on that buffer's IndelData
    (oracle/ref_harness_indel_reads.cpp).  Returns (results, maps): maps = the buffer's read_path_lnp maps of the loci, flattened in
    iteration order, as {read_off, reads, entry_id, alt_off, alt_gid}.  It is given IndelKeys only, no window index -> id table."""
    if "ref" not in _libs:
        _libs["ref"] = C.CDLL(REF_SO)
    samples = (_RefSample * 2)(*(_RefSample(C.pointer(b.c), A.ptr(l), A.ptr(b.ins_pool), A.ptr(b.ins_off), A.ptr(i)) for b, l, i in zip(batches, lnps, read_id)))
    pool = np.frombuffer("".join(loci.ins).encode() + b"\0", np.uint8).copy()
    off = np.concatenate([[0], np.cumsum([len(x) for x in loci.ins])]).astype(np.uint32)
    n, cap = loci.n_loci, sum(b.n_rec_slots for b in batches) + 1
    m = dict(read_off=np.zeros(2 * n + 1, np.uint32), reads=np.zeros(cap, A.SINDEL_READ_DT), entry_id=np.zeros(cap, np.uint32), alt_off=np.zeros(n + 1, np.uint32),
             alt_gid=np.zeros(2 * cap, np.uint32))
    maps = _RefMaps(*(A.ptr(m[k]) for k in ("read_off", "reads", "entry_id", "alt_off", "alt_gid")), cap, 2 * cap)
    out = np.zeros(max(1, n), A.SINDEL_RESULT_DT)
    err = C.create_string_buffer(1024)
    fn = _libs["ref"].ref_indel_reads_chain
    fn.argtypes = [C.POINTER(A.SxSindelOpts), C.POINTER(_RefSample), C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.POINTER(A.SxIndelLoci), C.c_void_p, C.c_uint32,
                   C.c_void_p, C.POINTER(_RefMaps), C.c_char_p, C.c_int]
    rc = fn(C.byref(opts), samples, A.ptr(loci.gid_key), A.ptr(pool), A.ptr(off), loci.n_gid, C.byref(loci.c), A.ptr(loci.err_prob), loci.err_prob.size, A.ptr(out),
            C.byref(maps), err, 1024)
    assert rc == 0, err.value.decode()
    ne, na = int(m["read_off"][-1]), int(m["alt_off"][-1])
    m["reads"], m["entry_id"], m["alt_gid"] = m["reads"][:ne], m["entry_id"][:ne], m["alt_gid"][:na]
    return out[:n], m


def inputs_digest(batches, lnps, key_gid, read_id, loci) -> str:
    import hashlib

    h = hashlib.sha256()
    for s in range(2):
        b = batches[s]
        for a in (b.region_read_off, b.region_key_off, b.keys, b.aln_off, b.aln_pos, b.aln_seg_off, b.segs, b.aln_key_off, b.aln_keys, b.read_len, b.non_ambig,
                  b.read_flags, b.rec_off, lnps[s], key_gid[s], read_id[s]):
            h.update(np.ascontiguousarray(a).tobytes())
    for a in (loci.gid, loci.is_forced_output, loci.err_idx, loci.gid_key, loci.err_prob):
        h.update(np.ascontiguousarray(a).tobytes())
    h.update("|".join(loci.ins).encode())
    return h.hexdigest()


def frozen_ref_chain(seed: int, digest: str):
    """What ref_chain returned for case `seed` when tests/golden/make_indel_reads_golden.py froze it."""
    g = np.load(GOLDEN)
    assert str(g[f"inputs{seed}"]) == digest, "the generator no longer makes the inputs the answers were frozen for"
    m = {k: g[f"{k}{seed}"] for k in ("read_off", "entry_id", "alt_off", "alt_gid")}
    m["reads"] = np.frombuffer(g[f"reads{seed}"].tobytes(), A.SINDEL_READ_DT)
    return np.frombuffer(g[f"ref{seed}"].tobytes(), A.SINDEL_RESULT_DT), m


def same_as_maps(linked: B.IndelReadsOut, maps: dict, loci) -> None:
    """The link's output against the reference buffer's flattened read_path_lnp maps: offsets, every entry byte, every table row."""
    assert not linked.status[: loci.n_loci].any()
    alt_off, alts, read_off, reads, _, _ = linked.trimmed()
    assert np.array_equal(read_off, maps["read_off"]) and np.array_equal(alt_off, maps["alt_off"])
    assert reads.tobytes() == maps["reads"].tobytes()
    assert alts.tobytes() == loci.gid_key[maps["alt_gid"]].tobytes()
    seg = np.repeat(np.arange(2 * loci.n_loci), np.diff(read_off).astype(np.int64))
    ids = maps["entry_id"].astype(np.int64)
    assert np.all((np.diff(ids) > 0) | (np.diff(seg) > 0))  # ascending read id inside every list
