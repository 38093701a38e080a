"""K6b indel_reads (include/strelka_b200.h): K6's per-read records regrouped into K5b's per-locus read lists.

CPU: three statements of the link -- the oracle on std::map containers (oracle/indel_reads_oracle.cpp), the numpy/dict host builder
(batch.link_indel_reads) and the kernels' own body compiled with g++ (tests/cpp/k6b_core_host.cpp) -- agree byte for byte on every
case; the cases are asserted to hold every shape the link must handle; and the chain K6 oracle -> link -> K5b oracle is compared with
the reference's own score_indels (both samples into ONE IndelBuffer) + get_somatic_indel on that buffer's IndelData
(oracle/ref_harness_indel_reads.cpp): live where oracle/_ref is built, and through tests/golden/indel_reads_ref.npz everywhere."""
import ctypes as C

import numpy as np
import pytest

import indel_reads_gen as G
import sindel_gen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B


@pytest.fixture(scope="module")
def cases():
    return [G.synth(i) for i in range(len(G.SYNTH_CASES))]


@pytest.fixture(scope="module")
def oracle_out(cases):
    out = []
    for normal, tumor, loci in cases:
        rc, o = G.ox_link(normal, tumor, loci)
        assert rc == 0, rc
        out.append(o)
    return out


def test_layouts():
    import os
    import re

    assert C.sizeof(A.SxIndelReadsSample) == 96 and C.sizeof(A.SxIndelLoci) == 48 and C.sizeof(A.SxIndelReadsOut) == 56
    hdr = open(os.path.join(G.ROOT, "include", "strelka_b200.h")).read()
    for name, cls in (("sx_indel_reads_sample", A.SxIndelReadsSample), ("sx_indel_loci", A.SxIndelLoci), ("sx_indel_reads_out", A.SxIndelReadsOut)):
        body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), hdr, re.S).group(1)
        body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
        fields = [f for decl in body.split(";") for f in re.findall(r"(\w+)\s*(?:,|$)", decl.strip())]
        assert fields == [f[0] for f in cls._fields_], name
    assert re.search(r"#define SX_INDEL_READS_ST_DUP_READ (0x[0-9a-f]+)u", hdr).group(1) == hex(A.SX_INDEL_READS_ST_DUP_READ)
    assert A.SX_INDEL_READS_ST_DUP_READ & A.SX_SINDEL_ST_CAP == 0


@pytest.mark.parametrize("i", range(len(G.SYNTH_CASES)))
def test_oracle_host_builder_and_kernel_body_agree(cases, oracle_out, i):
    normal, tumor, loci = cases[i]
    G.same(oracle_out[i], B.link_indel_reads(normal, tumor, loci))
    rc, core = G.core_link(normal, tumor, loci)
    assert rc == 0
    G.same(oracle_out[i], core)
    # the sort is the same network whichever memory it runs in: everything on the deep path, and everything on the shallow one
    for smem_sort in (0, 1 << 20):
        rc, core = G.core_link(normal, tumor, loci, smem_sort=smem_sort)
        assert rc == 0
        G.same(oracle_out[i], core)


def test_output_is_a_somatic_indel_batch(cases, oracle_out):
    """Lists in ascending read id, tables of distinct ascending ids, alternates inside their table: what K5b reads."""
    for (normal, tumor, loci), o in zip(cases, oracle_out):
        sb = o.batch(loci)
        assert sb.n_loci == loci.n_loci
        n_alts = np.diff(sb.alt_off).astype(np.int64)
        assert n_alts.max() <= A.SX_SINDEL_MAX_ALTS
        rl = np.repeat(np.arange(2 * sb.n_loci), np.diff(sb.read_off).astype(np.int64)) // 2
        for k in range(2):
            named = sb.reads["n_alt"] > k
            assert np.all(sb.reads["alt"][named, k] < n_alts[rl[named]])
        flagged = o.status[: loci.n_loci] != 0
        assert np.all(n_alts[flagged] == 0) and np.all(np.diff(sb.read_off).reshape(-1, 2)[flagged] == 0)


def test_cases_reach_every_branch(cases, oracle_out):
    hit = set()
    for (normal, tumor, loci), o in zip(cases, oracle_out):
        st = o.status[: loci.n_loci]
        depth = np.diff(o.read_off).reshape(-1, 2).astype(np.int64)
        if np.any(st & A.SX_SINDEL_ST_CAP):
            hit.add("more than 16 alternates")
        if np.any(st & A.SX_INDEL_READS_ST_DUP_READ):
            hit.add("duplicate read id")
        if depth.max() > G.SMEM_SORT:
            hit.add("deeper than the shared-memory sort")
        if np.any((loci.is_forced_output == 1) & (depth.sum(axis=1) == 0) & (st == 0)):
            hit.add("forced output without reads")
        per = [G.entries_of(s) for s in (normal, tumor)]
        for s, (g, r) in zip((normal, tumor), per):
            if s.read_id is not None and np.any(np.diff(s.read_id[: s.n_reads].astype(np.int64)) < 0):
                hit.add("read ids permuted against read order")
            region = np.repeat(np.arange(s.n_regions), np.diff(s.region_read_off.astype(np.int64)))
            listed = np.isin(g, loci.gid)
            # one id reached from regions whose windows hold it at different indices
            idx = {}
            for reg in range(s.n_regions):
                k0, k1 = int(s.region_key_off[reg]), int(s.region_key_off[reg + 1])
                for j, gid in enumerate(s.key_gid[k0:k1]):
                    idx.setdefault(int(gid), set()).add(j)
            multi = {gid for gid, js in idx.items() if len(js) > 1}
            if any(len(set(region[r[listed & (g == gid)]])) > 1 for gid in list(multi)[:50]):
                hit.add("a locus fed from regions that index it differently")
            used = np.zeros(s.n_reads, bool)
            used[r] = True
            if np.any((s.n_rec[: s.n_reads] > 0) & ~used):
                hit.add("suboverlap-only reads")
            if np.any(~listed):
                hit.add("records of unlisted indels")
        if np.any(o.reads["is_tier1"][: int(o.totals[0])] == 0) and np.any(o.reads["is_tier1"][: int(o.totals[0])] == 1):
            hit.add("tier1/tier2 mix")
        # alternates named by one sample only and by both
        sb = o.batch(loci)
        rl = np.repeat(np.arange(2 * sb.n_loci), np.diff(sb.read_off).astype(np.int64))
        for l in np.nonzero(np.diff(sb.alt_off) > 0)[0][:300]:
            seen = [set(), set()]
            for s in range(2):
                rr = sb.reads[rl == 2 * l + s]
                for k in range(2):
                    seen[s] |= set(rr["alt"][rr["n_alt"] > k, k].tolist())
            if seen[0] & seen[1]:
                hit.add("alternate named by both samples")
            if seen[0] ^ seen[1]:
                hit.add("alternate named by one sample")
        a = sb.alts
        if a.size:
            t = np.stack([a["pos"], a["del_len"], a["ins_len"]], axis=1)
            loc = np.repeat(np.arange(sb.n_loci), np.diff(sb.alt_off).astype(np.int64))
            full = np.concatenate([loc[:, None], t], axis=1)
            if np.unique(full, axis=0).shape[0] < full.shape[0]:
                hit.add("alternates apart by insert sequence only")
        for k in range(3):
            if np.any(sb.reads["n_alt"] == k):
                hit.add(f"{k} alternates in a read")
    want = {"more than 16 alternates", "duplicate read id", "deeper than the shared-memory sort", "forced output without reads", "read ids permuted against read order",
            "a locus fed from regions that index it differently", "suboverlap-only reads", "records of unlisted indels", "tier1/tier2 mix",
            "alternate named by both samples", "alternate named by one sample", "alternates apart by insert sequence only", "0 alternates in a read",
            "1 alternates in a read", "2 alternates in a read"}
    assert want <= hit, want - hit


def test_capacity_and_bad_ids(cases, oracle_out):
    normal, tumor, loci = cases[0]
    need = oracle_out[0].totals
    for fn in (G.ox_link, G.core_link):
        for cr, ca in ((int(need[0]) - 1, None), (None, int(need[1]) - 1)):
            rc, o = fn(normal, tumor, loci, cap_reads=cr, cap_alts=ca)
            assert rc == A.SX_ERR_CAPACITY and np.array_equal(o.totals, need)
            assert o.read_off.tobytes() == oracle_out[0].read_off.tobytes() and o.status.tobytes() == oracle_out[0].status.tobytes()
            assert not o.reads.view(np.uint8).any() and not o.alts.view(np.uint8).any()  # nothing truncated: nothing written
        rc, o = fn(normal, tumor, loci, cap_reads=int(need[0]), cap_alts=int(need[1]))
        assert rc == 0
        G.same(o, oracle_out[0])
    used = int(G.entries_of(normal)[0][0])  # an id a scored record names: every window entry holding it goes out of range
    bad = B.IndelReadsSample(normal, normal.recs, normal.n_rec, np.where(normal.key_gid == used, loci.n_gid, normal.key_gid), normal.read_id)
    assert G.ox_link(bad, tumor, loci)[0] == A.SX_ERR_ARG and G.core_link(bad, tumor, loci)[0] == A.SX_ERR_ARG


def test_empty_inputs():
    normal, tumor, loci = G.synthetic_case(50, n_regions=1, depth=0.0)
    assert normal.n_reads == 0 and tumor.n_reads == 0
    rc, o = G.ox_link(normal, tumor, loci)
    assert rc == 0
    G.same(o, B.link_indel_reads(normal, tumor, loci))
    rc, c = G.core_link(normal, tumor, loci)
    assert rc == 0
    G.same(o, c)
    none = B.IndelLoci(loci.gid[:0], loci.key[:0], loci.is_forced_output[:0], loci.err_idx[:0], loci.gid_key, loci.err_prob)
    for fn in (G.ox_link, G.core_link):
        rc, o = fn(normal, tumor, none)
        assert rc == 0 and not o.totals.any() and not o.read_off.any() and not o.alt_off.any()


# ------------------------------------------------------------------------------------------------------------------
# the chain: K6 -> K6b -> K5b, against the reference's score_indels + get_somatic_indel on ONE IndelBuffer
# ------------------------------------------------------------------------------------------------------------------
def ox_chain(seed):
    case = G.k6_case(seed)
    batches, lnps, key_gid, read_id, loci = case
    normal, tumor = (G.ox_k6_sample(batches[s], lnps[s], key_gid[s], read_id[s]) for s in range(2))
    rc, linked = G.ox_link(normal, tumor, loci)
    assert rc == 0
    return case, normal, tumor, linked


def _against(case, normal, tumor, linked, ref, maps):
    loci = case[4]
    G.same_as_maps(linked, maps, loci)
    sb = linked.batch(loci)
    o = A.default_sindel_opts()
    out = sindel_gen.ox_somatic_indel(o, sb)
    assert np.all(out["status"] == 0)
    sindel_gen.compare_to_reference(out, ref, sb, o)


@pytest.mark.parametrize("seed", range(G.K6_CASES))
def test_chain_matches_frozen_reference(seed):
    """K6 oracle -> link oracle -> K5b oracle against the frozen answers of the reference's score_indels (both samples, one IndelBuffer)
    + get_somatic_indel: the link's lists are that buffer's read_path_lnp maps byte for byte, and the calls are the reference's.  The
    three statements of the link agree on these records too."""
    case, normal, tumor, linked = ox_chain(seed)
    loci = case[4]
    G.same(linked, B.link_indel_reads(normal, tumor, loci))
    rc, core = G.core_link(normal, tumor, loci)
    assert rc == 0
    G.same(linked, core)
    ref, maps = G.frozen_ref_chain(seed, G.inputs_digest(*case))
    _against(case, normal, tumor, linked, ref, maps)


@pytest.mark.skipif(not G.have_ref(), reason="oracle/_ref/libstrelka_ref_indel_reads.so not built (no reference tree)")
@pytest.mark.parametrize("seed", range(G.K6_CASES))
def test_chain_matches_reference(seed):
    case, normal, tumor, linked = ox_chain(seed)
    batches, lnps, _, read_id, loci = case
    ref, maps = G.ref_chain(batches, lnps, read_id, loci, A.default_sindel_opts())
    _against(case, normal, tumor, linked, ref, maps)
    fref, fmaps = G.frozen_ref_chain(seed, G.inputs_digest(*case))
    assert fref.tobytes() == ref.tobytes() and all(fmaps[k].tobytes() == maps[k].tobytes() for k in maps), "frozen answers differ from the live reference"


def test_chain_cases_exercise_the_seam():
    """What a wrong link would get wrong is present in the K6 cases: loci fed by both samples and by regions that index them differently,
    alternates, read ids against read order, tier2 reads."""
    hit = set()
    for seed in range(G.K6_CASES):
        case, normal, tumor, linked = ox_chain(seed)
        loci = case[4]
        depth = np.diff(linked.read_off).reshape(-1, 2)
        if np.any((depth[:, 0] > 0) & (depth[:, 1] > 0)):
            hit.add("both samples")
        if int(linked.totals[1]) > 0:
            hit.add("alternates")
        if np.any(linked.reads["n_alt"][: int(linked.totals[0])] == 2):
            hit.add("two alternates in a read")
        if np.any(linked.reads["is_tier1"][: int(linked.totals[0])] == 0):
            hit.add("tier2")
        for s in (normal, tumor):
            g, r = G.entries_of(s)
            region = np.repeat(np.arange(s.n_regions), np.diff(s.region_read_off.astype(np.int64)))
            for gid in np.unique(g[np.isin(g, loci.gid)]):
                if len(set(region[r[g == gid]])) > 1:
                    hit.add("a locus fed from regions that index it differently")
            if np.any(np.diff(s.read_id[: s.n_reads].astype(np.int64)) < 0):
                hit.add("read ids against read order")
    assert hit == {"both samples", "alternates", "two alternates in a read", "tier2", "a locus fed from regions that index it differently", "read ids against read order"}, hit
