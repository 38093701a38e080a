"""K6g allele_groups (include/strelka_b200.h): one sample's K6 records regrouped into K5's per-group supporting-read lists.

CPU: three statements of the link -- the oracle on std::map containers in the reference's own steps (oracle/allele_groups_oracle.cpp), the
dict host builder (batch.link_allele_groups) and the kernels' own body compiled with g++ (tests/cpp/k6g_core_host.cpp) -- agree byte for byte
on every case; the cases are asserted to reach every branch of the link; the structs' ctypes layout is the C compiler's; and the chain K6
oracle -> link -> K5 oracle is compared with the reference's own score_indels into ONE IndelBuffer followed by its allele-group functions and
getVariantAlleleGroupGenotypeLhoodsForSample (oracle/ref_harness_germline_indel.cpp): live where oracle/_ref is built, and through
tests/golden/germline_indel_ref.npz everywhere."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import allele_groups_gen as AG
import indel_reads_gen as G
import reflib
from strelka_b200 import _abi as A
from strelka_b200 import batch as B


@pytest.fixture(scope="module")
def cases():
    return [AG.case(i) for i in range(len(AG.CASES))]


@pytest.fixture(scope="module")
def oracle_out(cases):
    out = []
    for sample, groups in cases:
        rc, o = AG.ox_link(sample, groups)
        assert rc == 0, rc
        out.append(o)
    return out


STRUCTS = [("sx_allele_groups", A.SxAlleleGroups), ("sx_allele_group_reads_out", A.SxAlleleGroupReadsOut)]


def test_struct_layouts(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "strelka_b200.h"', "int main(void) {"]
    for name, cls in STRUCTS:
        lines.append(f'printf("%zu", sizeof({name}));')
        lines += [f'printf(" %zu", offsetof({name}, {f}));' for f, _ in cls._fields_]
        lines.append('printf("\\n");')
    lines += ['printf("%d\\n", SX_INDEL_MAX_ALLELES);', "return 0; }"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.check_call([cc, "-std=c99", "-I", os.path.join(AG.ROOT, "include"), str(tmp_path / "layout.c"), "-o", str(tmp_path / "layout")])
    got = subprocess.check_output([str(tmp_path / "layout")], text=True).split("\n")
    for (name, cls), line in zip(STRUCTS, got):
        assert [int(x) for x in line.split()] == [C.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_], name
    assert int(got[len(STRUCTS)]) == A.SX_INDEL_MAX_ALLELES
    # the output's first ten arrays are an sx_indel_batch's, in its order
    assert [f for f, _ in A.SxAlleleGroupReadsOut._fields_[:10]] == [f for f, _ in A.SxIndelBatch._fields_[1:]]


@pytest.mark.parametrize("i", range(len(AG.CASES)))
def test_oracle_host_builder_and_kernel_body_agree(cases, oracle_out, i):
    sample, groups = cases[i]
    AG.same(oracle_out[i], B.link_allele_groups(sample, groups))
    for smem_sort in (G.SMEM_SORT, 0, 1 << 20):  # the sort is the same network whichever memory it runs in
        rc, core = AG.core_link(sample, groups, smem_sort=smem_sort)
        assert rc == 0
        AG.same(oracle_out[i], core)


def maps_of(sample):
    """{id: {read id: (ref, indel, read index, record flags)}} of every record in use, suboverlap marks included."""
    m = {}
    region = np.repeat(np.arange(sample.n_regions), np.diff(sample.region_read_off[: sample.n_regions + 1]).astype(np.int64))
    for r in range(sample.n_reads):
        k0 = int(sample.region_key_off[region[r]]) if sample.n_rec[r] else 0
        rid = r if sample.read_id is None else int(sample.read_id[r])
        for rec in sample.recs[int(sample.rec_off[r]) : int(sample.rec_off[r]) + int(sample.n_rec[r])]:
            m.setdefault(int(sample.key_gid[k0 + int(rec["key"])]), {})[rid] = (np.float32(rec["ref_lnp"]), np.float32(rec["indel_lnp"]), r, int(rec["flags"]))
    return m


def test_cases_reach_every_branch(cases, oracle_out):
    hit = set()
    for (sample, groups), o in zip(cases, oracle_out):
        m = maps_of(sample)
        scored = {x: {rid: v for rid, v in d.items() if v[3] & A.SX_RIS_SCORED} for x, d in m.items()}
        tier1 = lambda v: sample.read_flags[v[2]] & A.SX_SIF_TIER1
        n_reads = np.diff(o.read_off.astype(np.int64))
        st = o.status[: groups.n_groups]
        seen = {}
        for g in range(groups.n_groups):
            al, co, pl = groups.group(g)
            for x in set(al + co):
                seen[x] = seen.get(x, 0) + 1
            if st[g]:
                hit.add("duplicate read id flagged")
                continue
            if n_reads[g] == 0:
                hit.add("group without a supporting read")
            else:
                hit.add(f"A={len(al)} ploidy={pl}")
            hit.add("no contrast" if not co else ("one contrast" if len(co) == 1 else "several contrasts"))
            s0 = scored.get(al[0], {})
            for rid, v in s0.items():
                inall = all(rid in scored.get(x, {}) for x in al[1:])
                if inall and not tier1(v):
                    hit.add("tier-2 read excluded")
                if tier1(v) and not inall:
                    hit.add("read missing from one allele excluded")
                if tier1(v) and inall:
                    l0 = max(scored[x][rid][0] for x in al)
                    for c in co:
                        e = scored.get(c, {}).get(rid)
                        hit.add("contrast entry present" if e is not None else "contrast entry absent")
                        if e is not None and e[1] > max(l0, e[0]):
                            hit.add("contrast value above ref")
            for x in al + co:
                if any(not v[3] & A.SX_RIS_SCORED for v in m.get(x, {}).values()):
                    hit.add("suboverlap records on a named id")
        if any(k > 1 for k in seen.values()):
            hit.add("ids shared between groups")
        if max(len(scored.get(x, {})) for x in seen) > G.SMEM_SORT:
            hit.add("list deeper than the shared-memory sort")
    want = {f"A={a} ploidy={p}" for a in range(1, 5) for p in (1, 2)} | {
        "duplicate read id flagged", "group without a supporting read", "no contrast", "one contrast", "several contrasts", "tier-2 read excluded",
        "read missing from one allele excluded", "contrast entry present", "contrast entry absent", "contrast value above ref", "suboverlap records on a named id",
        "ids shared between groups", "list deeper than the shared-memory sort"}
    assert want <= hit, want - hit


def test_capacity_bad_groups_and_empty(cases, oracle_out):
    sample, groups = cases[0]
    need = oracle_out[0].totals
    for fn in (AG.ox_link, AG.core_link):
        for cr, cl in ((int(need[0]) - 1, None), (None, int(need[1]) - 1)):
            rc, o = fn(sample, groups, cap_reads=cr, cap_lnp=cl)
            assert rc == A.SX_ERR_CAPACITY and np.array_equal(o.totals, need)
            for k in ("read_off", "lnp_off", "allele_off", "status"):
                assert getattr(o, k).tobytes() == getattr(oracle_out[0], k).tobytes(), k
            assert not o.allele_lnp.any() and not o.read_length.any()  # nothing truncated: nothing written
        rc, o = fn(sample, groups, cap_reads=int(need[0]), cap_lnp=int(need[1]))
        assert rc == 0
        AG.same(o, oracle_out[0])
    for bad in bad_groups(groups):
        for fn in (AG.ox_link, AG.core_link):
            assert fn(sample, bad)[0] == A.SX_ERR_ARG
        with pytest.raises(ValueError):
            B.link_allele_groups(sample, bad)
    recs = sample.recs.copy()
    recs["key"] = 65535  # no window is that long
    outside = B.IndelReadsSample(sample, recs, sample.n_rec, sample.key_gid, sample.read_id)
    for fn in (AG.ox_link, AG.core_link):
        assert fn(outside, groups)[0] == A.SX_ERR_ARG
    with pytest.raises(ValueError):
        B.link_allele_groups(outside, groups)
    none = B.AlleleGroups.from_lists([], [], np.zeros(0, np.uint8), groups.gid_key)
    for fn in (AG.ox_link, AG.core_link):
        rc, o = fn(sample, none)
        assert rc == 0 and not o.totals.any() and not o.read_off.any()
    AG.same(AG.ox_link(sample, none)[1], B.link_allele_groups(sample, none))


def bad_groups(groups):
    """Groups the link refuses: 0 and 5 alleles, ploidy 0 and 3, an allele id and a contrast id at n_gid."""
    al = [groups.group(g)[0] for g in range(groups.n_groups)]
    co = [groups.group(g)[1] for g in range(groups.n_groups)]
    pl = groups.ploidy.copy()
    n = groups.n_gid
    out = []
    for edit in ("none", "five", "ploidy0", "ploidy3", "allele_id", "contrast_id"):
        a, c, p = [list(x) for x in al], [list(x) for x in co], pl.copy()
        if edit == "none":
            a[1] = []
        elif edit == "five":
            a[1] = [0, 1, 2, 3, 4]
        elif edit == "ploidy0":
            p[1] = 0
        elif edit == "ploidy3":
            p[1] = 3
        elif edit == "allele_id":
            a[1][0] = n
        else:
            c[1] = c[1] + [n]
        out.append(B.AlleleGroups.from_lists(a, c, p, groups.gid_key))
    return out


# ------------------------------------------------------------------------------------------------------------------
# the chain: K6 -> K6g -> K5 on one sample of the K6b reference cases
# ------------------------------------------------------------------------------------------------------------------
def k6_groups(loci, sample, seed):
    """Groups over a K6 case's candidate ids: singletons, and pairs of ids one read covers together with a third such id as contrast."""
    rng = np.random.default_rng(7700 + seed)
    gid = loci.gid.tolist()
    m = maps_of(sample)
    al = [[x] for x in gid]
    co = [[] for _ in gid]
    together = sorted({(a, b) for d in [m] for a in gid for b in gid if a < b and set(m.get(a, {})) & set(m.get(b, {}))})
    for a, b in together[:60]:
        al.append([b, a] if rng.random() < 0.5 else [a, b])
        others = [x for x in gid if x not in (a, b) and set(m.get(x, {})) & set(m.get(a, {}))]
        co.append(others[:2])
    return B.AlleleGroups.from_lists(al, co, rng.integers(1, 3, len(al)), loci.gid_key)


def k6_chain(seed, s):
    """(case, sample s's K6 oracle records as the link's input, its groups, the oracle link's output)"""
    case = G.k6_case(seed)
    batches, lnps, key_gid, read_id, loci = case
    sample = G.ox_k6_sample(batches[s], lnps[s], key_gid[s], read_id[s])
    groups = k6_groups(loci, sample, seed)
    rc, linked = AG.ox_link(sample, groups)
    assert rc == 0
    return case, sample, groups, linked


def supporting_ids(sample, groups):
    """per group the tier-1 read ids with a scored entry in every allele, ascending, from the sample's records directly"""
    m = maps_of(sample)
    out = []
    for g in range(groups.n_groups):
        al, _, _ = groups.group(g)
        sc = [{rid for rid, v in m.get(x, {}).items() if v[3] & A.SX_RIS_SCORED and sample.read_flags[v[2]] & A.SX_SIF_TIER1} for x in al]
        out.extend(sorted(set.intersection(*sc)))
    return np.array(out, np.uint32)


def _against_reference(case, s, sample, groups, linked, ref):
    batches = case[0]
    out = reflib.ox_indel_gl(AG.params_of(batches[s]), linked.batch())
    AG.same_as_reference(linked, groups, ref, out)
    assert ref["read_id"].tobytes() == supporting_ids(sample, groups).tobytes()


@pytest.mark.parametrize("seed", range(G.K6_CASES))
def test_chain_matches_frozen_reference(seed):
    """K6 oracle -> link -> K5 oracle on one sample of the K6 cases, against the frozen answers of the reference's own score_indels into ONE
    IndelBuffer followed by getAlleleGroupSupportingReadIds, getAlleleLogLhoodFromRead (the extended group, folded here as
    getVariantAlleleGroupGenotypeLhoodsForSample folds it) and getVariantAlleleGroupGenotypeLhoodsForSample: the supporting read ids, every
    allele likelihood, every exemplar field, every gt_lhood double and every support count.  The three link statements agree on these
    records too."""
    for s in range(2):
        case, sample, groups, linked = k6_chain(seed, s)
        AG.same(linked, B.link_allele_groups(sample, groups))
        rc, core = AG.core_link(sample, groups)
        assert rc == 0
        AG.same(linked, core)
        batches, lnps, _, read_id, loci = case
        ref = AG.frozen_ref_chain(f"{seed}_{s}", AG.inputs_digest(batches[s], lnps[s], read_id[s], loci, groups))
        _against_reference(case, s, sample, groups, linked, ref)


@pytest.mark.skipif(not AG.have_ref(), reason="oracle/_ref/libstrelka_ref_germline_indel.so not built (no reference tree)")
@pytest.mark.parametrize("seed", range(G.K6_CASES))
def test_chain_matches_reference(seed):
    for s in range(2):
        case, sample, groups, linked = k6_chain(seed, s)
        batches, lnps, _, read_id, loci = case
        ref = AG.ref_chain(batches[s], lnps[s], read_id[s], loci, groups)
        _against_reference(case, s, sample, groups, linked, ref)
        frozen = AG.frozen_ref_chain(f"{seed}_{s}", AG.inputs_digest(batches[s], lnps[s], read_id[s], loci, groups))
        assert all(frozen[k].tobytes() == ref[k].tobytes() for k in AG.REF_KEYS), "frozen answers differ from the live reference"


def test_chain_cases_have_support():
    """What the two untested behaviours of getAlleleLogLhoodFromRead need is in the reference cases: reads in one allele of a pair but not
    the other (not supporting), supporting reads without an entry in a contrast allele, and contrast values the fold moves into the
    reference allele."""
    hit = set()
    for seed in range(G.K6_CASES):
        for s in range(2):
            case, sample, groups, linked = k6_chain(seed, s)
            batches, lnps, _, read_id, loci = case
            ref = AG.frozen_ref_chain(f"{seed}_{s}", AG.inputs_digest(batches[s], lnps[s], read_id[s], loci, groups))
            n = np.diff(linked.read_off.astype(np.int64))
            A_ = np.diff(groups.allele_off.astype(np.int64))
            C_ = np.diff(groups.contrast_off.astype(np.int64))
            if np.any((A_ == 1) & (n > 0)):
                hit.add("singletons with reads")
            if np.any((A_ == 2) & (n > 0)):
                hit.add("pairs with reads")
            if np.any((C_ > 0) & (n > 0)):
                hit.add("contrasts with reads")
            m = maps_of(sample)
            for g in np.nonzero(A_ == 2)[0]:
                al = groups.group(int(g))[0]
                sc = [{rid for rid, v in m.get(x, {}).items() if v[3] & A.SX_RIS_SCORED} for x in al]
                if sc[0] ^ sc[1]:
                    hit.add("reads missing from one allele")
            for g in np.nonzero((C_ > 0) & (n > 0))[0]:
                w = 1 + int(A_[g]) + int(C_[g])
                for i in range(int(n[g])):
                    v = ref["ext_lnp"][int(ref["lnp_off"][g]) + i * w : int(ref["lnp_off"][g]) + (i + 1) * w]
                    rid = int(ref["read_id"][int(ref["read_off"][g]) + i])
                    for c, x in enumerate(groups.group(int(g))[1]):
                        if rid not in m.get(x, {}) or not m[x][rid][3] & A.SX_RIS_SCORED:
                            hit.add("contrast entry absent")
                        elif v[1 + int(A_[g]) + c] > v[0]:
                            hit.add("contrast value above ref")
                        else:
                            hit.add("contrast entry present")
    assert hit == {"singletons with reads", "pairs with reads", "contrasts with reads", "reads missing from one allele", "contrast entry absent",
                   "contrast value above ref", "contrast entry present"}, hit
