"""K2b's callable mode on the CPU: the oracle (oracle/somatic_callable_oracle.cpp), the kernel's non-somatic body compiled with g++
(tests/cpp/k2b_nonsomatic_host.cpp) and the reference's own position_somatic_snv_call(..., true, sgt) agree bit for bit on every field,
nonsomatic_qphred included, on the cases of tests/callable_gen.py; the host interval builder gives the reference's BED text; and the
cases reach every branch the mode adds."""
import numpy as np
import pytest

import callable_gen as G
import reflib
import site_params as SP
import specgen

KINDS = specgen.SOMATIC_EDGE_KINDS


@pytest.fixture(scope="module")
def runs():
    """per case: (params, normal, tumor, forced, oracle records, tier1 records)"""
    out = {}
    for name, p, n, t, forced in G.cases():
        out[name] = (p, n, t, forced, G.ox_callable(p, n, t, forced), G.tier1_records(p, n, t))
    return out


def test_frozen_inputs_are_the_generators():
    assert bytes(G.golden()["inputs"]).decode() == G.inputs_digest()


def test_host_body_equals_oracle(runs):
    for name, (p, n, t, forced, ox, t1) in runs.items():
        comp = ox["is_computed"] == 1
        got = G.host_nonsomatic(t1)
        assert np.array_equal(got[comp], ox["nonsomatic_qphred"][comp]), name
        assert np.all(ox["nonsomatic_qphred"][~comp] == 0), name


def test_oracle_equals_frozen_reference(runs):
    gold = G.golden()
    for name, (p, n, t, forced, ox, _) in runs.items():
        G.compare_fields(ox, gold[name + "__fields"], name)
        assert G.host_bed(ox) == bytes(gold[name + "__bed"]).decode(), name


@pytest.mark.ref
def test_oracle_equals_reference(runs):
    for name, (p, n, t, forced, ox, _) in runs.items():
        want, bed = G.reference_fields(p, n, t, forced)
        G.compare_fields(ox, want, name)
        assert G.host_bed(ox) == bed, name


def test_records_are_forced_records_plus_nqss(runs):
    """The oracle's records are the forced records plus NQSS by construction (oracle/somatic_callable_oracle.cpp: the mode and forcing open the
    same gates), so this only pins that construction.  What carries the claim is the comparison of every field with the reference's own
    position_somatic_snv_call(..., true, sgt): test_oracle_equals_reference, and the frozen answers in test_oracle_equals_frozen_reference."""
    for name, (p, n, t, forced, ox, _) in runs.items():
        f = reflib.ox_somatic(p, n, t, np.ones(n.n_sites, np.uint8))
        a = ox.copy()
        a["nonsomatic_qphred"] = 0
        assert a.tobytes() == f.tobytes(), name


def test_branches_reached(runs):
    _, kind = SP.k2b_edge_batch()[2:]
    hit = dict(nqss_only=0, qss_only=0, both=0, neither=0, allref_skipped=0, tier2_copy=0, kept=0, dropped_offdiag=0, dropped_opt=0, kept_far_diag=0, nan_tier=0, n_ref=0)
    for name, (p, n, t, forced, ox, t1) in runs.items():
        comp = ox["is_computed"] == 1
        q, nq = ox["qphred"] >= 15, ox["nonsomatic_qphred"] >= 15
        hit["nqss_only"] += int((comp & nq & ~q).sum())
        hit["qss_only"] += int((comp & q & ~nq).sum())
        hit["both"] += int((comp & q & nq).sum())
        hit["neither"] += int((comp & ~q & ~nq).sum())
        d = reflib.ox_somatic(p, n, t, forced)
        hit["allref_skipped"] += int((comp & (d["is_computed"] == 0) & (forced == 0) & (kind == KINDS.index("both_empty"))).sum())
        if n.t2_off is not None and t.t2_off is not None:
            hit["tier2_copy"] += int((comp & (t1["qphred"] == 0)).sum())
        o = G.host_outcomes(t1[comp])
        hit["kept"] += int(((o & 1) != 0).sum())
        hit["dropped_offdiag"] += int(((o & 2) != 0).sum())
        hit["dropped_opt"] += int(((o & 4) != 0).sum())
        hit["kept_far_diag"] += int(((o & 8) != 0).sum())
        hit["nan_tier"] += int((comp & SP.ntype_unset(p, n, t)).sum())
        hit["n_ref"] += int(((kind == KINDS.index("n_ref")) & ~comp).sum())
        assert np.all(ox[kind == KINDS.index("n_ref")].view(np.uint8) == 0), name
    assert all(v > 0 for v in hit.values()), hit


def test_host_builder_edges():
    from strelka_b200 import batch as B

    r = G.synthetic_records(np.random.default_rng(1), 0, 0.5)
    assert [x.size for x in B.somatic_callable_regions(r, 7)] == [0, 0]
    r = G.synthetic_records(np.random.default_rng(1), 10, 1.0)
    b, e = B.somatic_callable_regions(r, 7)
    assert b.tolist() == [7] and e.tolist() == [17]
    r["qphred"][1::2] = 0
    r["nonsomatic_qphred"][1::2] = 14
    b, e = B.somatic_callable_regions(r, 7)
    assert b.tolist() == [7, 9, 11, 13, 15] and e.tolist() == [8, 10, 12, 14, 16]
