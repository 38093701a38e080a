"""K5b somatic_indel (get_somatic_indel, applications/strelka/somatic_indel_grid.cpp:181-361).

CPU: the scalar oracle (oracle/somatic_indel_oracle.cpp) against the reference's own function, bit for bit on every defined field, through
the live harness where oracle/_ref is built and through the frozen answers of tests/golden/somatic_indel_ref.npz everywhere; the cases
are asserted to reach every branch the model has.
GPU: sx_somatic_indel and sx_somatic_indel_dev against the oracle, whole records byte for byte."""
import ctypes as C
import os

import numpy as np
import pytest

import sindel_gen as G
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "somatic_indel_ref.npz")


@pytest.fixture(scope="module")
def cases():
    return [G.case(i) for i in range(len(G.CASES))]


@pytest.fixture(scope="module")
def oracle_out(cases):
    return [G.ox_somatic_indel(o, sb) for sb, o in cases]


def test_layouts():
    assert A.SINDEL_READ_DT.itemsize == 24 and A.SINDEL_TIER_DT.itemsize == 188 and A.SINDEL_RESULT_DT.itemsize == 400
    assert C.sizeof(A.SxSindelOpts) == 64 and C.sizeof(A.SxSindelBatch) == 64
    o = A.default_sindel_opts()
    assert (o.somatic_indel_rate, o.bindel_diploid_theta, o.indel_contam_tolerance, o.shared_indel_error_factor) == (1e-6, 1e-4, 0.15, 1.65)
    assert (o.randomBaseMatchProb, o.tier2RandomBaseMatchProb, o.useTier2Evidence, list(o.min_read_bp_flank)) == (0.5, 0.25, 1, [1, 5])


@pytest.mark.parametrize("i", range(len(G.CASES)))
def test_oracle_matches_frozen_reference(cases, oracle_out, i):
    g = np.load(GOLDEN)
    sb, o = cases[i]
    assert str(g[f"inputs{i}"]) == G.inputs_digest(sb), "the generator no longer makes the inputs the answers were frozen for"
    ref = np.frombuffer(g[f"ref{i}"].tobytes(), A.SINDEL_RESULT_DT)
    G.compare_to_reference(oracle_out[i], ref, sb, o)


@pytest.mark.skipif(not G.have_ref(), reason="oracle/_ref/libstrelka_ref_sindel.so not built (no reference tree)")
@pytest.mark.parametrize("i", range(len(G.CASES)))
def test_oracle_matches_reference(cases, oracle_out, i):
    sb, o = cases[i]
    ref = G.ref_somatic_indel(o, sb)
    G.compare_to_reference(oracle_out[i], ref, sb, o)
    g = np.load(GOLDEN)
    assert np.frombuffer(g[f"ref{i}"].tobytes(), A.SINDEL_RESULT_DT).tobytes() == ref.tobytes(), "frozen answers differ from the live reference"


def test_alternate_tables_hold_distinct_keys(cases):
    """Each locus's table entries are distinct IndelKeys to the reference too (the harness spells equal insert lengths with equal
    sequences), so both sides key the same alternates apart."""
    for sb, _ in cases:
        n_alts = np.diff(sb.alt_off)
        loc = np.repeat(np.arange(sb.n_loci), n_alts)
        a = sb.alts
        assert np.all(a["ins_id"] == 0)
        t = np.stack([loc, a["pos"], a["del_len"], a["ins_len"], a["type"]], axis=1)
        assert np.unique(t, axis=0).shape[0] == t.shape[0]


def test_cases_reach_every_branch(cases, oracle_out):
    hit = set()
    for (sb, o), out in zip(cases, oracle_out):
        n = sb.n_loci
        depth = np.diff(sb.read_off).reshape(n, 2)
        if np.any(depth[:, 0] == 0):
            hit.add("normal depth 0")
        if np.any(depth[:, 1] == 0):
            hit.add("tumor depth 0")
        if np.any((depth[:, 0] == 0) & (depth[:, 1] == 0)):
            hit.add("both depths 0")
        r = sb.reads
        for k in range(3):
            if np.any(r["n_alt"] == k):
                hit.add(f"{k} alternates in a read")
        if np.any(r["is_tier1"] == 0) and np.any(r["is_tier1"] == 1):
            hit.add("tier1/tier2 mix")
        flank = o.min_read_bp_flank[1]
        if np.any(r["read_length"] + 1 < 2 * flank):
            hit.add("read below 2*flank")
        if np.any(r["read_length"] + 1 == 2 * flank):
            hit.add("read at 2*flank")
        locus = np.repeat(np.arange(2 * n), np.diff(sb.read_off)) // 2
        sample = np.repeat(np.arange(2 * n), np.diff(sb.read_off)) % 2
        for l in np.unique(locus[r["n_alt"] > 0])[:200]:
            m = locus == l
            seen = [set(), set()]
            for s in range(2):
                rr = r[m & (sample == s)]
                for j in range(2):
                    seen[s] |= set(rr["alt"][rr["n_alt"] > j, j].tolist())
            if seen[0] & seen[1]:
                hit.add("same alternate in both samples")
                break
        if np.any(sb.is_forced_output == 1):
            hit.add("forced output")
        if np.any((sb.is_forced_output == 1) & (out["tier"][:, 0]["multi_indel"] == 1)):
            hit.add("forced output through the multi-indel filter")
        hit.add("useTier2Evidence off" if o.useTier2Evidence == 0 else "useTier2Evidence on")
        if o.somatic_indel_rate != 1e-6:
            hit.add("non-default rates")
        t = out["tier"]
        if np.any(t["multi_indel"] == 1):
            hit.add("multi-indel filter")
        if np.any(t["is_overlap"] == 1):
            hit.add("overlap")
        if np.any(out["is_output"] & (out["qphred"] > 0)):
            hit.add("somatic call")
        if np.any((t[:, 0]["qphred"] == 0) & (t[:, 0]["multi_indel"] == 0) & (t[:, 0]["evaluated"] == 1) & (sb.is_forced_output == 0)):
            hit.add("tier1 qphred 0 skips tier2")
        if np.any(out["sindel_tier"] == 1):
            hit.add("tier2 chosen")
        if np.any(out["is_output"] & (out["ntype"] == 3)):
            hit.add("ntype conflict")
    want = {"normal depth 0", "tumor depth 0", "both depths 0", "0 alternates in a read", "1 alternates in a read", "2 alternates in a read",
            "tier1/tier2 mix", "read below 2*flank", "read at 2*flank", "same alternate in both samples", "forced output",
            "forced output through the multi-indel filter", "useTier2Evidence off", "useTier2Evidence on", "non-default rates", "multi-indel filter",
            "overlap", "somatic call", "tier1 qphred 0 skips tier2", "tier2 chosen", "ntype conflict"}
    assert want <= hit, want - hit


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("i", range(len(G.CASES)))
def test_device_matches_oracle(ctx, cases, oracle_out, i):
    from strelka_b200.api import DevSomaticIndelBatch

    sb, o = cases[i]
    got = ctx.somatic_indel(sb, o)
    assert got.tobytes() == oracle_out[i].tobytes()
    db = DevSomaticIndelBatch(ctx, sb)
    ctx.somatic_indel_dev(db, o)
    assert db.download().tobytes() == oracle_out[i].tobytes()


@pytest.mark.gpu
def test_device_large_batch(ctx):
    """More loci than the grid has warps (sm_count * 8 blocks of 4 warps), at user depths."""
    from strelka_b200.api import DevSomaticIndelBatch

    sb = G.random_somatic_indel_batch(np.random.default_rng(7), 120_000, normal_depth=20.0, tumor_depth=30.0)
    o = A.default_sindel_opts()
    want = G.ox_somatic_indel(o, sb)
    db = DevSomaticIndelBatch(ctx, sb)
    ctx.somatic_indel_dev(db, o)
    got = db.download()
    assert got.tobytes() == want.tobytes()
    assert int(got["is_output"].sum()) > 0


def _with(sb: B.SomaticIndelBatch, **over) -> B.SomaticIndelBatch:
    a = {n: getattr(sb, n).copy() for n in ("key", "is_forced_output", "err_idx", "err_prob", "alt_off", "alts", "read_off", "reads")}
    a.update(over)
    return B.SomaticIndelBatch(a["key"], a["is_forced_output"], a["err_idx"], a["err_prob"], a["alt_off"], a["alts"], a["read_off"], a["reads"])


@pytest.mark.gpu
def test_over_capacity_loci_are_flagged(ctx):
    sb = G.random_somatic_indel_batch(np.random.default_rng(11), 64, normal_depth=10.0, tumor_depth=10.0, max_alts=A.SX_SINDEL_MAX_ALTS + 4,
                                      zero_depth_frac=0.0)
    n_alts = np.diff(sb.alt_off).astype(np.int64)
    depth = np.diff(sb.read_off).reshape(-1, 2).sum(axis=1)
    within = np.nonzero((n_alts >= 3) & (n_alts <= A.SX_SINDEL_MAX_ALTS) & (depth > 0))[0]
    l3, lp = int(within[0]), int(within[1])  # loci whose tables fit: the cap comes from one read
    reads = sb.reads.copy()
    r3 = int(sb.read_off[2 * l3])
    reads["n_alt"][r3] = 3  # a read naming three alternates
    reads["alt"][r3] = (0, 1)
    rp = int(sb.read_off[2 * lp])
    reads["n_alt"][rp] = 1  # a read naming an alternate past its locus's table
    reads["alt"][rp, 0] = n_alts[lp]
    sb = _with(sb, reads=reads)
    o = A.default_sindel_opts()
    want = G.ox_somatic_indel(o, sb)
    got = ctx.somatic_indel(sb, o)
    assert got.tobytes() == want.tobytes()
    expect = n_alts > A.SX_SINDEL_MAX_ALTS
    assert expect.any()
    expect[[l3, lp]] = True
    assert np.array_equal(got["status"] == A.SX_SINDEL_ST_CAP, expect)
    assert np.all(got["status"][~expect] == 0)
    z = got[expect].copy()
    z["status"] = 0
    assert z.tobytes() == np.zeros(z.size, A.SINDEL_RESULT_DT).tobytes()  # no result beside the status


@pytest.mark.gpu
def test_bad_arguments_rejected(ctx):
    from strelka_b200.api import DevSomaticIndelBatch, SxError

    sb, o = G.case(0)
    lib = ctx.lib
    out = np.zeros(sb.n_loci, A.SINDEL_RESULT_DT)
    assert lib.sx_somatic_indel(ctx.h, None, C.byref(sb.c), A.ptr(sb.err_prob), sb.err_prob.size, out.ctypes.data) == A.SX_ERR_ARG
    assert lib.sx_somatic_indel(ctx.h, C.byref(o), None, A.ptr(sb.err_prob), sb.err_prob.size, out.ctypes.data) == A.SX_ERR_ARG
    assert lib.sx_somatic_indel(ctx.h, C.byref(o), C.byref(sb.c), None, 0, out.ctypes.data) == A.SX_ERR_ARG
    assert lib.sx_somatic_indel(ctx.h, C.byref(o), C.byref(sb.c), A.ptr(sb.err_prob), sb.err_prob.size, None) == A.SX_ERR_ARG
    bad_idx = sb.err_idx.copy()
    bad_idx[5] = sb.err_prob.size
    for fn in (ctx.somatic_indel,):
        with pytest.raises(SxError) as e:
            fn(_with(sb, err_idx=bad_idx), o)
        assert e.value.code == A.SX_ERR_ARG
    key = sb.key.copy()
    key["type"][3] = A.SX_INDEL_TYPE_MISMATCH
    for b in (_with(sb, err_idx=bad_idx), _with(sb, key=key)):
        db = DevSomaticIndelBatch(ctx, b)
        with pytest.raises(SxError) as e:
            ctx.somatic_indel_dev(db, o)
        assert e.value.code == A.SX_ERR_ARG
    with pytest.raises(SxError) as e:
        ctx.somatic_indel(_with(sb, key=key), o)
    assert e.value.code == A.SX_ERR_ARG
    # the context stays usable
    assert ctx.somatic_indel(sb, o).tobytes() == G.ox_somatic_indel(o, sb).tobytes()


@pytest.mark.gpu
def test_empty_batch(ctx):
    from strelka_b200.api import DevSomaticIndelBatch

    sb = G.random_somatic_indel_batch(np.random.default_rng(3), 0)
    o = A.default_sindel_opts()
    assert ctx.somatic_indel(sb, o).size == 0
    db = DevSomaticIndelBatch(ctx, sb)
    ctx.somatic_indel_dev(db, o)
