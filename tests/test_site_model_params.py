"""The somatic SNV model (K2b) and the indel genotype model (K5) away from their default parameters and at the edges of their input: the
oracle (oracle/strelka_oracle.cpp) against the reference's own code at every point of tests/site_params.py, on the edge batches of
tests/specgen.py, and the frozen answers of tests/golden/site_params_ref.npz (which the GPU tests compare with) against the reference."""
import numpy as np
import pytest

import reflib
import site_params as SP
import specgen

KINDS = specgen.SOMATIC_EDGE_KINDS
# the kinds computed without being forced at every parameter point; the other kinds that can be (SOMATIC_FORCED_ONLY_KINDS and 'n_ref'
# aside) are at some points only, test_k2b_unforced_kinds_over_the_sweep
UNFORCED_EVERYWHERE = ("plain", "q_extreme", "t1_tier_filtered", "alt_tie", "deep")


@pytest.fixture(scope="module")
def golden():
    with np.load(SP.GOLDEN) as z:
        return {k: z[k] for k in z.files}


def test_frozen_inputs_are_the_generators():
    """the edge batches are the ones whose reference answers are frozen (needs no reference)"""
    with np.load(SP.GOLDEN) as z:
        assert bytes(z["inputs"]).decode() == SP.inputs_digest()


def k2b_coverage(r, forced, kind):
    """per edge kind, the number of computed sites that were forced and that were not"""
    c = r["is_computed"] == 1
    return {KINDS[k]: (int((c & (kind == k) & (forced == 1)).sum()), int((c & (kind == k) & (forced == 0)).sum())) for k in range(len(KINDS))}


@pytest.mark.ref
@pytest.mark.parametrize("point", list(SP.K2B_POINTS))
def test_k2b_oracle_matches_the_reference(point, golden):
    npb, tpb, forced, kind = SP.k2b_edge_batch()
    p = SP.k2b(point)
    for mode in specgen.SOMATIC_TIER2_MODES:
        n, t = specgen.somatic_tier2_view(npb, tpb, mode)
        want = reflib.ref_somatic(p, n, t, forced)
        fields = SP.reference_fields(p, n, t, forced)
        SP.compare_fields(reflib.ox_somatic(p, n, t, forced), fields, (point, mode))
        assert np.array_equal(fields, golden[SP.golden_key("k2b", point, mode)]), (point, mode)
        cov = k2b_coverage(want, forced, kind)
        assert cov["n_ref"] == (0, 0)
        for k in KINDS:
            if k != "n_ref":
                assert cov[k][0] > 0, (point, mode, k)
        for k in UNFORCED_EVERYWHERE:
            assert cov[k][1] > 0, (point, mode, k)
        if mode in ("normal_only", "tumor_only"):  # tier2 on one sample: the tier1-only answer
            assert np.array_equal(fields, SP.reference_fields(p, *specgen.somatic_tier2_view(npb, tpb, "neither"), forced))


@pytest.mark.ref
def test_k2b_unforced_kinds_over_the_sweep():
    """the kinds that reach is_computed unforced at some points: each does somewhere in the sweep; and every point changes the reference's
    answer on the edge batch (so each parameter is read)"""
    npb, tpb, forced, kind = SP.k2b_edge_batch()
    unforced = {k: 0 for k in KINDS}
    answers = {}
    for point in SP.K2B_POINTS:
        r = reflib.ref_somatic(SP.k2b(point), npb, tpb, forced)
        answers[point] = SP.reference_fields(SP.k2b(point), npb, tpb, forced).tobytes()
        for k, (_, u) in k2b_coverage(r, forced, kind).items():
            unforced[k] += u
    for k in KINDS:
        if k in specgen.SOMATIC_FORCED_ONLY_KINDS or k == "n_ref":
            assert unforced[k] == 0, k
        else:
            assert unforced[k] > 0, k
    assert len(set(answers.values())) == len(answers)


@pytest.mark.ref
@pytest.mark.parametrize("point", list(SP.K5_POINTS))
def test_k5_oracle_matches_the_reference(point, golden):
    ib = SP.k5_edge_batch()
    p = SP.k5(point)
    want = reflib.ref_indel_gl(p, ib)
    got = reflib.ox_indel_gl(p, ib)
    assert np.array_equal(want["n_gt"], got["n_gt"])
    assert np.array_equal(want["support"], got["support"])
    assert np.array_equal(want["gt_lhood"].view(np.uint64), got["gt_lhood"].view(np.uint64))
    assert want.tobytes() == got.tobytes()
    assert want.tobytes() == golden[SP.golden_key("k5", point)].tobytes()
    n_reads = np.diff(ib.read_off.astype(np.int64))
    assert set(n_reads.tolist()) == set(specgen.INDEL_EDGE_READ_COUNTS) and want["n_gt"].max() == 15


@pytest.mark.ref
def test_k5_every_point_changes_the_answer():
    ib = SP.k5_edge_batch()
    answers = {point: reflib.ref_indel_gl(SP.k5(point), ib).tobytes() for point in SP.K5_POINTS}
    assert len(set(answers.values())) == len(answers)


@pytest.mark.ref
def test_strand_log_sum_nan_is_the_references():
    """Two quality-0 reference calls, one per strand, make both strand sums of the tumor's strand states -inf, and getLogSum<float>(-inf, -inf)
    NaN.  The reference's NaN is x86's default one, 0xffc00000, and it survives the + ln(1/2) after it; the oracle's strand states (and
    the device's, tests/test_gpu_site_model_params.py) carry the same bits."""
    from strelka_b200 import _abi as A
    from strelka_b200 import batch as B

    v = np.float32(reflib.ref().ref_getLogSum_float(float("-inf"), float("-inf")))
    assert int(v.view(np.uint32)) == 0xFFC00000
    assert int((v + np.float32(np.log(0.5))).view(np.uint32)) == 0xFFC00000
    calls = [list(B.pack_call([0, 0, 37, 37], [0, 0, 1, 1], [1, 0, 1, 0]))]
    pb = B.PileupBatch.from_sites(calls, "A")
    got = reflib.ox_somatic(A.default_params(), pb, pb, np.ones(1, np.uint8))
    assert got["is_computed"][0] == 1
    assert np.all(got["tumor_lhood"][0, 21:30].view(np.uint32) == 0xFFC00000)
