"""K2b's callable mode and the somatic callable regions on the GPU:
  - sx_site_gl_somatic_callable[_dev] against the oracle (oracle/somatic_callable_oracle.cpp) byte for byte, and against the reference's
    frozen answers (tests/golden/somatic_callable_ref.npz), at every case of tests/callable_gen.py;
  - sx_somatic_callable_regions_dev against the host builder (batch.somatic_callable_regions) on edge inputs and sizes across sx_scan's tiles;
  - the somatic window pass in callable mode on the seeded two-sample windows and on a bench-shaped window: its site_snv against
    sx_site_gl_somatic_callable_dev on the pass's own columns and the oracle, its records against a default-mode pass, its regions against the
    host builder, and a second run.  Its QSS, NQSS and regions equal the reference's position_somatic_snv_call(..., true, sgt) and
    SomaticCallableProcessor on the pass's columns where oracle/_ref is built, and everywhere their digest frozen from that reference run
    (tests/golden/make_somatic_callable_window_golden.py).
The error tests pass bad arguments only."""
import os
import sys

import numpy as np
import pytest

import json

import callable_gen as G
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import somatic_window_leg as SW  # noqa: E402
import window_workload as WW  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctxs():
    from strelka_b200.api import Context

    made = {}

    def get(p):
        key = bytes(p)
        if key not in made:
            made[key] = Context(0, params=p)
        return made[key]

    yield get
    for c in made.values():
        c.close()


@pytest.fixture(scope="module")
def ctx(ctxs):
    return ctxs(A.default_params())


def test_entries_equal_oracle_and_frozen_reference(ctxs):
    from strelka_b200.api import DeviceArray, DevPileupBatch

    gold = G.golden()
    assert bytes(gold["inputs"]).decode() == G.inputs_digest()
    for name, p, n, t, forced in G.cases():
        ctx = ctxs(p)
        want = G.ox_callable(p, n, t, forced)
        got = ctx.site_gl_somatic_callable(n, t, forced)
        assert got.tobytes() == want.tobytes(), name
        dn, dt = DevPileupBatch(ctx, n), DevPileupBatch(ctx, t)
        df = DeviceArray(ctx, forced.nbytes + 64).upload(forced)
        out = DeviceArray(ctx, want.nbytes + 64)
        ctx.site_gl_somatic_callable_dev(dn, dt, df, out)
        assert out.download(A.SSNV_RESULT_DT, n.n_sites).tobytes() == want.tobytes(), name
        for x in [df, out] + list(dn.bufs.values()) + list(dt.bufs.values()):
            x.free()
        G.compare_fields(got, gold[name + "__fields"], name)
        # the default entry is unchanged by the mode's existence: its records carry NQSS 0
        assert not ctx.site_gl_somatic(n, t, forced)["nonsomatic_qphred"].any()


def _regions_dev(ctx, r: np.ndarray, pos_begin: int, cap=None):
    from strelka_b200.api import DeviceArray

    cap = max(1, (r.size + 1) // 2) if cap is None else cap
    d = DeviceArray(ctx, r.nbytes + 64)
    if r.size:
        d.upload(r)
    rb, re = DeviceArray(ctx, 4 * cap + 64), DeviceArray(ctx, 4 * cap + 64)
    try:
        n = ctx.somatic_callable_regions_dev(d, r.size, pos_begin, rb, re, cap)
        return rb.download(np.int32, n), re.download(np.int32, n)
    finally:
        for x in (d, rb, re):
            x.free()


def _check_regions(ctx, r, pos_begin):
    gb, ge = _regions_dev(ctx, r, pos_begin)
    wb, we = B.somatic_callable_regions(r, pos_begin)
    assert np.array_equal(gb, wb) and np.array_equal(ge, we), (r.size, pos_begin)
    return gb.size


def test_regions_edges(ctx):
    rng = np.random.default_rng(5)
    assert _check_regions(ctx, G.synthetic_records(rng, 0, 0.5), 10) == 0
    assert _check_regions(ctx, G.synthetic_records(rng, 1000, 0.0), 10) == 0  # no callable position
    assert _check_regions(ctx, G.synthetic_records(rng, 1000, 1.0), 10) == 1  # all callable
    r = G.synthetic_records(rng, 1000, 0.0)
    r["qphred"][:3] = 15
    r["nonsomatic_qphred"][-2:] = 40
    assert _check_regions(ctx, r, -5) == 2  # an interval at each edge (and coordinates below 0)
    r = G.synthetic_records(rng, 1001, 1.0)
    r["qphred"][1::2] = 14
    r["nonsomatic_qphred"][1::2] = 14
    assert _check_regions(ctx, r, 0) == 501  # alternating
    r = G.synthetic_records(rng, 1, 1.0)
    assert _check_regions(ctx, r, 2**31 - 2) == 1


@pytest.mark.parametrize("n", [4095, 4096, 4097, 3 * 4096 + 1, 65536 * 3 + 7, 1_000_003])
def test_regions_sizes(ctx, n):
    rng = np.random.default_rng(n)
    for p in (0.3, 0.97):
        _check_regions(ctx, G.synthetic_records(rng, n, p), 1234)


def test_regions_capacity_and_arguments(ctx):
    from strelka_b200.api import DeviceArray, SxError

    r = G.synthetic_records(np.random.default_rng(9), 5000, 0.5)
    wb, we = B.somatic_callable_regions(r, 0)
    assert wb.size > 10
    with pytest.raises(SxError) as e:
        _regions_dev(ctx, r, 0, cap=wb.size - 1)
    assert e.value.code == A.SX_ERR_CAPACITY and int(e.value.totals[0]) == wb.size
    gb, ge = _regions_dev(ctx, r, 0, cap=wb.size)
    assert np.array_equal(gb, wb) and np.array_equal(ge, we)
    d = DeviceArray(ctx, r.nbytes).upload(r)
    rb = DeviceArray(ctx, 64)
    for args in ((None, 10, 0, rb, rb, 4), (d, 10, 0, None, rb, 4), (d, 10, 0, rb, None, 4), (d, 10, 2**31 - 5, rb, rb, 4)):
        with pytest.raises(SxError) as e:
            ctx.somatic_callable_regions_dev(*args)
        assert e.value.code == A.SX_ERR_ARG
    assert ctx.lib.sx_somatic_callable_regions_dev(ctx.h, d.ptr, 10, 0, rb.ptr, rb.ptr, 4, None) == A.SX_ERR_ARG
    d.free()
    rb.free()


def seeded_window_inputs():
    """(key, normal, tumor, loci, key_gid, forced, opts, use_tier2) of the seeded two-sample windows"""
    import test_zzzzzzzz_gpu_somatic_window as SWT

    for case in SWT.CASES:
        for key, normal, tumor, loci, key_gid, forced in SWT.case_inputs(case):
            yield f"seeded.{key}", normal[2], tumor[2], loci, key_gid, forced, SWT._opts(), False


def synthetic_window_inputs(tier2: bool):
    """the same of the bench-shaped window, every fourth read a tier2 mapping with tier2 evidence"""
    w = WW.make_window(WW.load_synth(), 400, 11)
    normal, tumor, loci, key_gid, forced = SW.two_sample_window(w, 11)
    if tier2:
        for x in (normal, tumor):
            x.a["read_flags"][: x.n_reads : 4] &= np.uint8(~A.SX_PRF_TIER1 & 0xFF)
    o = A.default_sindel_opts()
    o.useTier2Evidence = int(tier2)
    return f"synthetic.tier2_{int(tier2)}", normal, tumor, loci, key_gid, forced, o, tier2


def callable_pass(ctx, normal, tumor, loci, key_gid, forced, opts=None, use_tier2=False):
    """one callable-mode pass: (download, regions, the two samples' columns as K2b batches)"""
    from strelka_b200.api import DevSomaticWindow

    sw = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], compute_nonsomatic=True, snv_forced=forced, opts=opts, use_tier2=use_tier2)
    sw.run()
    got = sw.download()
    regions = sw.callable_regions()
    sw.free()
    t2 = (lambda x: (x["t2_off"], x["t2_calls"])) if use_tier2 else (lambda x: (None, None))
    pb = [B.PileupBatch(x["site_off"], x["calls"], ref_base_of(normal), None, *t2(x)) for x in (got["normal"], got["tumor"])]
    return got, regions, pb


def ref_base_of(w):
    return np.ascontiguousarray(w.a["ref"][w.report_begin - w.ref_begin : w.report_end - w.ref_begin])


def _callable_pass_check(ctx, key, normal, tumor, loci, key_gid, forced, opts=None, use_tier2=False):
    """one window in callable mode: returns (download, regions)"""
    from strelka_b200.api import DevSomaticWindow

    kw = dict(snv_forced=forced, opts=opts, use_tier2=use_tier2)
    sw = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], compute_nonsomatic=True, **kw)
    sw.run()
    got = sw.download()
    regions = sw.callable_regions()
    sw.run()  # run to run: the same bytes
    again = sw.download()
    for k in ("site_snv", "snv_calls", "indel", "indel_calls", "totals"):
        assert again[k].tobytes() == got[k].tobytes(), k
    for a, b in zip(sw.callable_regions(), regions):
        assert np.array_equal(a, b)
    sw.free()
    # K2b in callable mode on the pass's own columns, and the oracle on them
    t2 = (lambda x: (x["t2_off"], x["t2_calls"])) if use_tier2 else (lambda x: (None, None))
    pb = [B.PileupBatch(x["site_off"], x["calls"], ref_base_of(normal), None, *t2(x)) for x in (got["normal"], got["tumor"])]
    assert ctx.site_gl_somatic_callable(pb[0], pb[1], forced).tobytes() == got["site_snv"].tobytes()
    assert G.ox_callable(ctx.params, pb[0], pb[1], forced).tobytes() == got["site_snv"].tobytes()
    # the records: a default-mode pass's, but for nonsomatic_qphred
    sd = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], **kw)
    sd.run()
    dflt = sd.download()
    sd.free()
    a = got["snv_calls"].copy()
    assert np.array_equal(a["r"]["nonsomatic_qphred"], got["site_snv"]["nonsomatic_qphred"][a["pos"] - normal.report_begin])
    a["r"]["nonsomatic_qphred"] = 0
    assert a.tobytes() == dflt["snv_calls"].tobytes()
    for k in ("indel", "indel_calls", "totals"):
        assert got[k].tobytes() == dflt[k].tobytes(), k
    # the regions: the host builder, and the reference's SomaticCallableProcessor on the same columns
    wb, we = B.somatic_callable_regions(got["site_snv"], normal.report_begin)
    assert np.array_equal(regions[0], wb) and np.array_equal(regions[1], we)
    if G.have_ref():
        r, bed = G.ref_callable(ctx.params, pb[0], pb[1], forced, pos_begin=normal.report_begin)
        assert G.bed_text(*regions) == bed
        assert np.array_equal(r["nonsomatic_qphred"], got["site_snv"]["nonsomatic_qphred"]) and np.array_equal(r["qphred"], got["site_snv"]["qphred"])
    with open(G.WINDOW_GOLDEN) as f:
        want = json.load(f)[key]
    assert G.window_digest(got["site_snv"]["qphred"], got["site_snv"]["nonsomatic_qphred"], *regions) == want, (key, "regenerate the frozen digests")
    return got, regions


def test_callable_window_cases(ctx):
    n_windows = n_computed = 0
    for key, normal, tumor, loci, key_gid, forced, opts, tier2 in seeded_window_inputs():
        got, _ = _callable_pass_check(ctx, key, normal, tumor, loci, key_gid, forced, opts=opts, use_tier2=tier2)
        n_windows += 1
        n_computed += int(got["site_snv"]["is_computed"].sum())
    # (these shallow windows have no callable position: test_callable_synthetic_window has them)
    assert n_windows > 0 and n_computed > 0


@pytest.mark.parametrize("tier2", [False, True])
def test_callable_synthetic_window(ctx, tier2):
    key, normal, tumor, loci, key_gid, forced, o, tier2 = synthetic_window_inputs(tier2)
    got, regions = _callable_pass_check(ctx, key, normal, tumor, loci, key_gid, forced, opts=o, use_tier2=tier2)
    s = got["site_snv"]
    comp = s["is_computed"] == 1
    assert comp.sum() > 0.9 * s.size and regions[0].size > 0
    assert ((s["nonsomatic_qphred"] >= 15) & (s["qphred"] < 15)).any()
