"""K2b (somatic SNVs) and K5 (indel genotype likelihoods) on the GPU at every parameter point of tests/site_params.py, on the edge batches of
tests/specgen.py: one Context per point, built with that point's parameters.  Compared with the oracle on whole records, byte for byte,
through the host-array and the device-resident entries, and with the reference's answers frozen in tests/golden/site_params_ref.npz
(tests/test_site_model_params.py checks those against the reference and the oracle).  Also: a batch of ~200k sites at one point (several
waves of the grid-stride loop), and the somatic window pass on a context built at a non-default point."""
import contextlib
import ctypes as C
import os
import sys

import numpy as np
import pytest

import reflib
import site_params as SP
import specgen
from strelka_b200 import _abi as A

pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def context(params):
    from strelka_b200.api import Context

    c = Context(0, params)
    try:
        yield c
    finally:
        c.close()


@pytest.fixture(scope="module")
def golden():
    with np.load(SP.GOLDEN) as z:
        assert bytes(z["inputs"]).decode() == SP.inputs_digest()
        return {k: z[k] for k in z.files}


def _k2b_dev(ctx, n, t, forced):
    from strelka_b200.api import DeviceArray, DevPileupBatch

    dn, dt = DevPileupBatch(ctx, n), DevPileupBatch(ctx, t)
    f = DeviceArray(ctx, forced.nbytes + 64).upload(forced)
    out = DeviceArray(ctx, n.n_sites * A.SSNV_RESULT_DT.itemsize + 64)
    ctx.site_gl_somatic_dev(dn, dt, f, out)
    return out.download(A.SSNV_RESULT_DT, n.n_sites)


@pytest.mark.parametrize("point", list(SP.K2B_POINTS))
def test_k2b_at_parameter_point(point, golden):
    npb, tpb, forced, kind = SP.k2b_edge_batch()
    p = SP.k2b(point)
    with context(p) as ctx:
        for mode in specgen.SOMATIC_TIER2_MODES:
            n, t = specgen.somatic_tier2_view(npb, tpb, mode)
            want = reflib.ox_somatic(p, n, t, forced)
            got = ctx.site_gl_somatic(n, t, forced)
            # every record, computed or not, to the last padding byte
            assert got.tobytes() == want.tobytes(), (point, mode)
            assert _k2b_dev(ctx, n, t, forced).tobytes() == want.tobytes(), (point, mode)
            SP.compare_fields(got, golden[SP.golden_key("k2b", point, mode)], (point, mode))
            c = got["is_computed"] == 1
            assert all(((kind == k) & c & (forced == 1)).any() for k in range(len(specgen.SOMATIC_EDGE_KINDS)) if specgen.SOMATIC_EDGE_KINDS[k] != "n_ref")
        # no forced-output array (NULL): as all 0
        zeros = np.zeros(npb.n_sites, np.uint8)
        assert ctx.site_gl_somatic(npb, tpb).tobytes() == reflib.ox_somatic(p, npb, tpb, zeros).tobytes()


def test_k2b_large_batch():
    """~200k sites drawn from the edge batch in random order, tier2 on both samples, at one non-default point: every block walks several
    sites of the grid-stride loop"""
    npb, tpb, _, _ = SP.k2b_edge_batch()
    rng = np.random.default_rng(8300)
    idx = rng.integers(0, npb.n_sites, 200_000)
    n, t = specgen.pileup_take(npb, idx), specgen.pileup_take(tpb, idx)
    forced = (rng.random(idx.size) < 0.3).astype(np.uint8)
    p = SP.k2b(SP.K2B_LARGE_POINT)
    want = reflib.ox_somatic(p, n, t, forced)
    assert int((want["is_computed"] == 1).sum()) > 50_000
    with context(p) as ctx:
        got = ctx.site_gl_somatic(n, t, forced)
        assert got.tobytes() == want.tobytes()
        assert _k2b_dev(ctx, n, t, forced).tobytes() == want.tobytes()


@pytest.mark.parametrize("point", list(SP.K5_POINTS))
def test_k5_at_parameter_point(point, golden):
    from strelka_b200.api import DeviceArray, _device_twin

    ib = SP.k5_edge_batch()
    p = SP.k5(point)
    want = reflib.ox_indel_gl(p, ib)
    assert want.tobytes() == golden[SP.golden_key("k5", point)].tobytes()
    with context(p) as ctx:
        got = ctx.indel_gl(ib)
        assert got.tobytes() == want.tobytes(), point
        dev, _bufs = _device_twin(ctx, ib.c, ib, 64)
        out = DeviceArray(ctx, ib.n_loci * A.INDEL_RESULT_DT.itemsize + 64)
        ctx._chk(ctx.lib.sx_indel_gl_dev(ctx.h, C.byref(dev), out.ptr))
        assert out.download(A.INDEL_RESULT_DT, ib.n_loci).tobytes() == want.tobytes(), point


def test_somatic_window_pass_reads_the_context_parameters():
    """the somatic window pass on contexts built at non-default points: its SNV records are sx_site_gl_somatic's on the pass's own columns on
    that context, and the oracle's at that point.  (At ssebf = 0.5 this window's records happen to be the defaults' as well; at a somatic
    SNV rate of 0.1 they are not.)"""
    from strelka_b200.api import DevSomaticWindow
    from strelka_b200 import batch as B

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import somatic_window_leg as SW
    import window_workload as WW

    differs = {}
    for point in SP.WINDOW_POINTS:
        p = SP.k2b(point)
        with context(p) as ctx:
            w = WW.make_window(WW.load_synth(), 400, 11)
            normal, tumor, loci, key_gid, forced = SW.two_sample_window(w, 11)
            for x in (normal, tumor):  # every fourth read a tier2 mapping
                x.a["read_flags"][: x.n_reads : 4] &= np.uint8(~A.SX_PRF_TIER1 & 0xFF)
            sw = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced, use_tier2=True)
            sw.run()
            got = sw.download()
            sw.free()
            ref_base = np.ascontiguousarray(normal.a["ref"][normal.report_begin - normal.ref_begin : normal.report_end - normal.ref_begin])
            pb = [B.PileupBatch(x["site_off"], x["calls"], ref_base, None, x["t2_off"], x["t2_calls"]) for x in (got["normal"], got["tumor"])]
            assert int(pb[1].t2_off[-1]) > 0
            assert ctx.site_gl_somatic(pb[0], pb[1], forced).tobytes() == got["site_snv"].tobytes(), point
        f = None if forced is None else np.ascontiguousarray(forced, np.uint8)
        assert reflib.ox_somatic(p, pb[0], pb[1], f).tobytes() == got["site_snv"].tobytes(), point
        assert (got["site_snv"]["qphred"] != 0).sum() > 0
        differs[point] = reflib.ox_somatic(A.default_params(), pb[0], pb[1], f).tobytes() != got["site_snv"].tobytes()
    assert differs["snv_rate_0.1"]
