"""Every public entry point that launches work, through the public API only: what it returns, the launches it reports (sx_last_timing
and the sx_total_launches delta), its outputs against the oracle or against the other entry of its stage, a NULL-argument call (code and
message) and the empty batch (code, and the zeros written to totals and first offsets).  The values are the library's established ones: a
change in how a stage is enqueued must leave all of them as they are."""
import ctypes as C

import numpy as np
import pytest

import indel_reads_gen as G
import reflib
import sindel_gen
import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

pytestmark = pytest.mark.gpu

ENTRIES_DEV = ("score_alignments", "site_gl_germline", "site_gl_somatic", "global_align", "pileup_reads", "indel_gl", "somatic_indel", "score_indels",
               "link_indel_reads", "enumerate_alignments", "realign_gates", "alignment_indels", "link_alignments", "choose_realignment", "process_window")
# (entry, the name its NULL-argument message carries)
NULL_CASES = [(e + "_dev", e + "_dev") for e in ENTRIES_DEV] + [(e, e) for e in ENTRIES_DEV] + [
    ("read_max_dev", "read_max_dev"), ("dependent_eprob", "dependent_eprob"), ("somatic_indel_from_records_dev", "somatic_indel_from_records_dev")]


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


def _counted(ctx, call):
    """Runs call(); returns (what it returned, timing().launches, the sx_total_launches delta)."""
    before = ctx.total_launches()
    out = call()
    return out, int(ctx.timing().launches), ctx.total_launches() - before


def _null_args(fn, h):
    args = [h]
    for t in fn.argtypes[1:]:
        args.append(0 if isinstance(t, type) and issubclass(t, C._SimpleCData) and t._type_ in "bBhHiIlLqQ" else None)
    return args


@pytest.mark.parametrize("entry,name", NULL_CASES)
def test_null_argument(ctx, entry, name):
    fn = getattr(ctx.lib, "sx_" + entry)
    before = ctx.total_launches()
    assert fn(*_null_args(fn, ctx.h)) == A.SX_ERR_ARG
    assert ctx.last_error() == f"sx_{name}: NULL argument"
    assert ctx.total_launches() == before


def _dev_zeroed(ctx, words):
    from strelka_b200.api import DeviceArray

    return DeviceArray(ctx, 4 * words + 64).upload(np.full(words, 0xFFFFFFFF, np.uint32))


def test_empty_batches_write_zero_totals_and_offsets(ctx):
    """K7, K7a and K9 zero their totals and first offset, K6b its totals and both offset arrays' first entry; nothing is launched."""
    lib, h, byref = ctx.lib, ctx.h, C.byref
    dummy = _dev_zeroed(ctx, 16)
    eb = A.SxEnumBatch()
    cases = []
    # K7
    t, off = _dev_zeroed(ctx, 4), _dev_zeroed(ctx, 4)
    eo = A.SxEnumOut(0, 0, 0, t.ptr, off.ptr)
    cases.append(("enumerate_alignments_dev", lambda: lib.sx_enumerate_alignments_dev(h, byref(eb), byref(eo)), [(t, 3), (off, 1)]))
    # K7a
    t2, off2 = _dev_zeroed(ctx, 4), _dev_zeroed(ctx, 4)
    po = A.SxPrepOut(0, t2.ptr, off2.ptr)
    cases.append(("alignment_indels_dev", lambda: lib.sx_alignment_indels_dev(h, byref(eb), dummy.ptr, dummy.ptr, dummy.ptr, None, None, byref(po)),
                  [(t2, 1), (off2, 1)]))
    # K9
    t3, off3 = _dev_zeroed(ctx, 4), _dev_zeroed(ctx, 4)
    rb, ro = A.SxRealignBatch(), A.SxRealignOut(0, t3.ptr, off3.ptr)
    cases.append(("choose_realignment_dev", lambda: lib.sx_choose_realignment_dev(h, byref(rb), None, byref(ro)), [(t3, 1), (off3, 1)]))
    # K6b
    t4, ro4, ao4 = _dev_zeroed(ctx, 4), _dev_zeroed(ctx, 4), _dev_zeroed(ctx, 4)
    s, loci = A.SxIndelReadsSample(), A.SxIndelLoci()
    lo = A.SxIndelReadsOut(ao4.ptr, None, ro4.ptr, None, None, t4.ptr, 0, 0)
    th = np.full(2, 7, np.uint32)
    cases.append(("link_indel_reads_dev", lambda: lib.sx_link_indel_reads_dev(h, byref(s), byref(s), byref(loci), byref(lo), th.ctypes.data),
                  [(t4, 2), (ro4, 1), (ao4, 1)]))
    for name, call, zeroed in cases:
        rc, launches, delta = _counted(ctx, call)
        assert (rc, launches, delta) == (A.SX_OK, 0, 0), name
        for arr, n in zeroed:
            assert np.array_equal(arr.download(np.uint32, n), np.zeros(n, np.uint32)), name
    assert np.array_equal(th, np.zeros(2, np.uint32))
    # the host-array forms write the same zeros into the caller's arrays
    ht, hoff = np.full(4, 9, np.uint32), np.full(4, 9, np.uint32)
    eo_h = A.SxEnumOut(0, 0, 0, ht.ctypes.data, hoff.ctypes.data)
    assert lib.sx_enumerate_alignments(h, byref(eb), byref(eo_h)) == A.SX_OK and ht[:3].tolist() == [0, 0, 0] and hoff[0] == 0
    ht[:], hoff[:] = 9, 9
    po_h = A.SxPrepOut(0, ht.ctypes.data, hoff.ctypes.data)
    assert lib.sx_alignment_indels(h, byref(eb), dummy.ptr, dummy.ptr, dummy.ptr, None, None, byref(po_h)) == A.SX_OK and ht[0] == 0 and hoff[0] == 0
    ht[:], hoff[:] = 9, 9
    ro_h = A.SxRealignOut(0, ht.ctypes.data, hoff.ctypes.data)
    assert lib.sx_choose_realignment(h, byref(rb), None, byref(ro_h)) == A.SX_OK and ht[0] == 0 and hoff[0] == 0
    # the other device entries return at once on an empty batch
    for name, call in (("score_indels_dev", lambda: lib.sx_score_indels_dev(h, byref(A.SxScoreIndelsBatch()), None, byref(A.SxScoreIndelsOut()))),
                       ("realign_gates_dev", lambda: lib.sx_realign_gates_dev(h, byref(A.SxGateBatch()), byref(A.SxGateOut())))):
        assert _counted(ctx, call) == (A.SX_OK, 0, 0), name


def test_k1_k2_k3_launches_and_outputs(ctx):
    from strelka_b200.api import DevAlignBatch, DevGaBatch, DevPileupBatch, DeviceArray

    rng = np.random.default_rng(4040)
    hb = B.build_align_batch([specgen.simple_region(rng, n_reads=30) for _ in range(16)])
    want = reflib.ox_score(hb)
    got, launches, delta = _counted(ctx, lambda: ctx.score_alignments(hb))
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64)) and (launches, delta) == (1, 1)  # one per chunk
    db = DevAlignBatch(ctx, hb)
    assert _counted(ctx, lambda: ctx.score_alignments_dev(db))[1:] == (2, 2)
    assert np.array_equal(db.out.download(np.float64, hb.n_alns).view(np.uint64), want.view(np.uint64))
    ml, ma = DeviceArray(ctx, hb.n_reads * 8 + 16), DeviceArray(ctx, hb.n_reads * 4 + 16)
    assert _counted(ctx, lambda: ctx.read_max_dev(db, ml, ma))[1:] == (1, 1)

    pb = specgen.random_pileups(rng, 300, depth=30.0)
    want = ctx.site_gl_germline(pb, True)
    assert (int(ctx.timing().launches)) == 1
    dp = DevPileupBatch(ctx, pb)
    out = DeviceArray(ctx, pb.n_sites * A.DIGT_RESULT_DT.itemsize + 16)
    assert _counted(ctx, lambda: ctx.site_gl_germline_dev(dp, out, True))[1:] == (2, 2)
    assert out.download(A.DIGT_RESULT_DT, pb.n_sites).tobytes() == want.tobytes()
    w = reflib.ox_germline(A.default_params(), pb, True)
    assert np.array_equal(want["lhood"].view(np.uint32), w["lhood"].view(np.uint32))
    assert _counted(ctx, lambda: ctx.dependent_eprob(pb))[1:] == (1, 1)

    tpb = specgen.random_pileups(rng, 300, depth=30.0)
    want = ctx.site_gl_somatic(pb, tpb)
    assert int(ctx.timing().launches) == 1
    dt = DevPileupBatch(ctx, tpb)
    so = DeviceArray(ctx, pb.n_sites * A.SSNV_RESULT_DT.itemsize + 16)
    assert _counted(ctx, lambda: ctx.site_gl_somatic_dev(dp, dt, None, so))[1:] == (1, 1)
    assert so.download(A.SSNV_RESULT_DT, pb.n_sites).tobytes() == want.tobytes()

    qs, rs = specgen.random_ga_problems(rng, 64)
    gb = B.GaBatch(qs, rs, max_ops=400)
    sc = ctx.active_region_scores()
    (r1, c1), launches, delta = _counted(ctx, lambda: ctx.global_align(sc, gb))
    r2, c2 = reflib.ox_global_align(sc, gb)
    assert np.array_equal(r1, r2) and np.array_equal(c1, c2) and (launches, delta) == (1, 1)
    dg = DevGaBatch(ctx, gb)
    assert _counted(ctx, lambda: ctx.global_align_dev(sc, dg))[1:] == (4, 4)
    assert dg.res.download(A.GA_RESULT_DT, gb.n).tobytes() == r1.tobytes()


def _on_device(ctx, owner, c, outputs=False):
    """A copy of the ctypes struct `c` whose pointers to `owner`'s numpy arrays point at device copies of them.  With `outputs`, also a
    function that copies the device arrays back into `owner`'s."""
    from strelka_b200.api import DeviceArray

    arrays = {a.ctypes.data: a for a in vars(owner).values() if isinstance(a, np.ndarray)}
    d = type(c).from_buffer_copy(c)
    keep = []
    for name, t in c._fields_:
        p = getattr(c, name)
        if t is C.c_void_p and p:
            assert p in arrays, name  # every array the struct names goes to the device
            buf = DeviceArray(ctx, arrays[p].nbytes + 64).upload(arrays[p])
            keep.append((arrays[p], buf))
            setattr(d, name, buf.ptr)
    d._keep = keep

    def back():
        for a, buf in keep:
            a.reshape(-1).view(np.uint8)[:] = buf.download(np.uint8, a.nbytes)

    return (d, back) if outputs else d


def test_k4_k5_k6_launches_and_outputs(ctx):
    from strelka_b200.api import DeviceArray, DevScoreIndelsBatch

    rng = np.random.default_rng(4141)
    reads, ref, ref_begin, cand = specgen.random_pileup_reads(rng, n_reads=300, ref_len=1500)
    prb = B.PileupReadsBatch(reads, ref, ref_begin, ref_begin + 50, ref_begin + len(ref) - 50, cand)
    got, launches, delta = _counted(ctx, lambda: ctx.pileup_reads(prb))
    for a, b in zip(got, reflib.ox_pileup_reads(prb)):
        assert np.array_equal(a, b)
    assert (launches, delta) == (8, 8)  # count, two three-launch scans, fill
    cols = B.PileupColumns(prb)
    dev_b, dev_c, back = _on_device(ctx, prb, prb.c), *_on_device(ctx, cols, cols.c, outputs=True)
    assert _counted(ctx, lambda: ctx.lib.sx_pileup_reads_dev(ctx.h, C.byref(dev_b), C.byref(dev_c)))[1:] == (8, 8)
    back()
    for a, b in zip(cols.trimmed(), got):
        assert np.array_equal(a, b)

    ib = B.IndelBatch(specgen.random_indel_loci(rng, 200))
    gi, launches, delta = _counted(ctx, lambda: ctx.indel_gl(ib))
    assert gi.tobytes() == reflib.ox_indel_gl(A.default_params(), ib).tobytes() and (launches, delta) == (1, 1)
    out = DeviceArray(ctx, ib.n_loci * A.INDEL_RESULT_DT.itemsize + 16)
    dev_ib = _on_device(ctx, ib, ib.c)
    assert _counted(ctx, lambda: ctx.lib.sx_indel_gl_dev(ctx.h, C.byref(dev_ib), out.ptr))[1:] == (1, 1)
    assert out.download(A.INDEL_RESULT_DT, ib.n_loci).tobytes() == gi.tobytes()

    regions = [specgen.simple_region(rng, n_reads=30) for _ in range(16)]
    sb = B.score_indels_batch_from_regions(regions)
    lnp = np.concatenate([reflib.ox_score(B.build_align_batch(regions)), [0.0]])
    got, launches, delta = _counted(ctx, lambda: ctx.score_indels(sb, lnp))
    for a, b in zip(got, reflib.ox_score_indels(sb, lnp)):
        assert a.tobytes() == b.tobytes()
    assert (launches, delta) == (5, 5)
    ds = DevScoreIndelsBatch(ctx, sb)
    assert _counted(ctx, lambda: ctx.score_indels_dev(ds, DeviceArray(ctx, lnp.nbytes + 64).upload(lnp)))[1:] == (5, 5)
    for a, b in zip(ds.download(), got):
        assert a.tobytes() == b.tobytes()


def test_k5b_k6b_launches_and_outputs(ctx):
    from strelka_b200.api import DevIndelLoci, DevIndelReadsSample, DevSomaticIndelBatch, DevSomaticIndelChain

    sb, o = sindel_gen.case(0)[:2]
    want = sindel_gen.ox_somatic_indel(o, sb)
    got, launches, delta = _counted(ctx, lambda: ctx.somatic_indel(sb, o))
    assert got.tobytes() == want.tobytes() and (launches, delta) == (1, 1)
    db = DevSomaticIndelBatch(ctx, sb)
    assert _counted(ctx, lambda: ctx.somatic_indel_dev(db, o))[1:] == (1, 1)
    assert db.download().tobytes() == want.tobytes()

    normal, tumor, loci = G.synth(0)
    rc, linked = G.ox_link(normal, tumor, loci)
    assert rc == 0
    got, launches, delta = _counted(ctx, lambda: ctx.link_indel_reads(normal, tumor, loci))
    G.same(linked, got)
    assert (launches, delta) == (11, 11)
    dn, dt, dl = DevIndelReadsSample(ctx, normal), DevIndelReadsSample(ctx, tumor), DevIndelLoci(ctx, loci)
    got, launches, delta = _counted(ctx, lambda: ctx.link_indel_reads_dev(dn, dt, dl, int(linked.totals[0]), int(linked.totals[1])))
    G.same(linked, got)
    assert (launches, delta) == (11, 11)
    chain = DevSomaticIndelChain(ctx, dn, dt, loci)
    assert _counted(ctx, lambda: chain.run())[1:] == (13, 13)  # the link, K5b, the flag kernel
    st = linked.status[: loci.n_loci]
    want = sindel_gen.ox_somatic_indel(A.default_sindel_opts(), linked.batch(loci))
    want[st != 0] = np.zeros(1, A.SINDEL_RESULT_DT)
    want["status"] = st
    assert chain.download().tobytes() == want.tobytes()


class _LaunchLog:
    """Stands in for ctx.lib: after every call of a device entry, the launches it reported."""

    def __init__(self, ctx):
        self.ctx, self.lib, self.log = ctx, ctx.lib, []

    def __getattr__(self, name):
        fn = getattr(self.lib, name)
        if not name.endswith("_dev"):
            return fn

        def call(*args):
            rc = fn(*args)
            t = A.SxTiming()
            self.lib.sx_last_timing(self.ctx.h, C.byref(t))
            self.log.append((name, int(t.launches)))
            return rc

        return call


def _device_chain(ctx, eb, pools, raw=None):
    """DevRealignChain.run on `eb`; the launches each device entry reported, in call order, and the chain."""
    from strelka_b200.api import DevRealignChain

    chain = DevRealignChain(ctx, eb, pools, cap_alns_per_read=64, raw=raw)
    log = _LaunchLog(ctx)
    ctx.lib = log
    try:
        chain.run()
    finally:
        ctx.lib = log.lib
    return log.log, chain


# launches the K7 stages report on specgen.enum_case(1): {plan: (host K7, host K7a, chain without gates, chain with gates)}; the chain's
# entries in call order: [K7g,] K7a, K7, K7b, K1, K6, K9
K7_LAUNCHES = {
    "fast": (7, 6, [6, 7, 9, 2, 5, 5], [1, 7, 11, 9, 2, 5, 5]),
    "two_pass": (6, 6, [6, 6, 9, 2, 5, 5], [1, 7, 6, 9, 2, 5, 5]),
}


@pytest.mark.parametrize("plan", ["fast", "two_pass"])
def test_k7_chain_launches_and_outputs(ctx, plan):
    """K7g, K7a, K7, K7b, K1, K6 and K9 through their device entries (DevRealignChain) and their host entries on one batch: the launches
    each reports, and the device chain's outputs against the host entries' and the oracle's."""
    eb = specgen.enum_case(1)
    if plan == "two_pass":
        eb.opts.flags = 0
        eb.c.opts = eb.opts
    k7_host, k7a_host, chain_plain, chain_gated = K7_LAUNCHES[plan]
    want = reflib.ox_enumerate_alignments(eb)
    host, launches, delta = _counted(ctx, lambda: ctx.enumerate_alignments(eb))
    for a, b in zip(host.trimmed(), want.trimmed()):
        assert a.tobytes() == b.tobytes()
    assert (launches, delta) == (k7_host, k7_host)
    pools = B.read_pools_of(eb)
    prep, launches, delta = _counted(ctx, lambda: ctx.alignment_indels(eb, pools))
    assert (launches, delta) == (k7a_host, k7a_host)
    link, launches, delta = _counted(ctx, lambda: ctx.link_alignments(eb, host, pools.regions))
    assert (launches, delta) == (9, 9)
    lnp = reflib.ox_score(link.align_batch(pools))
    rb = B.RealignBatch(eb, host, k4_kinds=True)  # (the chain's K9 writes K4's segment kinds)
    real, launches, delta = _counted(ctx, lambda: ctx.choose_realignment(rb, lnp))
    assert (launches, delta) == (5, 5)

    log, chain = _device_chain(ctx, eb, pools)
    assert [n for _, n in log] == chain_plain, log
    n = eb.n_reads
    assert chain.prep["totals"].download(np.uint32, 1)[0] == prep.totals[0]
    assert np.array_equal(chain.prep["in_key_off"].download(np.uint32, n + 1), prep.in_key_off)
    assert np.array_equal(chain.prep["in_keys"].download(np.uint16, int(prep.totals[0])), prep.in_keys[: int(prep.totals[0])])
    for a, b in zip(chain.enum.download().trimmed(), want.trimmed()):
        assert a.tobytes() == b.tobytes()
    nS, nI = (int(x) for x in link.totals)
    L = chain.link
    assert tuple(L["totals"].download(np.uint32, 2)) == (nS, nI)
    assert L["alns"].download(A.ALN_DT, link.n_alns + 1).tobytes() == link.alns.tobytes()
    assert L["segs"].download(A.ALN_SEG_DT, nS).tobytes() == link.segs[:nS].tobytes()
    assert L["ins"].download(np.uint8, nI).tobytes() == link.ins[:nI].tobytes()
    assert chain.lnp.download(np.float64, link.n_alns).tobytes() == lnp[: link.n_alns].tobytes()
    pos, n_seg, status, seg_off, segs = chain.download_realignments()
    assert pos.tobytes() == real.pos[:n].tobytes() and n_seg.tobytes() == real.n_seg[:n].tobytes() and status.tobytes() == real.status[:n].tobytes()
    assert seg_off.tobytes() == real.seg_off[: n + 1].tobytes() and segs.tobytes() == real.segs[: int(seg_off[n])].tobytes()
    chain.free()

    # with the mapper's alignments: K7g's device entry first, its outputs against the host entry's
    gb = B.GateBatch(eb, specgen.raw_alignments_for(eb, 1))
    go, launches, delta = _counted(ctx, lambda: ctx.realign_gates(gb))
    assert (launches, delta) == (1, 1)
    log, chain = _device_chain(ctx, eb, pools, raw=gb)
    assert [n for _, n in log] == chain_gated, log
    assert log[0][0] == "sx_realign_gates_dev"
    assert chain.gates["gate"].download(np.uint8, n).tobytes() == go.gate[:n].tobytes()
    assert chain.gates["in_pos"].download(np.int32, n).tobytes() == go.in_pos[:n].tobytes()
    chain.free()


WINDOW_LAUNCHES = 59  # sx_process_window_dev on the smoke window


def test_window_pass_launches(ctx):
    """The window pass on the smoke window: its launch count, and its outputs against the digests the smoke checks."""
    import os
    import sys

    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    import refgold
    import window_workload as WW
    from strelka_b200.api import DevWindow

    win = WW.make_window(WW.load_synth(), 60, 3, qual_bits=4, ascii_reads=True)
    entry = refgold.golden()["synthetic"]["smoke"]
    assert entry["inputs"] == refgold.synthetic_inputs_digest(win)
    dw = DevWindow(ctx, win)
    _, launches, delta = _counted(ctx, dw.run)
    got = WW.window_items(win, dw.download())
    dw.free()
    assert (launches, delta) == (WINDOW_LAUNCHES, WINDOW_LAUNCHES)
    refgold.compare(got, None, entry)
