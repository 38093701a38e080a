"""The somatic window pass on the GPU (sx_process_somatic_window_dev): two samples of one window through the realignment / pile-up chain, K2b,
the link, K5b and the two record lists in one call.

Two-sample windows are made from the seeded window cases (window_check.window_case) and from the bench's synthetic windows: the reads with an
indel in their alignment go to the tumor sample with every other one of the rest, and tumor-only SNVs are injected, so that somatic calls occur.
Compared against
  - the existing entries on the same inputs (no reference needed): two DevWindow passes, sx_site_gl_somatic_dev on their columns,
    DevSomaticIndelChain on DevIndelReadsSample.from_window, and the host filter -- byte for byte;
  - the reference, where oracle/_ref is built: each sample through window_check.reference_window, the sites through reflib.ref_somatic on the
    reference's columns, the indels through the reference's records -> the oracle link -> sindel_gen.ref_somatic_indel.
The error tests pass bad arguments only."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import indel_reads_gen as G
import refgold
import reflib
import sindel_gen
import window_check as W
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import somatic_window_leg as SW  # noqa: E402
import window_workload as WW  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


def _opts():
    o = A.default_sindel_opts()
    o.useTier2Evidence = 0
    return o


def split_enum(eb, gb, flags, mapq, keep, snv_every=0, seed=0):
    """a single-region window case restricted to the reads in `keep` (read-buffer order kept), as (eb, gb, WindowBatch); with snv_every, the
    reads whose mapper's alignment is one match segment read the next base at every snv_every-th position"""
    rng = np.random.default_rng(seed)
    win = []
    for k in range(eb.n_keys):
        key = eb.keys[k]
        ins = bytes(eb.ins_pool[int(eb.ins_off[k]) : int(eb.ins_off[k + 1])]).decode()
        fl, hap = int(key["flags"]), eb.key_hap[k] if eb.has_hap else None
        win.append(B.EnumKeySpec(int(key["pos"]), int(key["del_len"]), ins, mismatch=int(key["type"]) == A.SX_INDEL_TYPE_MISMATCH, candidate=bool(fl & 1),
                                 not_discovered=bool(fl & 2), forced=bool(fl & 4), active_region=int(hap["active_region_id"]) if hap is not None else -1,
                                 hap_ids=tuple(int(x) for x in hap["haplotype_id"]) if hap is not None else (0, 0, 0, 0), bypass=int(hap["bypass_mask"]) if hap is not None else 0))
    ref = bytes(eb.ref_pool[int(eb.ref_off[0]) : int(eb.ref_off[1])]).decode()
    ref_begin = int(eb.ref_begin[0])
    sel = np.nonzero(keep)[0]
    reads, raw = [], []
    for r in sel:
        seq = list(bytes(eb.read_pool[int(eb.read_off[r]) : int(eb.read_off[r + 1])]).decode())
        (pos, _), raw_path = W.raw_of(gb, r)
        if snv_every and len(raw_path) == 1 and raw_path[0][0] == "M":
            for p in range(ref_begin + snv_every // 2, ref_begin + len(ref), snv_every):
                i = p - pos
                if 0 <= i < len(seq) and ref[p - ref_begin] in "ACGT" and rng.random() < 0.7:
                    seq[i] = "ACGT"[("ACGT".index(ref[p - ref_begin]) + 1) % 4]
        al = (int(eb.in_pos[r]), [(B.AP_CHAR[int(s["kind"])], int(s["len"])) for s in eb.in_segs[int(eb.in_seg_off[r]) : int(eb.in_seg_off[r + 1])]])
        use = [int(x) for x in eb.use_keys[int(eb.use_key_off[r]) : int(eb.use_key_off[r + 1])]]
        reads.append(B.EnumReadSpec("".join(seq), al[0], al[1], use))
        raw.append((pos, raw_path))
    eb1 = B.EnumBatch([(ref, ref_begin, (int(eb.realign_begin[0]), int(eb.realign_end[0])), win, reads)], eb.opts, strict=False)
    gb1 = B.GateBatch(eb1, raw)
    pad = lambda x: np.concatenate([np.asarray(x)[sel], [0]]).astype(np.uint8)
    w = B.WindowBatch.from_enum(eb1, gb1, B.read_pools_of(eb1), read_flags=pad(flags), mapq=pad(mapq), do_site_gl=False)
    return eb1, gb1, w


def case_windows(case):
    """(normal, tumor) as (eb, gb, WindowBatch) of every single-region window of seeded case `case` with reads in both samples"""
    for eb, gb, flags, mapq in W.window_case(case):
        n = eb.n_reads
        ind = np.array([any(t in "ID" for t, _ in W.raw_of(gb, r)[1]) for r in range(n)], bool)
        tumor = ind | ((np.cumsum(~ind) % 2 == 0) & ~ind)
        if tumor.all() or not tumor.any():
            continue
        yield split_enum(eb, gb, flags, mapq, ~tumor), split_enum(eb, gb, flags, mapq, tumor, snv_every=7, seed=case)


def composed_check(ctx, normal, tumor, loci, key_gid, forced, opts):
    """the one-call pass against the composition it replaces, byte for byte; returns the pass's download"""
    from strelka_b200.api import DevSomaticWindow

    sw = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced, opts=opts)
    stage_ms = sw.run()
    assert set(stage_ms) == set(A.SX_SWIN_STAGE_NAMES)
    got = sw.download()
    first = {k: (v.tobytes() if isinstance(v, np.ndarray) else v) for k, v in got.items() if k not in ("normal", "tumor")}
    sw.run()  # run to run: the same bytes
    again = sw.download()
    for k, v in first.items():
        assert (again[k].tobytes() if isinstance(again[k], np.ndarray) else again[k]) == v, k
    for s in ("normal", "tumor"):
        for k, v in got[s].items():
            assert np.asarray(again[s][k]).tobytes() == np.asarray(v).tobytes(), (s, k)
    sw.free()
    comp = SW.Composed(ctx, normal, tumor, loci, key_gid, forced)
    comp.run(opts)
    d, snv, snv_rec, indel, indel_rec = comp.results(opts)
    comp.free()
    for s, (name, w) in enumerate(zip(("normal", "tumor"), (normal, tumor))):
        for k, v in d[s].items():
            if k == "recs":  # (the slots past a read's n_rec are never written)
                v, g = (_used_recs(x, w) for x in (d[s], got[name]))
            else:
                g = got[name][k]
            assert np.asarray(g).tobytes() == np.asarray(v).tobytes(), (name, k)
    assert got["site_snv"].tobytes() == snv.tobytes()
    assert got["indel"].tobytes() == indel.tobytes()
    assert got["snv_calls"].tobytes() == snv_rec.tobytes()
    assert got["indel_calls"].tobytes() == indel_rec.tobytes()
    assert list(got["totals"][:2]) == [snv_rec.size, indel_rec.size]
    return got


def _used_recs(d, w):
    ro = w.a["rec_off"]
    return b"".join(d["recs"][int(ro[r]) : int(ro[r]) + int(d["n_rec"][r])].tobytes() for r in range(w.n_reads))


def _sample_items(d, w, gb, threw):
    """a sample's per-read and column outputs as window_check's comparison items"""
    n = w.n_reads
    submapped = (w.a["read_flags"][:n] & A.SX_PRF_TIER1OR2) == 0
    seg_off, segs = d["best_seg_off"], d["best_segs"]
    reads = []
    for r in range(n):
        if submapped[r] or r in threw:
            continue
        got = (int(d["best_pos"][r]), W.cigar_of(segs[int(seg_off[r]) : int(seg_off[r]) + int(d["best_n_seg"][r])]))
        o, k = int(w.a["rec_off"][r]), int(d["n_rec"][r])
        reads.append((r, bool(int(d["realign_status"][r]) & A.SX_REALIGN_ST_REALIGNED), got, k, d["recs"][o : o + k].tobytes()))
    it = {"reads": reads}
    it.update(zip(W.COL_NAMES, (d["site_off"], d["calls"], d["t2_off"], d["t2_calls"], d["n_spandel"], d["n_submapped"])))
    return it


SNV_FIELDS = ("ref_gt", "snv_tier", "snv_from_ntype_tier", "ntype", "max_gt", "qphred", "from_ntype_qphred", "normal_alt_id", "tumor_alt_id")
INDEL_FIELDS = ("is_output", "qphred", "from_ntype_qphred", "max_gt", "sindel_tier", "sindel_from_ntype_tier", "is_overlap")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "somatic_window_ref_digests.json")
CASES = (0, 2, 3, 4, 5)  # (case 1 has no window with reads in both samples)


def case_inputs(case):
    """the seeded two-sample windows of case `case`: (key, normal, tumor, loci, key_gid, forced); forced positions, and forced loci whose lists
    are empty (ids no read names), among them"""
    for i, (normal, tumor) in enumerate(case_windows(case)):
        w = normal[2]
        loci, key_gid = SW.somatic_loci(w, case)
        forced = SW.forced_positions(w, case)
        forced[:: max(1, w.n_sites // 3)] = 1
        yield f"{case}.{i}", normal, tumor, loci, key_gid, forced


def inputs_digest(normal, tumor, loci, forced):
    return refgold.inputs_digest(normal[2].a["seq4"], tumor[2].a["seq4"], normal[2].a["raw_pos"], tumor[2].a["raw_pos"], loci.gid, loci.is_forced_output, loci.err_idx, forced)


def somatic_items(sample_items, site_snv, indel, status, snv_calls, indel_calls):
    """what is compared with the reference: each sample's reads and columns (window_check's items), K2b's defined fields where the model ran,
    K5b's where the link left the locus unflagged, the link's status, and the two record lists' positions / depths / loci"""
    it = {f"{name}.{k}": v for name, si in sample_items.items() for k, v in si.items()}
    m = site_snv["is_computed"] == 1
    it["snv.is_computed"] = site_snv["is_computed"]
    for f in SNV_FIELDS:
        it["snv." + f] = site_snv[f][m]
    it["snv.strandBias"] = site_snv["strandBias"][m].view(np.uint32)
    ok = status == 0
    it["indel.status"] = status
    for f in INDEL_FIELDS:
        it["indel." + f] = indel[f][ok]
    it["snv_calls.pos"], it["snv_calls.n_calls"], it["indel_calls.locus"] = snv_calls["pos"], snv_calls["n_calls"].reshape(-1), indel_calls["locus"]
    return it


def device_items(got, samples):
    return somatic_items({name: _sample_items(got[name], w, gb, []) for name, (eb, gb, w) in zip(("normal", "tumor"), samples)}, got["site_snv"], got["indel"],
                         got["indel"]["status"], got["snv_calls"], got["indel_calls"])


def reference_items(samples, loci, key_gid, forced, opts):
    """the window through the reference stage by stage (oracle/_ref): each sample through window_check.reference_window, the sites through
    the reference's position_somatic_snv_call on its two column sets, the indels through its records -> the oracle link (pinned to the
    reference's read_path_lnp maps) -> its get_somatic_indel, the record lists by its is_output and empty-list rules.  None where the
    reference threw on a read of the window (its process would have stopped there: nothing to compare)."""
    exps = []
    for eb, gb, w in samples:
        exp = W.reference_window(eb, gb, w)
        if exp["cols"] is None or (exp["status"] == 2).any():
            return None
        exps.append(exp)
    per_sample = {}
    for (eb, gb, w), exp, name in zip(samples, exps, ("normal", "tumor")):
        want = W.reference_items(exp, w)
        per_sample[name] = {k: v for k, v in want.items() if k in W.COL_NAMES or k == "reads"}  # (no germline site model in the somatic pass)
    w0 = samples[0][2]
    ref_base = np.frombuffer(bytes(w0.a["ref"][w0.report_begin - w0.ref_begin : w0.report_end - w0.ref_begin]), np.uint8).copy()
    pbs = [B.PileupBatch(e["cols"][0].copy(), np.concatenate([e["cols"][1], np.zeros(16, np.uint16)]), ref_base, None) for e in exps]
    want_snv = reflib.ref_somatic(A.default_params(), pbs[0], pbs[1], forced)
    irs = []
    for (eb, gb, w), exp in zip(samples, exps):
        n = w.n_reads
        n_rec = np.asarray(exp["n_rec"], np.uint32).copy()
        n_rec[:n][(w.a["read_flags"][:n] & A.SX_PRF_TIER1OR2) == 0] = 0
        sb = type("S", (), dict(n_regions=w.n_regions, n_reads=n, n_keys=w.n_keys, region_read_off=w.a["region_read_off"], region_key_off=w.a["region_key_off"],
                                rec_off=w.a["rec_off"], read_len=w.a["read_len"], non_ambig=SW.non_ambig_of(w), read_flags=w.a["read_flags"]))
        irs.append(B.IndelReadsSample(sb, exp["recs"], n_rec, key_gid))
    rc, linked = G.ox_link(irs[0], irs[1], loci)
    assert rc == 0
    st = linked.status[: loci.n_loci]
    want_indel = sindel_gen.ref_somatic_indel(opts, linked.batch(loci))
    depth = [np.diff(e["cols"][0].astype(np.int64)) for e in exps]
    snv_rec, indel_rec = SW.host_records(want_snv, forced, ref_base, depth[0], depth[1], w0.report_begin, want_indel, loci, st, linked.read_off)
    return somatic_items(per_sample, want_snv, want_indel, st, snv_rec, indel_rec)


def have_reference() -> bool:
    return reflib.have_ref() and G.have_ref() and sindel_gen.have_ref()


def records_only_check(ctx, normal, tumor, loci, key_gid, forced, opts, want, **kw):
    """the pass with every output but the record lists left to the context (out.sample[s], site_snv, indel NULL: the normal sample's columns
    and records live in the SX_SLOT_SWIN_* bank across the tumor sample's pass) gives the records and totals of the run with every output"""
    from strelka_b200.api import DevSomaticWindow

    sw = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced, opts=opts, records_only=True, **kw)
    assert not any(getattr(sw.out.sample[s], k) for s in (0, 1) for k in ("recs", "n_rec")) and not sw.out.sample[0].cols.calls and not sw.out.site_snv
    sw.run()
    got = sw.download()
    sw.free()
    for k in ("snv_calls", "indel_calls", "totals"):
        assert got[k].tobytes() == want[k].tobytes(), k


@pytest.mark.parametrize("case", CASES)
def test_window_cases(ctx, case):
    """every window of a seeded case: the one call against the composed route and in records-only form, and against the reference where
    oracle/_ref is built, else against the reference's frozen digests (tests/golden/make_somatic_window_golden.py)"""
    import json

    with open(GOLDEN) as f:
        gold = json.load(f)["window"]
    opts = _opts()
    n_windows = n_ref = n_forced_empty = 0
    for key, normal, tumor, loci, key_gid, forced in case_inputs(case):
        w = normal[2]
        got = composed_check(ctx, w, tumor[2], loci, key_gid, forced, opts)
        records_only_check(ctx, w, tumor[2], loci, key_gid, forced, opts, got)
        n_windows += 1
        # ids no read names: empty lists in both samples.  A forced one is a record; an unforced one is not -- K5b answers QSI 0 on empty lists,
        # so on these inputs the device's empty-list skip (strelka_pos_processor.cpp:324-327) and the QSI rule agree.
        extra = np.nonzero(loci.gid >= w.n_keys)[0]
        fe = extra[loci.is_forced_output[extra] != 0]
        assert set(fe) <= set(got["indel_calls"]["locus"]) and not set(extra[loci.is_forced_output[extra] == 0]) & set(got["indel_calls"]["locus"])
        assert not got["indel"]["qphred"][extra].any()
        n_forced_empty += fe.size
        entry = gold.get(key)
        if have_reference():
            want = reference_items((normal, tumor), loci, key_gid, forced, opts)
            if want is None:
                continue
        else:
            assert entry is not None and entry["inputs"] == inputs_digest(normal, tumor, loci, forced), (key, "regenerate tests/golden/somatic_window_ref_digests.json")
            if not entry["compared"]:
                continue
            want = None
        refgold.compare(device_items(got, (normal, tumor)), want, entry)
        n_ref += 1
    assert n_windows > 0 and n_ref > 0 and n_forced_empty > 0


@pytest.mark.parametrize("tier2", [False, True])
def test_synthetic_window(ctx, tier2):
    """a bench-shaped window split in two: somatic calls with QSS and QSI occur, and the one call equals the composed route byte for byte"""
    from strelka_b200.api import DevSomaticWindow

    w = WW.make_window(WW.load_synth(), 400, 11)
    normal, tumor, loci, key_gid, forced = SW.two_sample_window(w, 11)
    opts = _opts()
    assert tumor.n_reads > normal.n_reads  # (the tumor sample's pass grows the buffers the normal sample's results must not share)
    if not tier2:
        got = composed_check(ctx, normal, tumor, loci, key_gid, forced, opts)
        records_only_check(ctx, normal, tumor, loci, key_gid, forced, opts, got)
    else:  # (the composed route's K2b reads tier1 only: with tier2 evidence the pass is checked against K2b on both tiers here)
        for x in (normal, tumor):  # every fourth read a tier2 mapping
            x.a["read_flags"][: x.n_reads : 4] &= np.uint8(~A.SX_PRF_TIER1 & 0xFF)
        sw = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced, use_tier2=True)
        sw.run()
        got = sw.download()
        n, t = got["normal"], got["tumor"]
        assert int(t["t2_off"][-1]) > 0
        ref_base = np.ascontiguousarray(normal.a["ref"][normal.report_begin - normal.ref_begin : normal.report_end - normal.ref_begin])
        pb = [B.PileupBatch(x["site_off"], x["calls"], ref_base, None, x["t2_off"], x["t2_calls"]) for x in (n, t)]
        assert ctx.site_gl_somatic(pb[0], pb[1], forced).tobytes() == got["site_snv"].tobytes()
        sw.free()
        records_only_check(ctx, normal, tumor, loci, key_gid, forced, None, got, use_tier2=True)
        # the indels with tier2 evidence: DevSomaticIndelChain on the records of two DevWindow passes (K6 does not read the pile-up options)
        o2 = A.default_sindel_opts()
        o2.useTier2Evidence = 1
        comp = SW.Composed(ctx, normal, tumor, loci, key_gid, forced)
        comp.run(o2)
        assert comp.chain.download().tobytes() == got["indel"].tobytes()
        comp.free()
    assert (got["site_snv"]["qphred"] != 0).sum() > 0 and (got["indel"]["qphred"] != 0).sum() > 0
    assert got["totals"][0] > 0 and got["totals"][1] > 0


def test_empty_windows(ctx):
    """no reads in either sample, and no loci: the pass runs and reports nothing"""
    from strelka_b200.api import DevSomaticWindow

    w = WW.make_window(WW.load_synth(), 40, 3)
    none = np.zeros(w.n_reads, bool)
    e = SW.split_window(w, none)
    loci, key_gid = SW.somatic_loci(w, 3)
    sw = DevSomaticWindow(ctx, e, e, loci, [key_gid, key_gid], records_only=True)  # (a window without reads has no per-read output to download)
    sw.run()
    got = sw.download()
    assert got["snv_calls"].size == 0 and int(got["totals"][0]) == 0
    assert set(got["indel_calls"]["locus"]) <= set(np.nonzero(loci.is_forced_output)[0])
    sw.free()
    n, t, _, _, _ = SW.two_sample_window(w, 3)
    no_loci = B.IndelLoci(loci.gid[:0], loci.key[:0], loci.is_forced_output[:0], loci.err_idx[:0], loci.gid_key, loci.err_prob)
    sw = DevSomaticWindow(ctx, n, t, no_loci, [key_gid, key_gid])
    sw.run()
    got = sw.download()
    assert got["indel"].size == 0 and got["indel_calls"].size == 0 and int(got["totals"][1]) == 0
    sw.free()


def test_capacities(ctx):
    """a record array one short: SX_ERR_CAPACITY with the totals of both lists, and the records that fit"""
    from strelka_b200.api import DevSomaticWindow, SxError

    w = WW.make_window(WW.load_synth(), 200, 5)
    normal, tumor, loci, key_gid, forced = SW.two_sample_window(w, 5)
    full = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced)
    full.run()
    want = full.download()
    full.free()
    n_snv, n_indel = int(want["totals"][0]), int(want["totals"][1])
    assert n_snv > 1 and n_indel > 1
    for caps in ((n_snv - 1, None), (None, n_indel - 1)):
        sw = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced, cap_snv_calls=caps[0], cap_indel_calls=caps[1])
        with pytest.raises(SxError) as e:
            sw.run()
        assert e.value.code == A.SX_ERR_CAPACITY and np.array_equal(e.value.totals, want["totals"])
        got = sw.download()
        k, name = (0, "snv_calls") if caps[0] is not None else (1, "indel_calls")
        assert got[name].tobytes() == want[name][: caps[k]].tobytes()
        sw.free()


def test_bad_arguments(ctx):
    """each SX_ERR_ARG condition of the entry; the context stays usable"""
    from strelka_b200.api import DevSomaticWindow, SxError

    w = WW.make_window(WW.load_synth(), 40, 9)
    normal, tumor, loci, key_gid, forced = SW.two_sample_window(w, 9)
    sw = DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced)
    lib = ctx.lib
    assert lib.sx_process_somatic_window_dev(ctx.h, None, C.byref(sw.out), None) == A.SX_ERR_ARG
    assert lib.sx_process_somatic_window_dev(ctx.h, C.byref(sw.c), None, None) == A.SX_ERR_ARG

    def bad(edit_batch=None, edit_out=None):
        b = A.SxSomaticWindowBatch.from_buffer_copy(sw.c)
        o = A.SxSomaticWindowOut.from_buffer_copy(sw.out)
        if edit_batch:
            edit_batch(b)
        if edit_out:
            edit_out(o)
        return lib.sx_process_somatic_window_dev(ctx.h, C.byref(b), C.byref(o), None)

    def setf(path, value):
        def f(x):
            obj = x
            for p in path[:-1]:
                obj = obj[p] if isinstance(p, int) else getattr(obj, p)
            setattr(obj, path[-1], value)
        return f

    cases = [
        setf(("sample", 0, "do_site_gl"), 1),
        setf(("sample", 1, "do_site_gl"), 1),
        setf(("sample", 1, "report_begin"), normal.report_begin + 1),
        setf(("sample", 1, "report_end"), normal.report_end - 1),
        setf(("sample", 1, "ref_begin"), normal.ref_begin - 16),
        setf(("sample", 1, "pileup_opts", "useTier2Evidence"), 1),
        setf(("sindel_opts", "useTier2Evidence"), 1),
        lambda b: (setf(("sample", 0, "pileup_opts", "useTier2Evidence"), 1)(b), setf(("sample", 1, "pileup_opts", "useTier2Evidence"), 1)(b)),
        setf(("n_err",), 0),
        setf(("loci", "gid"), None),
    ]
    for edit in cases:
        assert bad(edit_batch=edit) == A.SX_ERR_ARG
    kg = lambda b: b.key_gid.__setitem__(0, None)
    assert bad(edit_batch=kg) == A.SX_ERR_ARG
    for s in (0, 1):
        assert bad(edit_out=setf(("sample", s, "site_gl"), sw.obufs["site_snv"].ptr)) == A.SX_ERR_ARG
        assert bad(edit_out=setf(("sample", s, "variant_sites"), sw.obufs["snv_calls"].ptr)) == A.SX_ERR_ARG
    sw.run()  # the context stays usable
    assert sw.download()["totals"][0] > 0
    sw.free()
