"""K6g allele_groups on the GPU: sx_link_allele_groups[_dev] against the oracle, whole arrays byte for byte; the chain
sx_score_indels_dev -> sx_indel_gl_from_records_dev against the reference's own score_indels + allele-group functions +
getVariantAlleleGroupGenotypeLhoodsForSample (tests/golden/germline_indel_ref.npz, and live where oracle/_ref is built); and the chain on a
DevWindow pass's records against the host route on the downloaded records.  The error tests pass bad arguments
only."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import allele_groups_gen as AG
import indel_reads_gen as G
import reflib
import test_allele_groups as T
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import germline_indel_leg as GL  # noqa: E402
import window_workload as WW  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


def _dev(ctx, sample, groups):
    from strelka_b200.api import DevAlleleGroups, DevIndelReadsSample

    return DevIndelReadsSample(ctx, sample), DevAlleleGroups(ctx, groups)


@pytest.mark.parametrize("i", range(len(AG.CASES)))
def test_device_matches_oracle(ctx, i):
    sample, groups = AG.case(i)
    rc, want = AG.ox_link(sample, groups)
    assert rc == 0
    AG.same(want, ctx.link_allele_groups(sample, groups))
    ds, dg = _dev(ctx, sample, groups)
    cr, cl = int(want.totals[0]), int(want.totals[1])  # exactly what the call needs
    first = ctx.link_allele_groups_dev(ds, dg, cr, cl)
    AG.same(want, first)
    AG.same(first, ctx.link_allele_groups_dev(ds, dg, cr + 100, cl + 100))  # run to run


def test_large_batch(ctx):
    """More groups than the grids have warps: 1.2e5 groups over ~2e5 ids, lists deeper than the shared-memory sort."""
    _, sample, loci = G.synthetic_case(77, n_gid=200_000, n_regions=150_000, depth=10.0, max_width=6, special=[(5000, 3, 4000)])
    rng = np.random.default_rng(77)
    groups = AG.random_groups(rng, sample, loci.n_gid, loci.gid_key, 120_000)
    rc, want = AG.ox_link(sample, groups)
    assert rc == 0 and groups.n_groups >= 100_000 and int(want.totals[0]) > 0
    ds, dg = _dev(ctx, sample, groups)
    cr, cl = B.allele_group_caps(sample, groups)
    got = ctx.link_allele_groups_dev(ds, dg, cr, cl)
    AG.same(want, got)
    AG.same(got, ctx.link_allele_groups_dev(ds, dg, cr, cl))


@pytest.mark.parametrize("seed", range(G.K6_CASES))
def test_chain_from_k6_on_the_device(seed):
    """K6 on the device for one sample, then the link and K5 without a host step (sx_indel_gl_from_records_dev), against the reference: the
    frozen answers of its own score_indels into one IndelBuffer and getVariantAlleleGroupGenotypeLhoodsForSample (and the live reference where
    oracle/_ref is built) -- every gt_lhood double and support count; the link alone on the records K6 left in HBM carries the reference's
    supporting reads and allele likelihoods.  Each sample runs on a context made with its own min_read_bp_flank."""
    from strelka_b200.api import Context, DeviceArray, DevAlleleGroups, DevGermlineIndelChain, DevIndelReadsSample, DevScoreIndelsBatch

    batches, lnps, key_gid, read_id, loci = G.k6_case(seed)
    for s in range(2):
        case, host_sample, groups, _ = T.k6_chain(seed, s)
        ctx = Context(0, AG.params_of(batches[s]))
        try:
            db = DevScoreIndelsBatch(ctx, batches[s])
            ctx.score_indels_dev(db, DeviceArray(ctx, lnps[s].nbytes + 64).upload(lnps[s]))
            sample = DevIndelReadsSample.from_score_indels(ctx, db, key_gid[s], read_id[s])
            chain = DevGermlineIndelChain(ctx, sample, groups)
            chain.run()
            got, st = chain.download()
            assert not st.any()
            linked = ctx.link_allele_groups_dev(sample, DevAlleleGroups(ctx, groups), *B.allele_group_caps(host_sample, groups))
            refs = [AG.frozen_ref_chain(f"{seed}_{s}", AG.inputs_digest(batches[s], lnps[s], read_id[s], loci, groups))]
            if AG.have_ref():
                refs.append(AG.ref_chain(batches[s], lnps[s], read_id[s], loci, groups))
            for ref in refs:
                AG.same_as_reference(linked, groups, ref, got)
        finally:
            ctx.close()


def test_chain_keeps_the_links_flags(ctx):
    from strelka_b200.api import DevGermlineIndelChain

    sample, groups = AG.case(4)
    rc, linked = AG.ox_link(sample, groups)
    st = linked.status[: groups.n_groups]
    assert rc == 0 and np.any(st & A.SX_INDEL_READS_ST_DUP_READ)
    ds, _ = _dev(ctx, sample, groups)
    chain = DevGermlineIndelChain(ctx, ds, groups)
    chain.run()
    got, got_st = chain.download()
    want = reflib.ox_indel_gl(A.default_params(), linked.batch())
    want[st != 0] = np.zeros(1, A.INDEL_RESULT_DT)  # a flagged group: its status and no result
    assert got.tobytes() == want.tobytes() and got_st.tobytes() == st.tobytes()


@pytest.mark.parametrize("seed", [3, 5, 11])
def test_chain_on_a_window_pass(ctx, seed):
    """A DevWindow pass's records through DevIndelReadsSample.from_window and the chain, against the host route on the downloaded records
    (host builder + K5's host entry)."""
    from strelka_b200.api import DevGermlineIndelChain, DevIndelReadsSample, DevWindow

    w = WW.make_window(WW.load_synth(), 300, seed)
    groups = GL.window_groups(w, seed)
    assert groups.n_groups > 0
    dw = DevWindow(ctx, w)
    dw.run()
    sample = DevIndelReadsSample.from_window(ctx, dw, np.arange(w.n_keys, dtype=np.uint32), None, GL.SW.non_ambig_of(w))
    chain = DevGermlineIndelChain(ctx, sample, groups)
    chain.run()
    got, st = chain.download()
    want, want_st, linked = GL.host_route(ctx, dw, groups)
    assert int(linked.totals[0]) > 0 and np.any(np.diff(groups.allele_off) == 2)
    assert got.tobytes() == want.tobytes() and st.tobytes() == want_st.tobytes()
    chain.run()
    assert chain.download()[0].tobytes() == got.tobytes()
    dw.free()


def test_capacity_bad_arguments_and_empty(ctx):
    from strelka_b200.api import DevAlleleGroups, DevGermlineIndelChain, SxError

    sample, groups = AG.case(0)
    rc, want = AG.ox_link(sample, groups)
    ds, dg = _dev(ctx, sample, groups)
    for cr, cl in ((int(want.totals[0]) - 1, int(want.totals[1])), (int(want.totals[0]), int(want.totals[1]) - 1)):
        for call in (lambda: ctx.link_allele_groups(sample, groups, cr, cl), lambda: ctx.link_allele_groups_dev(ds, dg, cr, cl)):
            with pytest.raises(SxError) as e:
                call()
            assert e.value.code == A.SX_ERR_CAPACITY and np.array_equal(e.value.totals, want.totals)
    lib = ctx.lib
    out = B.AlleleGroupReadsOut(groups.n_groups, int(groups.allele_off[-1]), *B.allele_group_caps(sample, groups))
    args = [C.byref(sample.c), C.byref(groups.c), C.byref(out.c)]
    for k in range(3):
        assert lib.sx_link_allele_groups(ctx.h, *(None if j == k else a for j, a in enumerate(args)), None) == A.SX_ERR_ARG
    for bad in T.bad_groups(groups):
        with pytest.raises(SxError) as e:
            ctx.link_allele_groups(sample, bad)
        assert e.value.code == A.SX_ERR_ARG
        # the device entries check the groups themselves
        with pytest.raises(SxError) as e:
            ctx.link_allele_groups_dev(ds, DevAlleleGroups(ctx, bad), *B.allele_group_caps(sample, groups))
        assert e.value.code == A.SX_ERR_ARG
        with pytest.raises(SxError) as e:
            DevGermlineIndelChain(ctx, ds, bad).run()
        assert e.value.code == A.SX_ERR_ARG
    no_contrast_ids = B.AlleleGroups.from_lists([groups.group(g)[0] for g in range(groups.n_groups)], [groups.group(g)[1] for g in range(groups.n_groups)],
                                                groups.ploidy, groups.gid_key)
    no_contrast_ids.c.contrast_gid = None
    assert lib.sx_link_allele_groups(ctx.h, C.byref(sample.c), C.byref(no_contrast_ids.c), C.byref(out.c), None) == A.SX_ERR_ARG
    AG.same(want, ctx.link_allele_groups(sample, groups))  # the context stays usable
    none = B.AlleleGroups.from_lists([], [], np.zeros(0, np.uint8), groups.gid_key)
    o = ctx.link_allele_groups(sample, none)
    assert not o.totals.any() and not o.read_off.any()
    chain = DevGermlineIndelChain(ctx, ds, none)
    chain.run()
    e_n, e_t, e_l = G.synthetic_case(50, n_regions=1, depth=0.0)
    eg = B.AlleleGroups.from_lists([[int(e_l.gid[0])], [int(e_l.gid[1]), int(e_l.gid[2])]], [[], [int(e_l.gid[3])]], [2, 1], e_l.gid_key)
    AG.same(AG.ox_link(e_t, eg)[1], ctx.link_allele_groups(e_t, eg))
