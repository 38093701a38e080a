"""K6b indel_reads on the GPU: sx_link_indel_reads[_dev] against the oracle, whole arrays byte for byte, and the chain
sx_score_indels_dev -> sx_somatic_indel_from_records_dev against the frozen answers of the reference's own score_indels (both samples,
one IndelBuffer) + get_somatic_indel, and against the live reference where oracle/_ref is built.  The error tests pass bad arguments only."""
import ctypes as C

import numpy as np
import pytest

import indel_reads_gen as G
import sindel_gen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


def _dev(ctx, normal, tumor, loci):
    from strelka_b200.api import DevIndelLoci, DevIndelReadsSample

    return DevIndelReadsSample(ctx, normal), DevIndelReadsSample(ctx, tumor), DevIndelLoci(ctx, loci)


@pytest.mark.parametrize("i", range(len(G.SYNTH_CASES)))
def test_device_matches_oracle(ctx, i):
    normal, tumor, loci = G.synth(i)
    rc, want = G.ox_link(normal, tumor, loci)
    assert rc == 0
    G.same(want, ctx.link_indel_reads(normal, tumor, loci))
    assert ctx.timing().launches == 11
    dn, dt, dl = _dev(ctx, normal, tumor, loci)
    cr, ca = int(want.totals[0]), int(want.totals[1])  # exactly what the batch needs
    first = ctx.link_indel_reads_dev(dn, dt, dl, cr, ca)
    G.same(want, first)
    G.same(first, ctx.link_indel_reads_dev(dn, dt, dl, cr + 100, ca + 100))  # run to run


def test_large_batch(ctx):
    """More loci than the grids have warps and more reads than they have threads: 1.2e5 loci, ~1e7 records in use."""
    normal, tumor, loci = G.synthetic_case(77, n_gid=200_000, n_regions=180_000, depth=14.0, max_width=9, locus_frac=0.6, special=[(5000, 3, 4000), (9000, 28, 500)])
    assert loci.n_loci >= 100_000 and G.caps(normal, tumor, loci)[0] > 9_000_000
    rc, want = G.ox_link(normal, tumor, loci)
    assert rc == 0 and np.any(want.status & A.SX_SINDEL_ST_CAP) and np.diff(want.read_off).max() > G.SMEM_SORT
    dn, dt, dl = _dev(ctx, normal, tumor, loci)
    cr, ca = G.caps(normal, tumor, loci)
    got = ctx.link_indel_reads_dev(dn, dt, dl, cr, ca)
    G.same(want, got)
    G.same(got, ctx.link_indel_reads_dev(dn, dt, dl, cr, ca))


@pytest.mark.parametrize("seed", range(G.K6_CASES))
def test_chain_from_k6_on_the_device(ctx, seed):
    """K6 on the device for both samples on ONE context (each DevScoreIndelsBatch owns its record arrays), then the link and K5b without
    a host step: the results are the oracles' chain's, whole records."""
    from strelka_b200.api import DeviceArray, DevIndelLoci, DevIndelReadsSample, DevScoreIndelsBatch, DevSomaticIndelChain

    batches, lnps, key_gid, read_id, loci = G.k6_case(seed)
    samples = []
    for s in range(2):
        db = DevScoreIndelsBatch(ctx, batches[s])
        ctx.score_indels_dev(db, DeviceArray(ctx, lnps[s].nbytes + 64).upload(lnps[s]))
        samples.append(DevIndelReadsSample.from_score_indels(ctx, db, key_gid[s], read_id[s]))
    chain = DevSomaticIndelChain(ctx, samples[0], samples[1], loci)
    o = A.default_sindel_opts()
    chain.run(o)
    got = chain.download()
    # the link alone on the records K6 left in HBM: the reference buffer's read_path_lnp maps, byte for byte
    cr, ca = sum(b.n_rec_slots for b in batches), A.SX_SINDEL_MAX_ALTS * loci.n_loci
    linked = ctx.link_indel_reads_dev(samples[0], samples[1], DevIndelLoci(ctx, loci), cr, ca)
    ref, maps = G.frozen_ref_chain(seed, G.inputs_digest(batches, lnps, key_gid, read_id, loci))
    G.same_as_maps(linked, maps, loci)
    sb = linked.batch(loci)
    sindel_gen.compare_to_reference(got, ref, sb, o)
    assert got.tobytes() == sindel_gen.ox_somatic_indel(o, sb).tobytes()
    if G.have_ref():
        live, live_maps = G.ref_chain(batches, lnps, read_id, loci, o)
        G.same_as_maps(linked, live_maps, loci)
        sindel_gen.compare_to_reference(got, live, sb, o)


def test_chain_keeps_the_links_flags(ctx):
    from strelka_b200.api import DevSomaticIndelChain

    normal, tumor, loci = G.synth(6)
    rc, linked = G.ox_link(normal, tumor, loci)
    st = linked.status[: loci.n_loci]
    assert rc == 0 and np.any(st & A.SX_SINDEL_ST_CAP) and np.any(st & A.SX_INDEL_READS_ST_DUP_READ)
    dn, dt, _ = _dev(ctx, normal, tumor, loci)
    chain = DevSomaticIndelChain(ctx, dn, dt, loci)
    chain.run()
    got = chain.download()
    want = sindel_gen.ox_somatic_indel(A.default_sindel_opts(), linked.batch(loci))
    want[st != 0] = np.zeros(1, A.SINDEL_RESULT_DT)  # a flagged locus: its status and no result
    want["status"] = st
    assert got.tobytes() == want.tobytes()


def test_capacity_bad_arguments_and_the_empty_batch(ctx):
    from strelka_b200.api import SxError

    normal, tumor, loci = G.synth(0)
    rc, want = G.ox_link(normal, tumor, loci)
    dn, dt, dl = _dev(ctx, normal, tumor, loci)
    for cr, ca in ((int(want.totals[0]) - 1, int(want.totals[1])), (int(want.totals[0]), int(want.totals[1]) - 1)):
        for call in (lambda: ctx.link_indel_reads(normal, tumor, loci, cr, ca), lambda: ctx.link_indel_reads_dev(dn, dt, dl, cr, ca)):
            with pytest.raises(SxError) as e:
                call()
            assert e.value.code == A.SX_ERR_CAPACITY and np.array_equal(e.value.totals, want.totals)
    lib, out = ctx.lib, B.IndelReadsOut(loci.n_loci, *G.caps(normal, tumor, loci))
    args = [C.byref(normal.c), C.byref(tumor.c), C.byref(loci.c), C.byref(out.c)]
    for k in range(4):
        assert lib.sx_link_indel_reads(ctx.h, *(None if j == k else a for j, a in enumerate(args)), None) == A.SX_ERR_ARG
    unsorted = B.IndelLoci(loci.gid[::-1], loci.key[::-1], loci.is_forced_output, loci.err_idx, loci.gid_key, loci.err_prob)
    past = B.IndelReadsSample(normal, normal.recs, normal.n_rec, np.full(normal.n_keys, loci.n_gid, np.uint32), normal.read_id)
    recs = normal.recs.copy()
    recs["key"] = 65535  # no window is that long
    outside = B.IndelReadsSample(normal, recs, normal.n_rec, normal.key_gid, normal.read_id)
    for n_, l_ in ((normal, unsorted), (past, loci), (outside, loci)):
        with pytest.raises(SxError) as e:
            ctx.link_indel_reads(n_, tumor, l_)
        assert e.value.code == A.SX_ERR_ARG
    # the device entries check the loci's order themselves: an unsorted or repeated id is an error there too, not a race
    repeated = B.IndelLoci(np.maximum(loci.gid, loci.gid[1]), loci.key, loci.is_forced_output, loci.err_idx, loci.gid_key, loci.err_prob)
    for l_ in (unsorted, repeated):
        with pytest.raises(SxError) as e:
            ctx.link_indel_reads_dev(dn, dt, _dev(ctx, normal, tumor, l_)[2], *G.caps(normal, tumor, loci))
        assert e.value.code == A.SX_ERR_ARG
    out.c.reads = None
    assert lib.sx_link_indel_reads(ctx.h, *args, None) == A.SX_ERR_ARG
    G.same(want, ctx.link_indel_reads(normal, tumor, loci))  # the context stays usable
    none = B.IndelLoci(loci.gid[:0], loci.key[:0], loci.is_forced_output[:0], loci.err_idx[:0], loci.gid_key, loci.err_prob)
    o = ctx.link_indel_reads(normal, tumor, none)
    assert not o.totals.any() and not o.read_off.any()
    e_n, e_t, e_l = G.synthetic_case(50, n_regions=1, depth=0.0)
    G.same(G.ox_link(e_n, e_t, e_l)[1], ctx.link_indel_reads(e_n, e_t, e_l))
