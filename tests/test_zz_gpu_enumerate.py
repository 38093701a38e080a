"""GPU parity of K7 enumerate_alignments (SURVEY 8a row a3 / 8f3): the CUDA kernels through the C ABI (host-buffer entry and
device-resident entry) against the CPU oracle (oracle/enumerate_oracle.cpp), the frozen output of the reference's own
getCandidateAlignments (tests/golden/enumerate_ref.npz) and, where oracle/_ref/libstrelka_ref.so travelled, the reference itself.
Every field is an integer: bit-exact."""
import os

import numpy as np
import pytest

import reflib
import specgen
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

# This file sorts after every other test file on purpose: K7 / K7b had not run on a GPU when this was written (the round's GPU
# minutes were spent), so under `pytest -x` a first-run failure here must not mask the parity tests of the measured kernels; the
# timeout (pytest-timeout, thread method: the process is ended even if a kernel never returns) bounds a runaway search.
pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method="thread")]
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD_NAMES = ("aln_off", "status", "aln_pos", "aln_seg_off", "segs", "aln_key_off", "aln_keys", "lead", "trail")


@pytest.fixture(scope="module")
def ctx():
    from strelka_b200.api import Context

    c = Context(0)
    yield c
    c.close()


def _same(want: B.EnumOut, got: B.EnumOut):
    for name, x, y in zip(GOLD_NAMES, want.trimmed(), got.trimmed()):
        assert x.tobytes() == y.tobytes(), name


def _big_opts(opts):
    opts.max_alns_per_read = 6000
    return opts


@pytest.mark.parametrize("case", range(24))
def test_k7_enumerate_alignments(ctx, case):
    eb = specgen.enum_case(case)
    _big_opts(eb.opts)
    eb.c.opts = eb.opts
    cap = eb.n_reads * 6000 + 64
    got = ctx.enumerate_alignments(eb, cap_alns=cap)
    assert ctx.timing().launches in (7, 8)  # the default launch plan: frame count, local tier, one or two arena tiers, 3 scan kernels, gather
    _same(reflib.ox_enumerate_alignments(eb, cap_alns=cap), got)
    if case < specgen.ENUM_GOLDEN_CASES:
        gold = np.load(os.path.join(HERE, "golden", "enumerate_ref.npz"))
        for name, arr in zip(GOLD_NAMES, got.trimmed()):
            assert arr.tobytes() == gold[f"{name}{case}"].tobytes(), name
    if reflib.have_ref():
        _same(reflib.ref_enumerate_alignments(eb, cap_alns=cap), got)


def test_k7_device_resident_many_regions(ctx):
    """a batch large enough that every thread of the persistent grid strides over several reads and the scan runs over many tiles;
    default per-read capacity (64 alignments): deeper reads come back flagged SX_ENUM_ST_LIMIT exactly as the oracle flags them."""
    from strelka_b200.api import DevEnumBatch

    rng = np.random.default_rng(77)
    regions = [specgen.random_enum_region(rng, n_reads=int(rng.integers(1, 9)), cluster=bool(i % 3 == 0), n_keys=(1, 6)) for i in range(3000)]
    eb = B.EnumBatch(regions)
    want = reflib.ox_enumerate_alignments(eb, cap_alns=eb.n_reads * 64 + 64)
    db = DevEnumBatch(ctx, eb, cap_alns=eb.n_reads * 64 + 64)
    ctx.enumerate_alignments_dev(db)
    got = db.download()
    _same(want, got)
    st = want.status[: eb.n_reads]
    assert int(want.totals[0]) > 50000 and (st & A.SX_ENUM_ST_LIMIT).any() and (st == 0).sum() > eb.n_reads // 2


def test_k7_capacity_error_reports_the_needed_sizes(ctx):
    from strelka_b200.api import SxError

    eb = specgen.enum_case(1)
    full = ctx.enumerate_alignments(eb)
    with pytest.raises(SxError) as e:
        ctx.enumerate_alignments(eb, cap_alns=int(full.totals[0]) - 1)
    assert e.value.code == A.SX_ERR_CAPACITY and str(int(full.totals[0])) in str(e.value)
    again = ctx.enumerate_alignments(eb)  # the context is usable afterwards
    _same(full, again)


def test_k7_feeds_k6(ctx):
    """the enumerator's output IS K6's alignment description: same order (std::set<CandidateAlignment>), same key lists.  Score the
    enumerated alignments of a batch with synthetic scores and run score_indels on them: records identical to the oracle's."""
    eb = specgen.enum_case(0)
    out = ctx.enumerate_alignments(eb)
    sb = specgen.score_indels_batch_from_enumeration(eb, out)
    rng = np.random.default_rng(3)
    lnp = np.concatenate([-rng.random(sb.n_alns) * 30.0, [0.0]])
    got = ctx.score_indels(sb, lnp)
    for a, b in zip(reflib.ox_score_indels(sb, lnp), got):
        assert a.tobytes() == b.tobytes()


# ------------------------------------------------------------------------------------------------------------------------------
# K7b link_alignments, and the chain K7 -> K7b -> K1 -> K6 through the C ABI
# ------------------------------------------------------------------------------------------------------------------------------
def _pad(s):
    return s[~((s["kind"] == A.SX_SEG_HARDCLIP) & (s["len"] == 0))]


@pytest.mark.parametrize("case", range(12))
def test_k7b_link_alignments_and_the_chain(ctx, case):
    """enumerate on the GPU, link on the GPU, score the linked batch on the GPU: the alignment description equals the host
    flattening of the same alignments, and K1's scores of it equal the oracle's scores of the host-built batch bit for bit."""
    eb = specgen.enum_case(case)
    out = ctx.enumerate_alignments(eb)
    _same(reflib.ox_enumerate_alignments(eb), out)
    rng = np.random.default_rng(case)
    regions = B.regions_from_enumeration(eb, out, lambda r, n: rng.choice([11, 25, 37], n).astype(np.uint8))
    want = B.build_align_batch(regions)
    lo = ctx.link_alignments(eb, out, want.regions)
    assert ctx.timing().launches == 9
    got = lo.align_batch(want)
    assert got.n_alns == want.n_alns and not (got.regions["seg_begin"] % 8).any() and not (got.regions["ins_begin"] % 16).any()
    for i in range(want.n_alns):
        ws = _pad(want.segs[int(want.alns["seg_off"][i]) : int(want.alns["seg_off"][i + 1])])
        gs = _pad(got.segs[int(got.alns["seg_off"][i]) : int(got.alns["seg_off"][i + 1])])
        n_ins = int(ws["len"][ws["kind"] == A.SX_SEG_INSERT].sum())
        assert ws.tobytes() == gs.tobytes(), i
        assert bytes(want.ins[int(want.alns["ins_off"][i]) : int(want.alns["ins_off"][i]) + n_ins]) == bytes(got.ins[int(got.alns["ins_off"][i]) : int(got.alns["ins_off"][i]) + n_ins])
    lnp = ctx.score_alignments(got)
    assert np.array_equal(lnp.view(np.uint64), reflib.ox_score(want).view(np.uint64))
    # ... and K6 on those scores, in the enumerator's order
    sb = specgen.score_indels_batch_from_enumeration(eb, out, k6_segs=lo.k6_segs)
    lnp1 = np.concatenate([lnp, [0.0]])
    for a, b in zip(reflib.ox_score_indels(sb, lnp1), ctx.score_indels(sb, lnp1)):
        assert a.tobytes() == b.tobytes()


def test_k7b_capacity_error(ctx):
    from strelka_b200.api import SxError

    eb = specgen.enum_case(1)
    out = ctx.enumerate_alignments(eb)
    regions = B.regions_from_enumeration(eb, out)
    want = B.build_align_batch(regions)
    full = ctx.link_alignments(eb, out, want.regions)
    with pytest.raises(SxError) as e:
        ctx.link_alignments(eb, out, want.regions, cap_segs=int(full.totals[0]) - 1)
    assert e.value.code == A.SX_ERR_CAPACITY


def test_cpp_host_mirror_k7(tmp_path):
    """sx::AlignmentSearchBatch (the C++ layer a reference developer programs against) through libstrelka_b200.so against the
    reference's getCandidateAlignments results frozen in tests/golden/k7_cases.tsv."""
    import subprocess

    root = os.path.dirname(HERE)
    exe = str(tmp_path / "test_k7_mirror")
    lib = os.path.join(root, "strelka_b200", "csrc")
    subprocess.check_call(["g++", "-std=c++14", "-O1", "-I" + os.path.join(root, "include"), "-I" + os.path.join(root, "strelka_b200", "host"),
                           os.path.join(HERE, "cpp", "test_k7_mirror.cpp"), "-o", exe, "-L" + lib, "-lstrelka_b200", "-Wl,-rpath," + lib])
    out = subprocess.run([exe, os.path.join(HERE, "golden")], capture_output=True, text=True)
    assert out.returncode == 0 and "0 failures" in out.stdout, out.stdout + out.stderr


@pytest.mark.parametrize("case", range(16))
def test_k7a_alignment_indels(ctx, case):
    """K7a on the GPU: the keys of every input alignment from K1's packed read / reference pools == the host builder's (which is
    pinned against the reference's getAlignmentIndels in tests/test_enumerate.py), tidy and awkward inputs; then K7 on the device-made
    arrays == the oracle."""
    eb = specgen.enum_edge_case(case) if case % 2 else specgen.enum_case(case)
    po = ctx.alignment_indels(eb, B.read_pools_of(eb))
    assert ctx.timing().launches == 6
    n = eb.n_reads
    want = (eb.in_key_off[: n + 1], eb.in_keys[: int(eb.in_key_off[n])], eb.in_lead_key[:n], eb.in_trail_key[:n])
    for x, y in zip(po.trimmed(), want):
        assert np.array_equal(x, y)
    # swap the device-made arrays in and enumerate
    eb.in_key_off, eb.in_keys, eb.in_lead_key, eb.in_trail_key = po.in_key_off, po.in_keys, po.in_lead_key, po.in_trail_key
    eb.c.in_key_off, eb.c.in_keys, eb.c.in_lead_key, eb.c.in_trail_key = A.ptr(po.in_key_off), A.ptr(po.in_keys), A.ptr(po.in_lead_key), A.ptr(po.in_trail_key)
    _same(reflib.ox_enumerate_alignments(eb), ctx.enumerate_alignments(eb))


@pytest.mark.parametrize("case", [0, 1, 2, 3, 5, 7])
def test_device_resident_chain(ctx, case):
    """K7a -> K7 -> K7b -> K1 -> K6 + K9 with every intermediate in HBM (strelka_b200.api.DevRealignChain) against the chain run step by step
    through the CPU oracles: alignments, scores (bit for bit), score_indels records (byte for byte).  The same check on the CPU with a
    mock context: tests/test_chain_plumbing.py."""
    from strelka_b200.api import DevRealignChain
    from test_chain_plumbing import check_chain

    eb = specgen.enum_edge_case(case) if case % 2 else specgen.enum_case(case)
    chain = DevRealignChain(ctx, eb, B.read_pools_of(eb), cap_alns_per_read=64)
    chain.run()
    check_chain(chain, eb)
    chain.run()
    check_chain(chain, eb)
    chain.free()


@pytest.mark.parametrize("which", range(len(specgen.REALIGN_GOLDEN_CASES)))
def test_k9_choose_realignment(ctx, which):
    """K9 on the GPU with the REFERENCE's scores: rseg.realignment of every read as the reference's scoreCandidateAlignments wrote it
    (tests/golden/realign_ref.npz): default smoothing range, smoothing off, two wide ranges."""
    name, case = specgen.REALIGN_GOLDEN_CASES[which]
    gold = np.load(os.path.join(HERE, "golden", "realign_ref.npz"))
    eb = specgen.realign_case_batch(name, case)
    out = ctx.enumerate_alignments(eb)
    for tag, (smooth, rng_) in specgen.REALIGN_MODES.items():
        lnp = gold[f"lnp_{name}{case}_{tag}"]
        assert len(lnp) == int(out.totals[0])
        got = ctx.choose_realignment(B.RealignBatch(eb, out, is_smoothed=smooth, smoothed_lnp_range=rng_), np.concatenate([lnp, [0.0]]))
        assert ctx.timing().launches == 5
        pos, cig = gold[f"pos_{name}{case}_{tag}"], gold[f"cigar_{name}{case}_{tag}"]
        for r in range(eb.n_reads):
            want = (int(pos[r]), str(cig[r])) if str(cig[r]) else None
            assert got.realignment_of(r) == want, (tag, r)


@pytest.mark.parametrize("case", range(8))
def test_k9_choose_realignment_against_the_oracle(ctx, case):
    """K9 on the GPU == oracle/realign_oracle.cpp, every output array, on scores with many exact ties and on distinct ones."""
    eb = specgen.enum_edge_case(case) if case % 3 == 0 else specgen.enum_case(case)
    out = ctx.enumerate_alignments(eb)
    rng = np.random.default_rng(case)
    nA = int(out.totals[0])
    for lnp in (-rng.random(nA + 1) * 40.0, -rng.integers(0, 4, nA + 1) * 2.0):
        for k4 in (False, True):
            rb = B.RealignBatch(eb, out, k4_kinds=k4)
            want, got = reflib.ox_choose_realignment(rb, lnp), ctx.choose_realignment(rb, lnp)
            for nm in ("seg_off", "pos", "n_seg", "status", "best_aln"):
                assert np.array_equal(getattr(want, nm)[: eb.n_reads], getattr(got, nm)[: eb.n_reads]), nm
            assert want.segs[: int(want.totals[0])].tobytes() == got.segs[: int(got.totals[0])].tobytes()


@pytest.mark.parametrize("case", range(10))
def test_k7g_realign_gates(ctx, case):
    """K7g on the GPU == its host-compiled body (which tests/test_enumerate.py pins against the reference's own gate functions), and
    where the reference library travelled, == the reference."""
    eb = specgen.enum_edge_case(case) if case % 2 else specgen.enum_case(case)
    gb = B.GateBatch(eb, specgen.raw_alignments_for(eb, case))
    got = ctx.realign_gates(gb)
    assert ctx.timing().launches == 1
    rc, want = reflib.k7gcore_gates(gb)
    assert np.array_equal(got.gate[: eb.n_reads], want.gate[: eb.n_reads]) and np.array_equal(got.in_pos[: eb.n_reads], want.in_pos[: eb.n_reads])
    assert got.in_segs[: gb.n_segs].tobytes() == want.in_segs[: gb.n_segs].tobytes()
    gold = np.load(os.path.join(HERE, "golden", "gates_ref.npz"))  # the reference's own answers, frozen
    assert np.array_equal(got.gate[: eb.n_reads], gold[f"gate{case}"])
    for r in range(eb.n_reads):
        ref = (int(gold[f"pos{case}"][r]), str(gold[f"cigar{case}"][r])) if int(gold[f"gate{case}"][r]) & A.SX_GATE_REALIGN else None
        assert got.alignment_of(r) == ref, r


def test_k7_honours_the_gate_array(ctx):
    """a read K7g gated out is answered with no alignments / no keys by the kernels exactly as by the oracle."""
    eb = specgen.enum_case(1)
    rng = np.random.default_rng(5)
    eb.set_gate((rng.random(eb.n_reads + 1) < 0.6).astype(np.uint8) * A.SX_GATE_REALIGN)
    _same(reflib.ox_enumerate_alignments(eb), ctx.enumerate_alignments(eb))
    eb.opts.flags = 0  # the two-pass plan
    eb.c.opts = eb.opts
    _same(reflib.ox_enumerate_alignments(eb), ctx.enumerate_alignments(eb))


@pytest.mark.parametrize("case", [0, 1, 3, 4])
def test_device_resident_chain_from_the_mappers_alignments(ctx, case):
    """K7g -> K7a -> K7 -> K7b -> K1 -> K6 + K9 on device-resident data, the mapper's alignments in: identical to the chain run through the
    oracles on the batch a host shim would build from the gates' answers (tests/test_chain_plumbing.py does the same on a mock context)."""
    from strelka_b200.api import DevRealignChain
    from test_chain_plumbing import check_chain, normalized_batch

    eb = specgen.enum_edge_case(case) if case % 2 else specgen.enum_case(case)
    gb = B.GateBatch(eb, specgen.raw_alignments_for(eb, case))
    chain = DevRealignChain(ctx, eb, B.read_pools_of(eb), cap_alns_per_read=64, raw=gb)
    chain.run()
    gates = ctx.realign_gates(gb)
    check_chain(chain, normalized_batch(eb, gb, gates))
    chain.free()


@pytest.mark.parametrize("block", range(10))
def test_chain_equals_the_references_realignAndScoreRead(ctx, block):
    """K7g -> K7a -> K7 -> K7b -> K1 -> K6 + K9 on the GPU against the reference's own realignAndScoreRead (oracle/_ref where it is built,
    its frozen digests elsewhere) on 200 seeded batches: is_realigned, rseg.realignment segment for segment -- hard clips included --,
    getBestAlignment() of the reads that keep the mapper's alignment, and the ReadPathScores score_indels left in the indel buffer.
    (tests/test_chain_plumbing.py runs the same function on the CPU mock.)"""
    from test_chain_plumbing import chain_case, chain_vs_realign_and_score_read

    n_real = n_recs = 0
    for case in range(20 * block, 20 * block + 20):
        eb, gb = chain_case(case)
        a, b, _c = chain_vs_realign_and_score_read(ctx, eb, gb, case)
        n_real += a
        n_recs += b
    assert n_real > 100 and n_recs > 100
