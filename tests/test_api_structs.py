"""The Python face of the ABI builds its structs by field name, and every device twin (api.Dev*) is its host struct with each array moved
to device memory: checked on the CPU, "device" memory being host memory (tests/mockctx.py)."""
import ast
import ctypes as C
import inspect
from types import SimpleNamespace

import numpy as np
import pytest

import indel_reads_gen as G
import reflib
import sindel_gen
import specgen
import window_check as W
from mockctx import MockContext, _MockLib
from strelka_b200 import _abi as A
from strelka_b200 import api
from strelka_b200 import batch as B


def test_abi_structs_are_built_by_field_name():
    """no A.Sx*(...) with positional arguments, no method attached to Context from outside its class, no `_ARRAYS` name list"""
    for mod in (api, B):
        for node in ast.walk(ast.parse(inspect.getsource(mod))):
            where = f"{mod.__name__}:{getattr(node, 'lineno', '?')}"
            if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and isinstance(node.func.value, ast.Name) and node.func.value.id == "A":
                assert not (node.func.attr.startswith("Sx") and node.args), f"{where}: A.{node.func.attr} with positional arguments"
            if isinstance(node, ast.Assign):
                for t in node.targets:
                    assert not (isinstance(t, ast.Attribute) and isinstance(t.value, ast.Name) and t.value.id == "Context"), f"{where}: Context.{t.attr} assigned"
                    assert not (isinstance(t, ast.Name) and t.id.endswith("_ARRAYS")), f"{where}: {t.id}"
        for node in ast.parse(inspect.getsource(mod)).body:
            assert not (isinstance(node, ast.FunctionDef) and node.args.args and node.args.args[0].arg == "self"), f"{mod.__name__}.{node.name} takes self"


@pytest.fixture(scope="module")
def ctx():
    c = MockContext.__new__(MockContext)  # only its memory is used here: no kernel is called
    c.lib, c.h = _MockLib(), 1
    return c


def _check_twin(host, dev, owner, slack, adopted=None):
    """dev (an api.Dev* object) against the host struct: non-pointer fields equal, pointers NULL exactly where the host's are, adopted
    pointers kept, every other pointer at a buffer of `slack` bytes more than owner's array of the field's name, holding its bytes."""
    adopted = adopted or {}
    ptrs = [n for n, t in type(host)._fields_ if t is C.c_void_p]
    h, d = type(host).from_buffer_copy(host), type(host).from_buffer_copy(dev.c)
    for n in ptrs:
        setattr(h, n, None)
        setattr(d, n, None)
    assert bytes(h) == bytes(d)
    for n in ptrs:
        hp, dp = getattr(host, n), getattr(dev.c, n)
        assert bool(hp) == bool(dp), n
        if not hp:
            continue
        if n in adopted:
            assert dp == adopted[n], n
            continue
        arr = np.ascontiguousarray(getattr(owner, n))
        assert dev.bufs[n].ptr == dp and dev.bufs[n].nbytes == arr.nbytes + slack, n
        assert C.string_at(dp, arr.nbytes) == arr.tobytes(), n


def _regions(seed, n=3):
    rng = np.random.default_rng(seed)
    return [specgen.simple_region(rng, n_reads=12) for _ in range(n)]


def _score_indels_from_arrays():
    eb = specgen.enum_case(0)
    return specgen.score_indels_batch_from_enumeration(eb, reflib.ox_enumerate_alignments(eb))


HOST_BATCHES = {  # name -> (api class, seeded host batch)
    "align": lambda: (api.DevAlignBatch, B.build_align_batch(_regions(1))),
    "align_baseq": lambda: (api.DevAlignBatch, B.build_align_batch(_regions(2), qual_bits=2, compact=True)),
    "pileup": lambda: (api.DevPileupBatch, specgen.random_pileups(np.random.default_rng(3), 60)),
    "pileup_tier2": lambda: (api.DevPileupBatch, specgen.random_pileups(np.random.default_rng(4), 60, with_tier2=True)),
    "ga": lambda: (api.DevGaBatch, B.GaBatch(*specgen.random_ga_problems(np.random.default_rng(5), 16))),
    "somatic_indel": lambda: (api.DevSomaticIndelBatch, sindel_gen.case(0)[0]),
    "score_indels": lambda: (api.DevScoreIndelsBatch, B.score_indels_batch_from_regions(_regions(6))),
    "score_indels_arrays": lambda: (api.DevScoreIndelsBatch, _score_indels_from_arrays()),
    "indel_reads_sample": lambda: (api.DevIndelReadsSample, G.synth(0)[0]),
    "indel_loci": lambda: (api.DevIndelLoci, G.synth(0)[2]),
    "enum": lambda: (api.DevEnumBatch, specgen.enum_case(0)),
    "enum_hap": lambda: (api.DevEnumBatch, specgen.enum_case(8)),
}


@pytest.mark.parametrize("name", sorted(HOST_BATCHES))
def test_device_twin_is_the_host_struct_on_the_device(ctx, name):
    cls, hb = HOST_BATCHES[name]()
    if name == "align_baseq":
        assert hb.exc_off is not None and hb.fmt & A.SX_FMT_BASEQ
    if name.startswith("pileup"):
        assert (hb.t2_off is not None) == name.endswith("tier2")
    if name.startswith("enum"):
        assert hb.has_hap == name.endswith("hap")
    _check_twin(hb.c, cls(ctx, hb), hb, 64)


def test_device_twin_keeps_adopted_pointers(ctx):
    """DevIndelReadsSample.from_score_indels points the sample's read arrays and recs / n_rec at the DevScoreIndelsBatch's buffers and
    uploads only key_gid and read_id"""
    batches, _lnps, key_gid, read_id, _loci = G.k6_case(0)
    db = api.DevScoreIndelsBatch(ctx, batches[0])
    ds = api.DevIndelReadsSample.from_score_indels(ctx, db, key_gid[0], read_id[0])
    adopted = {n: db.bufs[n].ptr for n in ("region_read_off", "region_key_off", "rec_off", "read_len", "non_ambig", "read_flags")}
    adopted.update(recs=db.recs.ptr, n_rec=db.n_rec.ptr)
    _check_twin(ds.host.c, ds, ds.host, 64, adopted)
    assert set(ds.bufs) == {"key_gid", "read_id"}


def test_device_window_inputs(ctx):
    """DevWindow: every array of the window batch in a buffer 80 bytes longer, NULL where the batch has none (key_hap without haplotypes,
    cand_snv); the scalars from the batch"""
    for case, has_hap in ((0, False), (8, True)):
        eb1, gb1, flags, mapq = next(W.window_case(case))
        assert eb1.has_hap == has_hap
        w = B.WindowBatch.from_enum(eb1, gb1, B.read_pools_of(eb1), read_flags=flags, mapq=mapq)
        dw = api.DevWindow(ctx, w)
        host = A.SxWindowBatch.from_buffer_copy(dw.c)
        for name in B.WindowBatch.ARRAYS:
            setattr(host, name, A.ptr(w.a.get(name)))
        _check_twin(host, dw, SimpleNamespace(**w.a), 80)
        c = dw.c
        assert (c.n_regions, c.n_reads, c.n_keys, c.n_cand_snv) == (w.n_regions, w.n_reads, w.n_keys, 0)
        assert (c.seq4_bytes, c.qual_bytes, c.ref_bytes, c.qual_bits) == (w.used["seq4"], w.used["qual"], w.used["ref"], w.qual_bits)
        assert (c.ref_begin, c.report_begin, c.report_end, c.max_read_len, c.do_site_gl) == (w.ref_begin, w.report_begin, w.report_end, w.max_read_len, 1)
        assert c.enum_opts.max_indel_size == eb1.opts.max_indel_size and bool(c.key_hap) == eb1.has_hap
        dw.free()


def test_device_twin_refuses_a_set_field_without_an_array(ctx):
    gb = B.GaBatch(["ACGT"], ["ACGT"])
    with pytest.raises(ValueError, match="query_off"):
        api._device_twin(ctx, gb.c, SimpleNamespace(query=gb.query, ref=gb.ref, ref_off=gb.ref_off), 64)
