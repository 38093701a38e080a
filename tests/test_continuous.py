"""K2c site_continuous on the CPU: the oracle (oracle/continuous_oracle.cpp), the host builder and the kernels' body compiled with g++
(tests/cpp/k2c_core_host.cpp) agree byte for byte on seeded multi-sample columns that reach every branch of the model; the body's qscore
equals the reference's frozen answers over the whole grid with no tie flag, and its strand bias is within continuous_gen.SB_BOUND of them;
with oracle/_ref built (`ref`), the frozen answers are the reference's own; the structs' ctypes layout is the C compiler's."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import continuous_gen as G
from strelka_b200 import _abi as A
from strelka_b200 import batch as B

OPTS = [G.default_opts(), A.SxContOpts(0.2, 5.0, 10, 30), A.SxContOpts(0.45, 0.0, 0, 60)]


def test_struct_layouts(tmp_path):
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    structs = [("sx_cont_opts", A.SxContOpts), ("sx_cont_batch", A.SxContBatch), ("sx_cont_out", A.SxContOut)]
    dts = [("sx_cont_locus", A.CONT_LOCUS_DT), ("sx_cont_sample", A.CONT_SAMPLE_DT)]
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "strelka_b200.h"', "int main(void) {"]
    for name, cls in structs:
        lines.append(f'printf("%zu", sizeof({name}));')
        lines += [f'printf(" %zu", offsetof({name}, {f}));' for f, _ in cls._fields_]
        lines.append('printf("\\n");')
    for name, dt in dts:
        lines.append(f'printf("%zu", sizeof({name}));')
        lines += [f'printf(" %zu", offsetof({name}, {f}));' for f in dt.names]
        lines.append('printf("\\n");')
    lines += ['printf("%d %d %d\\n", SX_CONT_MAX_SAMPLES, SX_CONT_REF_LOCUS, SX_CONT_ST_QSCORE_TIE);', "return 0; }"]
    (tmp_path / "layout.c").write_text("\n".join(lines))
    subprocess.check_call([cc, "-std=c99", "-I", os.path.join(G.ROOT, "include"), str(tmp_path / "layout.c"), "-o", str(tmp_path / "layout")])
    got = subprocess.check_output([str(tmp_path / "layout")], text=True).split("\n")
    for (name, cls), line in zip(structs, got):
        assert [int(x) for x in line.split()] == [C.sizeof(cls)] + [getattr(cls, f).offset for f, _ in cls._fields_], name
    for (name, dt), line in zip(dts, got[len(structs):]):
        assert [int(x) for x in line.split()] == [dt.itemsize] + [dt.fields[f][1] for f in dt.names], name
    assert [int(x) for x in got[len(structs) + len(dts)].split()] == [A.SX_CONT_MAX_SAMPLES, A.SX_CONT_REF_LOCUS, A.SX_CONT_ST_QSCORE_TIE]


@pytest.mark.parametrize("S", [1, 2, 3, 8])
@pytest.mark.parametrize("k", range(len(OPTS)))
def test_oracle_and_kernel_body_agree(S, k):
    b = G.case(100 * S + k, S)
    G.same(G.ox_run(b, OPTS[k]), G.core_run(b, OPTS[k]))


def test_cases_reach_every_branch():
    opts = G.default_opts()
    seen = set()
    for S in (1, 2, 3):
        b = G.case(100 * S, S)
        o = G.ox_run(b, opts)
        loci, ent, off = o.trimmed()
        forced = b.forced_output if b.forced_output is not None else np.zeros(b.n_sites, np.uint8)
        raw = sum(np.diff(p.site_off) for p in b.samples)
        n_rec = np.diff(off)
        if np.any((n_rec == 0) & (raw == 0) & (forced == 0)):
            seen.add("skip")
        assert not np.any((n_rec == 0) & ((raw > 0) | (forced > 0))), "a site with calls or forced output has a record"
        if np.any(loci["ref"] == 4):
            seen.add("n_ref")
        if np.any((loci["ref"] == 4) & (n_rec[np.searchsorted(off, np.arange(len(loci)), side="right") - 1] == 4)):
            seen.add("n_ref_four_alts")
        if np.any(loci["forced"] == 1):
            seen.add("forced")
        if np.any(loci["alt"] == A.SX_CONT_REF_LOCUS):
            seen.add("ref_fallback")
        if np.any(n_rec >= 2):
            seen.add("several_alts")
        if np.any((ent["af"] == opts.min_het_vf)):
            seen.add("af_at_min_het_vf")
        if np.any((ent["af"] == 1 - opts.min_het_vf)):
            seen.add("af_at_1_minus_min_het_vf")
        if np.any((ent["used"] > 0) & (ent["total_depth"] == 0)):
            seen.add("only_any")
        if np.any((ent["used"] == 0) & (ent["unused"] > 0)):
            seen.add("only_filtered")
        for gt in (0, 1, 2):
            if np.any((ent["gt"] == gt) & (np.repeat(loci["alt"], S).reshape(-1, S) != 4)):
                seen.add(f"gt{gt}")
        if np.any(np.isin(ent["strand_bias"], [99.0, -99.0])):
            seen.add("sb_clamped")
        if np.any((ent["gq"] > 0) & (ent["gq"] < 40)) and np.any(ent["gq"] == 40):
            seen.add("gq_range")
        # count ties: two alt loci of one site with the same depth in a sample
        for i in range(len(off) - 1):
            if off[i + 1] - off[i] >= 2 and len(np.unique(ent["allele_depth"][off[i]:off[i + 1], 0])) < off[i + 1] - off[i]:
                seen.add("count_ties")
                break
    want = {"skip", "n_ref", "n_ref_four_alts", "forced", "ref_fallback", "several_alts", "af_at_min_het_vf", "af_at_1_minus_min_het_vf", "only_any",
            "only_filtered", "gt0", "gt1", "gt2", "sb_clamped", "gq_range", "count_ties"}
    assert want <= seen, want - seen


def test_spanning_deletions_only_column():
    """a forced position with no calls (a column under spanning deletions only): every alt record, depth 0, AF 0, GQ 0"""
    p = B.PileupBatch.from_sites([[]], "C")
    o = G.core_run(B.ContBatch([p], 7, np.ones(1, np.uint8)), G.default_opts())
    loci, ent, _ = o.trimmed()
    assert list(loci["alt"]) == [0, 2, 3] and list(loci["pos"]) == [7, 7, 7]
    assert np.all(ent["total_depth"] == 0) and np.all(ent["af"] == 0) and np.all(ent["gq"] == 0) and np.all(ent["gt"] == 0)


def test_capacity():
    b = G.case(5, 2)
    full = G.core_run(b, G.default_opts())
    n = int(full.totals[0])
    short = G.core_run(b, G.default_opts(), cap=n - 1)
    assert int(short.totals[0]) == n and np.array_equal(short.site_rec_off, full.site_rec_off)
    assert not short.loci.view(np.uint8).any() and not short.samples.view(np.uint8).any()


def test_qscore_grid_equals_reference_frozen():
    g = np.load(G.GOLDEN)
    a, n = G.grid_pairs()
    gq, st = G.core_qscore(a, n)
    assert np.array_equal(gq, G.gq_from_thresholds(g["first"], a, n))
    assert not st.any(), "no tie flag on the grid"
    gq, st = G.core_qscore(g["large_a"], g["large_n"])
    assert np.all(gq == 40) and not st.any()


def test_strand_bias_within_bound_of_reference_frozen():
    g = np.load(G.GOLDEN)
    got, want = G.core_strand_bias(g["sb_counts"]), g["sb_ref"]
    for f in (np.isnan, np.isposinf, np.isneginf):
        assert np.array_equal(f(got), f(want))
    fin = np.isfinite(want)
    d = float(np.max(np.abs(got[fin] - want[fin])))
    print(f"largest |strandBias - reference| {d:.3g} over {int(fin.sum())} finite answers")
    assert d <= G.SB_BOUND


@pytest.mark.ref
def test_frozen_answers_are_the_references():
    if not G.have_ref():
        pytest.skip("oracle/_ref/libstrelka_ref_continuous.so not built")
    g = np.load(G.GOLDEN)
    a, n = G.grid_pairs()
    first, top = G.grid_thresholds(a, n, G.ref_qscore(a, n))
    assert np.array_equal(first, g["first"]) and np.array_equal(top, g["top"])
    assert np.all(G.ref_qscore(g["large_a"], g["large_n"]) == 40)
    assert np.array_equal(G.ref_strand_bias(g["sb_counts"]).view(np.uint64), g["sb_ref"].view(np.uint64))


@pytest.mark.ref
def test_seeded_columns_strand_bias_against_reference():
    if not G.have_ref():
        pytest.skip("oracle/_ref/libstrelka_ref_continuous.so not built")
    for S in (1, 3):
        loci, ent, _ = G.core_run(G.case(100 * S, S), G.default_opts()).trimmed()
        alt = loci["alt"] != A.SX_CONT_REF_LOCUS
        c = np.stack([loci["sb_fwd_alt"], loci["sb_rev_alt"], loci["sb_fwd_other"], loci["sb_rev_other"]], 1)[alt]
        want, got = G.ref_strand_bias(c), loci["strand_bias"][alt]
        fin = np.isfinite(want)
        assert np.array_equal(np.isfinite(got), fin) and np.max(np.abs(got[fin] - want[fin])) <= G.SB_BOUND
        gq = ent["gq"].ravel()
        assert np.array_equal(gq, G.ref_qscore(ent["allele_depth"].ravel(), ent["total_depth"].ravel()))
