"""Freezes what the reference's own realignAndScoreRead, pileup_read_segment and position_snp_call_pprob_digt (oracle/_ref/libstrelka_ref.so)
answer on the seeded inputs of the whole-pass comparisons -- test_chain_plumbing.chain_vs_realign_and_score_read, window_check.check_window,
the synthetic windows of tests/test_zzzz_gpu_window.py and smoke()'s window -- as the digests tests/refgold.py compares with, into
tests/golden/window_ref_digests.json.  Run where the reference tree is built (oracle/build_ref.sh)."""
import json
import os
import sys
from concurrent.futures import ProcessPoolExecutor

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.dirname(HERE), HERE, os.path.join(os.path.dirname(HERE), "tools")]

import numpy as np  # noqa: E402

import refgold  # noqa: E402
import reflib  # noqa: E402
import window_check as W  # noqa: E402
import window_workload as WW  # noqa: E402
from strelka_b200 import batch as B  # noqa: E402
from test_chain_plumbing import chain_case, chain_inputs_digest, chain_reference, use_the_references_bound  # noqa: E402

CASES = 200
SYNTHETIC = [(4, 1), (8, 2), (4, 3)]  # (qual_bits, seed) of test_synthetic_cfg2_window_equals_the_reference


def chain_entry(case):
    eb, gb = chain_case(case)
    use_the_references_bound(eb)
    items, threw = chain_reference(eb, gb)
    return str(case), refgold.record(items, inputs=chain_inputs_digest(eb, gb), threw=threw)


def window_entries(case):
    out = {}
    for i, (eb1, gb1, flags, mapq) in enumerate(W.window_case(case)):
        w = B.WindowBatch.from_enum(eb1, gb1, B.read_pools_of(eb1), read_flags=flags, mapq=mapq)
        exp = W.reference_window(eb1, gb1, w)
        out[f"{case}.{i}"] = refgold.record(W.reference_items(exp, w), threw=[int(r) for r in np.nonzero(exp["status"] == 2)[0]], piled=exp["cols"] is not None)
    return out


def synthetic_entry(n_cells, qual_bits, seed, tile):
    w = WW.make_window(WW.load_synth(), n_cells, seed, tile=tile, qual_bits=qual_bits, ascii_reads=True)
    return refgold.record(WW.reference_items(w, WW.reference_pass(w)[0]), inputs=refgold.synthetic_inputs_digest(w))


def main():
    assert reflib.have_ref(), "oracle/_ref/libstrelka_ref.so not built"
    with ProcessPoolExecutor() as ex:
        chain = dict(ex.map(chain_entry, range(CASES)))
        window = {}
        for d in ex.map(window_entries, range(CASES)):
            window.update(d)
        synthetic = dict(zip((f"{q}-{s}" for q, s in SYNTHETIC), ex.map(synthetic_entry, [400] * 3, *zip(*[(q, s, s) for q, s in SYNTHETIC]))))
        synthetic["smoke"] = synthetic_entry(60, 4, 3, 0)  # __graft_entry__.smoke()'s window
    with open(refgold.GOLDEN, "w") as f:  # one entry per line
        sections = [("chain", chain), ("synthetic", synthetic), ("window", window)]
        f.write("{\n")
        for i, (name, sec) in enumerate(sections):
            f.write(f'"{name}": {{\n' + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, separators=(',', ':'))}" for k, v in sorted(sec.items())) + "\n}")
            f.write(",\n" if i + 1 < len(sections) else "\n}\n")


if __name__ == "__main__":
    main()
