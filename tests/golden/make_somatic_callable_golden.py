"""Freezes the reference's answers for K2b's callable mode into tests/golden/somatic_callable_ref.npz: for every case of
tests/callable_gen.py, the fields oracle/ref_harness_somatic_callable.cpp returns (nonsomatic_qphred included; ntype 0 where the reference
leaves it unassigned) and the BED text of its SomaticCallableProcessor, with a digest of the inputs.  Written without time stamps, so that
a second run writes the same bytes.  Needs oracle/_ref (the reference tree at build time).

    python tests/golden/make_somatic_callable_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE), HERE]

import callable_gen as G  # noqa: E402
from make_site_params_golden import write_npz  # noqa: E402


def reference_answers() -> dict:
    out = {"inputs": np.frombuffer(G.inputs_digest().encode(), np.uint8)}
    for name, p, n, t, forced in G.cases():
        f, bed = G.reference_fields(p, n, t, forced)
        out[name + "__fields"] = f
        out[name + "__bed"] = np.frombuffer(bed.encode(), np.uint8)
    return out


if __name__ == "__main__":
    arrays = reference_answers()
    write_npz(G.GOLDEN, arrays)
    print(G.GOLDEN, len(arrays), "arrays,", os.path.getsize(G.GOLDEN), "bytes")
