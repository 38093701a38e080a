"""Freezes the reference's answers for the parameter sweep of the somatic SNV model (K2b) and the indel genotype model (K5) into
tests/golden/site_params_ref.npz: at every point of tests/site_params.py, the fields oracle/ref_harness.cpp returns for the K2b edge
batch (tier2 calls on both samples, on neither and on one only; ntype 0 where the reference leaves it unassigned) and the whole sx_indel_result records of the K5 edge batch, with a digest
of the inputs.  Written without time stamps, so that a second run writes the same bytes.  Needs oracle/_ref (the reference tree at build
time).

    python tests/golden/make_site_params_golden.py"""
import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]

import reflib  # noqa: E402
import site_params as SP  # noqa: E402
import specgen  # noqa: E402


def reference_answers() -> dict:
    out = {"inputs": np.frombuffer(SP.inputs_digest().encode(), np.uint8)}
    npb, tpb, forced, _ = SP.k2b_edge_batch()
    for point in SP.K2B_POINTS:
        p = SP.k2b(point)
        for mode in specgen.SOMATIC_TIER2_MODES:
            n, t = specgen.somatic_tier2_view(npb, tpb, mode)
            out[SP.golden_key("k2b", point, mode)] = SP.reference_fields(p, n, t, forced)
    ib = SP.k5_edge_batch()
    for point in SP.K5_POINTS:
        out[SP.golden_key("k5", point)] = np.frombuffer(reflib.ref_indel_gl(SP.k5(point), ib).tobytes(), np.uint8)
    return out


def write_npz(path: str, arrays: dict) -> None:
    """np.savez_compressed without the zip entries' modification times"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.ascontiguousarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


if __name__ == "__main__":
    arrays = reference_answers()
    write_npz(SP.GOLDEN, arrays)
    print(SP.GOLDEN, len(arrays), "arrays,", os.path.getsize(SP.GOLDEN), "bytes")
