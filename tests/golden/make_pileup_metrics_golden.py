"""Freezes the reference's K4m answers (oracle/ref_harness_pileup_metrics.cpp, the unmodified pileup_read_segment with the scoring metrics on)
for every case of pileup_metrics_gen.golden_cases() into tests/golden/pileup_metrics_ref.npz.  Needs oracle/_ref built:
    python tests/golden/make_pileup_metrics_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import pileup_metrics_gen as G  # noqa: E402

assert G.have_ref(), "oracle/_ref/libstrelka_ref_pileup_metrics.so is not built"
out = {key: G.ref_metrics(pb, mode) for key, pb, mode in G.golden_cases()}
np.savez_compressed(G.GOLDEN, **out)
print(f"{len(out)} cases -> {G.GOLDEN}")
