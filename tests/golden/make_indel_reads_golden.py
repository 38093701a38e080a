"""Freezes the reference's answers for the K6 -> K6b -> K5b chain cases (tests/indel_reads_gen.py k6_case) into
tests/golden/indel_reads_ref.npz: per case the inputs' digest, the sx_sindel_result records of the reference's get_somatic_indel and the
IndelBuffer's read_path_lnp maps flattened (oracle/ref_harness_indel_reads.cpp).  Needs oracle/_ref (the reference tree at build time).

    python tests/golden/make_indel_reads_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]

import indel_reads_gen as G  # noqa: E402
from strelka_b200 import _abi as A  # noqa: E402

out = {}
for seed in range(G.K6_CASES):
    case = G.k6_case(seed)
    batches, lnps, _, read_id, loci = case
    ref, maps = G.ref_chain(batches, lnps, read_id, loci, A.default_sindel_opts())
    out[f"inputs{seed}"] = np.array(G.inputs_digest(*case))
    out[f"ref{seed}"] = np.frombuffer(ref.tobytes(), np.uint8)
    out[f"reads{seed}"] = np.frombuffer(maps["reads"].tobytes(), np.uint8)
    for k in ("read_off", "entry_id", "alt_off", "alt_gid"):
        out[f"{k}{seed}"] = maps[k]
    print(seed, loci.n_loci, "loci,", maps["reads"].size, "entries,", int(ref["is_output"].sum()), "calls")
np.savez_compressed(G.GOLDEN, **out)
