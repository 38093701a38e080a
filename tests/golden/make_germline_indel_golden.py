"""Freezes the reference's answers for the K6 -> K6g -> K5 chain cases (tests/test_allele_groups.py k6_chain: one sample of each
tests/indel_reads_gen.py k6_case, with groups over its ids) into tests/golden/germline_indel_ref.npz: per case and sample the inputs' digest,
the supporting read ids of getAlleleGroupSupportingReadIds, getAlleleLogLhoodFromRead of each on the extended group, the exemplar's fields,
and the sx_indel_result records of getVariantAlleleGroupGenotypeLhoodsForSample (oracle/ref_harness_germline_indel.cpp).  Needs oracle/_ref
(the reference tree at build time).

    python tests/golden/make_germline_indel_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(os.path.dirname(HERE)), os.path.dirname(HERE)]

import allele_groups_gen as AG  # noqa: E402
import indel_reads_gen as G  # noqa: E402
import test_allele_groups as T  # noqa: E402

out = {}
for seed in range(G.K6_CASES):
    for s in range(2):
        case, sample, groups, _ = T.k6_chain(seed, s)
        batches, lnps, _, read_id, loci = case
        ref = AG.ref_chain(batches[s], lnps[s], read_id[s], loci, groups)
        key = f"{seed}_{s}"
        out[f"inputs{key}"] = np.array(AG.inputs_digest(batches[s], lnps[s], read_id[s], loci, groups))
        for k in AG.REF_KEYS:
            out[f"{k}{key}"] = np.frombuffer(ref[k].tobytes(), np.uint8) if k == "out" else ref[k]
        print(key, groups.n_groups, "groups,", int(ref["read_off"][-1]), "supporting reads")
np.savez_compressed(AG.GOLDEN, **out)
