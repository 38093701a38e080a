"""Freezes what the reference answers on the seeded two-sample windows of tests/test_zzzzzzzz_gpu_somatic_window.py -- each sample through its own
realignAndScoreRead / pileup_read_segment, position_somatic_snv_call on the two column sets, get_somatic_indel on the read_path_lnp lists of
its records, and the record lists its is_output and empty-list rules select -- as the digests tests/refgold.py compares with, into
tests/golden/somatic_window_ref_digests.json.  Run where the reference tree is built (oracle/build_ref.sh, build_ref_somatic_indel.sh,
build_ref_indel_reads.sh)."""
import json
import os
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.dirname(HERE), HERE, os.path.join(os.path.dirname(HERE), "tools")]

import refgold  # noqa: E402
import test_zzzzzzzz_gpu_somatic_window as T  # noqa: E402


def main():
    assert T.have_reference(), "oracle/_ref not built"
    opts = T._opts()
    window = {}
    for case in T.CASES:
        for key, normal, tumor, loci, key_gid, forced in T.case_inputs(case):
            items = T.reference_items((normal, tumor), loci, key_gid, forced, opts)
            inputs = T.inputs_digest(normal, tumor, loci, forced)
            window[key] = refgold.record(items, inputs=inputs, compared=True) if items is not None else {"inputs": inputs, "compared": False}
    with open(T.GOLDEN, "w") as f:  # one entry per line
        f.write('{\n"window": {\n' + ",\n".join(f"{json.dumps(k)}: {json.dumps(v, separators=(',', ':'))}" for k, v in sorted(window.items())) + "\n}\n}\n")


if __name__ == "__main__":
    main()
