"""Freezes the reference's own get_somatic_indel answers (oracle/_ref/libstrelka_ref_sindel.so) for the K5b parity cases of
tests/sindel_gen.py into tests/golden/somatic_indel_ref.npz, with a digest of the inputs they were computed for."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import sindel_gen as G  # noqa: E402


def main():
    assert G.have_ref(), "build oracle/_ref first (oracle/build_ref.sh, oracle/build_ref_somatic_indel.sh)"
    arrays = {}
    for i in range(len(G.CASES)):
        sb, o = G.case(i)
        arrays[f"inputs{i}"] = np.array(G.inputs_digest(sb))
        arrays[f"ref{i}"] = np.frombuffer(G.ref_somatic_indel(o, sb).tobytes(), np.uint8)
    np.savez_compressed(os.path.join(HERE, "somatic_indel_ref.npz"), **arrays)


if __name__ == "__main__":
    main()
