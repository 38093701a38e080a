"""GPU: strelka2_sx (integration/build_patched.py) with the somatic caller's indel call site routed through sx_somatic_indel (K5b) on the
reference's bundled demo: its indels.vcf and snvs.vcf bodies equal src/demo/expectedResults/somatic.{indels,snvs}.vcf.gz, the shim report counts
the somatic indel calls the library made, and the same binary with SX_SHIM_OFF=1 (every call on the reference's CPU functions) writes the
same bodies.  The binaries and demo inputs are built / staged where /root/reference exists (oracle/_ref/bin, oracle/_ref/demo)."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import run_demo as R  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]


def _indel_calls(stderr):
    """The count the shim appends to its report line: '..., N somatic indel calls'."""
    for ln in stderr.splitlines():
        if ln.startswith("sx_shim:"):
            parts = ln.split()
            assert parts[-3:] == ["somatic", "indel", "calls"], ln
            return int(parts[-4])
    return -1


def test_somatic_demo_indels_through_the_library(tmp_path):
    if not os.path.exists(os.path.join(R.BIN, "strelka2_sx")) or not os.path.isdir(R.DEMO):
        pytest.skip("oracle/_ref/bin or oracle/_ref/demo missing: run integration/build_patched.py where the reference tree exists")
    got, err = R.run("somatic", "strelka2_sx", str(tmp_path / "gpu"), env={"SX_SHIM_REPORT": "1"})
    n = _indel_calls(err)
    print(f"somatic indel calls through libstrelka_b200.so: {n}")
    assert n >= 2, err[-500:]
    exp = {f: R.body(os.path.join(R.DEMO, "expected", f"somatic.{f}.gz")) for f in ("indels.vcf", "snvs.vcf")}
    assert len(exp["indels.vcf"]) == 2
    for f in exp:
        assert got[f] == exp[f], f
    off, err_off = R.run("somatic", "strelka2_sx", str(tmp_path / "cpu"), env={"SX_SHIM_REPORT": "1", "SX_SHIM_OFF": "1"})
    assert _indel_calls(err_off) in (0, -1), err_off[-500:]
    for f in exp:
        assert off[f] == got[f], f
