"""GPU: strelka2_sx (integration/build_patched.py) with the callable regions written (integration/run_demo.py somatic-callable: the somatic demo's
command line plus --somatic-callable-regions-file, as strelkaSomaticWorkflow.py issues it for --outputCallableRegions).  The somatic SNV call site
then goes through K2b's callable mode (sx_site_gl_somatic_callable), whose nonsomatic_qphred feeds the reference's own SomaticCallableProcessor.
Its snvs.vcf, indels.vcf and callable.bed bodies are the unmodified strelka2's (tests/golden/somatic_callable_demo_bodies.json), line for line,
with the route on and with SX_SHIM_OFF=1.  With the route on, the report's somatic site counter equals that of the plain somatic demo: one call
per position the caller visits (every position with coverage), none left on the CPU."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import run_demo as R  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "somatic_callable_demo_bodies.json")))["somatic-callable"]


def _need():
    if not os.path.exists(os.path.join(R.BIN, "strelka2_sx")) or not os.path.isdir(R.DEMO):
        pytest.skip("oracle/_ref/bin or oracle/_ref/demo missing: run integration/build_patched.py where the reference tree exists")


def _somatic_calls(stderr):
    """the second field of the report line: '..., N somatic site calls, ...'"""
    for ln in stderr.splitlines():
        if ln.startswith("sx_shim:"):
            parts = ln.split()
            assert parts[6:9] == ["somatic", "site", "calls,"], ln
            return int(parts[5])
    return -1


def test_somatic_callable_demo_through_the_library(tmp_path):
    _need()
    assert len(GOLD["snvs.vcf"]) == 17 and len(GOLD["indels.vcf"]) == 2 and len(GOLD["callable.bed"]) > 10
    got, err = R.run("somatic-callable", "strelka2_sx", str(tmp_path / "callable"), env={"SX_SHIM_REPORT": "1"})
    n = _somatic_calls(err)
    _, err_plain = R.run("somatic", "strelka2_sx", str(tmp_path / "plain"), env={"SX_SHIM_REPORT": "1"})
    print(f"callable-mode somatic site calls through libstrelka_b200.so: {n}")
    assert n > 1000 and n == _somatic_calls(err_plain), (err[-500:], err_plain[-500:])
    for f, want in GOLD.items():
        assert got[f] == want, f
    if os.path.exists(os.path.join(R.BIN, "strelka2")):  # and against the unmodified binary run on this very box
        ref, _ = R.run("somatic-callable", "strelka2", str(tmp_path / "ref"))
        for f in ref:
            assert got[f] == ref[f], f


def test_somatic_callable_demo_shim_off(tmp_path):
    _need()
    got, err = R.run("somatic-callable", "strelka2_sx", str(tmp_path), env={"SX_SHIM_OFF": "1", "SX_SHIM_REPORT": "1"})
    assert _somatic_calls(err) in (0, -1), err[-500:]
    for f, want in GOLD.items():
        assert got[f] == want, f
