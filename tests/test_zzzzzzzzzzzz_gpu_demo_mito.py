"""GPU: starling2_sx (integration/build_patched.py) routes process_pos_snp_continuous through sx_site_continuous (K2c) and the continuous
indel GQ through sx_cont_qscore.  On the reference's mitochondrial demo (integration/run_demo.py mito: chrM with --call-continuous-vf) its
VCF bodies are the unmodified binary's (tests/golden/mito_demo_vcf_bodies.json), line for line, with the route on and with SX_SHIM_OFF=1.
With the route on, every position the continuous path sees goes through K2c: the report's counter equals the positions with a non-empty raw
column, 199 (chrM:101-299, read off the unmodified binary's genome VCF by tests/golden/make_mito_demo_golden.py; the demo forces none)."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import run_demo as R  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "mito_demo_vcf_bodies.json")))
POSITIONS = 199


def _need():
    if not os.path.exists(os.path.join(R.BIN, "starling2_sx")) or not os.path.isdir(os.path.join(R.DEMO, "dataMito")):
        pytest.skip("oracle/_ref/bin or oracle/_ref/demo/dataMito missing: run integration/build_patched.py where the reference tree exists")


def _continuous_calls(err):
    """the counter at the end of the report line (it is appended only when the route ran: no field is 0)"""
    line = [ln for ln in err.splitlines() if ln.startswith("sx_shim:")]
    assert line, err[-500:]
    last = line[0].split(",")[-1].strip()
    if not last.endswith("continuous site calls"):
        assert last.endswith("germline indel calls"), line[0]
        return 0
    return int(last.split()[0])


def test_mito_demo_through_the_library(tmp_path):
    _need()
    assert GOLD["continuous_positions"] == POSITIONS
    got, err = R.run("mito", "starling2_sx", str(tmp_path), env={"SX_SHIM_REPORT": "1"})
    assert _continuous_calls(err) == POSITIONS
    assert any("\t150\t" in r for r in got["seg.variants.vcf"]), "the demo's continuous-VF SNVs"
    for f, want in GOLD["mito"].items():
        assert got[f] == want, f


def test_mito_demo_shim_off(tmp_path):
    _need()
    got, err = R.run("mito", "starling2_sx", str(tmp_path), env={"SX_SHIM_OFF": "1", "SX_SHIM_REPORT": "1"})
    assert _continuous_calls(err) == 0
    for f, want in GOLD["mito"].items():
        assert got[f] == want, f
