"""GPU: starling2_sx (integration/build_patched.py) routes updateIndelLocusWithSampleInfo's getVariantAlleleGroupGenotypeLhoodsForSample
through sx_indel_gl on the reference's bundled germline demo: it reports germline indel calls through the library, and its VCF bodies are
the unmodified binary's (tests/golden/demo_vcf_bodies.json; the demo has indel records at demo20:1148 and 3664)."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import run_demo as R  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method="thread")]
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "demo_vcf_bodies.json")))


def test_germline_demo_indels_through_the_library(tmp_path):
    if not os.path.exists(os.path.join(R.BIN, "starling2_sx")) or not os.path.isdir(R.DEMO):
        pytest.skip("oracle/_ref/bin or oracle/_ref/demo missing: run integration/build_patched.py where the reference tree exists")
    got, err = R.run("germline", "starling2_sx", str(tmp_path), env={"SX_SHIM_REPORT": "1"})
    line = [ln for ln in err.splitlines() if ln.startswith("sx_shim:")]
    assert line, err[-500:]
    fields = line[0].split(",")
    assert fields[-1].strip().endswith("germline indel calls")
    assert int(fields[-1].split()[0]) > 0, line[0]
    assert any("\t1148\t" in r or "\t3664\t" in r for f in got for r in got[f]), "the demo's indel records"
    for f, want in GOLD["germline"].items():
        assert got[f] == want, f
