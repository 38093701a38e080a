"""Freezes the unmodified strelka2's output bodies on the reference's somatic demo with the callable regions written (integration/run_demo.py
somatic-callable: the somatic command line plus --somatic-callable-regions-file, as strelkaSomaticWorkflow.py issues it for
--outputCallableRegions) into tests/golden/somatic_callable_demo_bodies.json: snvs.vcf, indels.vcf and callable.bed.
Needs integration/build_patched.py to have built oracle/_ref/bin and staged oracle/_ref/demo.

    python tests/golden/make_somatic_callable_demo_golden.py"""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import run_demo as R  # noqa: E402

with tempfile.TemporaryDirectory() as d:
    bodies, _ = R.run("somatic-callable", "strelka2", d)
with open(os.path.join(ROOT, "tests", "golden", "somatic_callable_demo_bodies.json"), "w") as f:
    json.dump({"somatic-callable": bodies}, f, indent=1)
    f.write("\n")
print({k: len(v) for k, v in bodies.items()})
