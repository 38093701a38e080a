"""Freezes the unmodified starling2's VCF bodies on the reference's mitochondrial demo (integration/run_demo.py mito: chrM of
src/demo/dataMito with --call-continuous-vf) into tests/golden/mito_demo_vcf_bodies.json, with
  continuous_positions  the positions the continuous-frequency path sees: those inside genome-VCF records with a called GT (a position
                        with an empty raw column and no forced output is skipped and left as '.'; the demo forces none)
  equals_expected_results  whether the genome VCF body equals src/demo/expectedResultsMito/genome.vcf.gz (written in 2016)
Needs integration/build_patched.py to have built oracle/_ref/bin and staged oracle/_ref/demo."""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "integration"))
import run_demo as R  # noqa: E402


def continuous_positions(genome_body):
    n = 0
    for ln in genome_body:
        f = ln.split("\t")
        gt = f[9].split(":")[0]
        if gt.startswith("."):
            continue
        end = int(f[7].split("END=")[1].split(";")[0]) if "END=" in f[7] else int(f[1])
        n += end - int(f[1]) + 1
    return n


with tempfile.TemporaryDirectory() as d:
    bodies, _ = R.run("mito", "starling2", d)
expected = R.body(os.path.join(R.DEMO, "expected", "mito.genome.vcf.gz"))
out = {"mito": bodies, "continuous_positions": continuous_positions(bodies["seg.genome.S1.vcf"]),
       "equals_expected_results": bodies["seg.genome.S1.vcf"] == expected}
json.dump(out, open(os.path.join(ROOT, "tests", "golden", "mito_demo_vcf_bodies.json"), "w"), indent=1)
print({k: (len(v) if isinstance(v, list) else v) for k, v in bodies.items()}, out["continuous_positions"], out["equals_expected_results"])
