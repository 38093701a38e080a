#!/usr/bin/env python
"""integration/run_demo.py -- runs the reference's bundled demo (SURVEY.md Appendix B: the command lines the python2 workflows would issue) with a
binary from oracle/_ref/bin/ on the inputs staged under oracle/_ref/demo/ and returns the VCF bodies.
    python integration/run_demo.py somatic strelka2_sx /tmp/out      ->  /tmp/out/snvs.vcf, indels.vcf
    python integration/run_demo.py somatic-callable strelka2_sx /tmp/out  ->  the same and /tmp/out/callable.bed (--outputCallableRegions)
    python integration/run_demo.py germline starling2_sx /tmp/out    ->  /tmp/out/seg.variants.vcf, seg.genome.S1.vcf, seg.genome.S2.vcf
    python integration/run_demo.py mito starling2_sx /tmp/out        ->  /tmp/out/seg.variants.vcf, seg.genome.S1.vcf (chrM, --call-continuous-vf)"""
import gzip
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "oracle", "_ref", "bin")
DEMO = os.path.join(ROOT, "oracle", "_ref", "demo")


def body(path):
    op = gzip.open if path.endswith(".gz") else open
    with op(path, "rt") as f:
        return [ln for ln in f.read().splitlines() if not ln.startswith("#")]


def run(mode, binary, out, env=None, timeout=1200):
    os.makedirs(out, exist_ok=True)
    D, Cf = os.path.join(DEMO, "data"), os.path.join(DEMO, "config")
    exe = os.path.join(BIN, binary)
    if mode in ("somatic", "somatic-callable"):
        cmd = [exe, "--region", "demo20:1-5000", "--ref", f"{D}/demo20.fa", "--max-indel-size", "49", "--min-mapping-quality", "20", "--somatic-snv-rate", "0.0001",
               "--shared-site-error-rate", "0.0000000005", "--shared-site-error-strand-bias-fraction", "0.0", "--somatic-indel-rate", "0.000001", "--shared-indel-error-factor", "2.2",
               "--tier2-min-mapping-quality", "0", "--strelka-snv-max-filtered-basecall-frac", "0.4", "--strelka-snv-max-spanning-deletion-frac", "0.75",
               "--strelka-snv-min-qss-ref", "15", "--strelka-indel-max-window-filtered-basecall-frac", "0.3", "--strelka-indel-min-qsi-ref", "40", "--ssnv-contam-tolerance", "0.15",
               "--indel-contam-tolerance", "0.15", "--somatic-snv-scoring-model-file", f"{Cf}/somaticSNVScoringModels.json", "--somatic-indel-scoring-model-file",
               f"{Cf}/somaticIndelScoringModels.json", "--normal-align-file", f"{D}/NA12892_demo20.bam", "--tumor-align-file", f"{D}/NA12891_demo20.bam",
               "--somatic-snv-file", f"{out}/snvs.vcf", "--somatic-indel-file", f"{out}/indels.vcf", "--stats-file", f"{out}/stats.xml"]
        files = ["snvs.vcf", "indels.vcf"]
        if mode == "somatic-callable":  # strelkaSomaticWorkflow.py:125-128 with isOutputCallableRegions
            cmd += ["--somatic-callable-regions-file", f"{out}/callable.bed"]
            files.append("callable.bed")
    elif mode == "mito":
        # strelkaGermlineWorkflow.py:81-148 for the one chrM segment of runMitoWorkflowDemo.bash (--exome --callContinuousVf chrM): no EVS model
        # files, the default indel error model, the VF header and --call-continuous-vf
        M = os.path.join(DEMO, "dataMito")
        cmd = [exe, "--region", "chrM:1-16571", "--ref", f"{M}/chrM_hg19.fa", "--max-indel-size", "49", "--min-mapping-quality", "20", "--gvcf-output-prefix",
               f"{out}/seg.", "--gvcf-min-gqx", "15", "--gvcf-min-homref-gqx", "15", "--gvcf-max-snv-strand-bias", "10", "--enable-read-backed-phasing",
               "--stats-file", f"{out}/stats.xml", "--align-file", f"{M}/NA12878_chrM_200-200.bam", "--gvcf-include-header", "VF", "--call-continuous-vf",
               "--indel-error-models-file", f"{Cf}/indelErrorModel.json", "--theta-file", f"{Cf}/theta.json"]
        files = ["seg.variants.vcf", "seg.genome.S1.vcf"]
    else:
        cmd = [exe, "--region", "demo20:1-5000", "--ref", f"{D}/demo20.fa", "--max-indel-size", "49", "--min-mapping-quality", "20", "--gvcf-output-prefix", f"{out}/seg.",
               "--gvcf-min-gqx", "15", "--gvcf-min-homref-gqx", "15", "--gvcf-max-snv-strand-bias", "10", "--enable-read-backed-phasing", "--stats-file", f"{out}/stats.xml",
               "--snv-scoring-model-file", f"{Cf}/germlineSNVScoringModels.json", "--indel-scoring-model-file", f"{Cf}/germlineIndelScoringModels.json",
               "--align-file", f"{D}/NA12891_demo20.bam", "--align-file", f"{D}/NA12892_demo20.bam", "--indel-error-models-file", f"{Cf}/indelErrorModel.json",
               "--theta-file", f"{Cf}/theta.json"]
        files = ["seg.variants.vcf", "seg.genome.S1.vcf", "seg.genome.S2.vcf"]
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, env=e)
    if r.returncode != 0:
        raise RuntimeError(f"{binary} failed (rc {r.returncode}):\n{(r.stdout + r.stderr)[-3000:]}")
    return {f: body(os.path.join(out, f)) for f in files}, r.stderr


if __name__ == "__main__":
    res, err = run(sys.argv[1], sys.argv[2], sys.argv[3])
    for k, v in res.items():
        print(k, len(v), "records")
    print(err[-500:])
