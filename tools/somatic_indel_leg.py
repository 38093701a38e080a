"""K5b somatic_indel leg: sx_somatic_indel_dev on a seeded synthetic batch of user scale (default 10^6 candidate indels, normal ~40 and
tumor ~60 reads, 20 % tier2, 0-2 alternates per read), timed with CUDA events after warm-up; prints one JSON line with loci/s, the card's
name and power limit.  A seeded subset of the outputs is checked against the scalar oracle byte for byte; where oracle/_ref is built the
reference's own get_somatic_indel is timed on one host core for a slice of the same batch (the time inside that function only), for context.

    python tools/somatic_indel_leg.py [--loci N] [--reps R] [--check M]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import sindel_gen as G  # noqa: E402
from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200 import batch as B  # noqa: E402
from strelka_b200.api import Context, DevSomaticIndelBatch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, pl = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
        return name, pl
    except Exception:
        return "unknown", "unknown"


def subset(sb: B.SomaticIndelBatch, idx: np.ndarray) -> B.SomaticIndelBatch:
    """The loci idx of sb as a batch of their own (same error table)."""
    alt_n = np.diff(sb.alt_off)[idx]
    rd = np.diff(sb.read_off).reshape(-1, 2)[idx]
    alts = np.concatenate([sb.alts[sb.alt_off[i]: sb.alt_off[i + 1]] for i in idx]) if alt_n.sum() else np.zeros(0, A.INDEL_KEY_DT)
    reads = np.concatenate([sb.reads[sb.read_off[2 * i]: sb.read_off[2 * i + 2]] for i in idx])
    alt_off = np.concatenate([[0], np.cumsum(alt_n)]).astype(np.uint32)
    read_off = np.concatenate([[0], np.cumsum(rd.ravel())]).astype(np.uint32)
    return B.SomaticIndelBatch(sb.key[idx], sb.is_forced_output[idx], sb.err_idx[idx], sb.err_prob, alt_off, alts, read_off, reads)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loci", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--check", type=int, default=20_000)
    ap.add_argument("--ref-loci", type=int, default=20_000)
    a = ap.parse_args()
    rng = np.random.default_rng(2024)
    sb = G.random_somatic_indel_batch(rng, a.loci, normal_depth=40.0, tumor_depth=60.0, tier2_frac=0.2)
    o = A.default_sindel_opts()
    ctx = Context(0)
    db = DevSomaticIndelBatch(ctx, sb)
    for _ in range(a.warmup):
        ctx.somatic_indel_dev(db, o)
    ms = []
    for _ in range(a.reps):
        ctx.somatic_indel_dev(db, o)
        ms.append(ctx.timing().kernel_ms)
    got = db.download()
    idx = np.sort(np.random.default_rng(5).choice(a.loci, min(a.check, a.loci), replace=False))
    want = G.ox_somatic_indel(o, subset(sb, idx))
    ok = got[idx].tobytes() == want.tobytes()
    name, pl = card()
    med = float(np.median(ms))
    res = {"leg": "somatic_indel", "loci": a.loci, "reads": int(sb.read_off[-1]), "kernel_ms_median": med, "kernel_ms_all": ms,
           "loci_per_s": a.loci / (med / 1e3), "calls": int(got["is_output"].sum()), "checked_loci": int(idx.size), "oracle_match": ok,
           "gpu": name, "power_limit": pl}
    if G.have_ref():
        rs = subset(sb, np.arange(min(a.ref_loci, a.loci)))
        res["reference_one_core_loci_per_s"] = rs.n_loci / G.ref_somatic_indel_seconds(o, rs)  # time inside get_somatic_indel only
    print(json.dumps(res))
    ctx.close()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
