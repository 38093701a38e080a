"""K2c site_continuous leg: times sx_site_continuous_dev with CUDA events at two sizes and reports the bytes it must read over that time
against the H100 SXM's 3.35 TB/s, with the card's name and power limit read in the same run.
  mito  a synthetic chrM (16 569 positions) at about 5 000 calls per column, with 1, 2 and 3 samples
  cfg2  200 000 positions at about 30 calls per column, one sample (the germline window pass's column shape)
The time is the whole stage between two events (count, scan, the record count's host round trip, write), the best of --reps after a warm-up.
Usage: python tools/continuous_leg.py [--reps 10]"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200 import api  # noqa: E402
from strelka_b200 import batch as B  # noqa: E402


def columns(rng, ref_id, depth):
    """one sample's columns: Poisson depths, the reference base with a minor allele at a per-site fraction, 1 % ANY, 3 % filtered"""
    n_sites = ref_id.size
    d = rng.poisson(depth, n_sites).astype(np.uint32)
    off = np.zeros(n_sites + 1, np.uint32)
    off[1:] = np.cumsum(d)
    n = int(off[-1])
    site = np.repeat(np.arange(n_sites), d)
    af = rng.choice([0.0, 0.0, 0.005, 0.02, 0.3, 1.0], n_sites)[site]
    base = np.where(rng.random(n) < af, (ref_id[site] + 1) % 4, ref_id[site])
    base = np.where(rng.random(n) < 0.01, 4, base)
    filt = rng.random(n) < 0.03
    calls = B.pack_call(rng.integers(2, 41, n), base, rng.random(n) < 0.5, rng.random(n) < 0.1, filt, filt)
    return off, np.asarray(calls, np.uint16)


def run(ctx, name, n_sites, depth, S, reps, seed=0):
    rng = np.random.default_rng(seed)
    ref_id = rng.integers(0, 4, n_sites)
    ref = np.frombuffer("".join("ACGT"[i] for i in ref_id).encode(), np.uint8)
    samples = [B.PileupBatch(*columns(rng, ref_id, depth), ref) for _ in range(S)]
    hb = B.ContBatch(samples, 0)
    db = api.DevContBatch(ctx, hb)
    best = None
    for r in range(reps + 1):
        out = ctx.site_continuous_dev(db)
        ms = ctx.timing().kernel_ms
        if r:
            best = ms if best is None else min(best, ms)
    n_calls = sum(p.n_calls for p in samples)
    n_rec = int(out.totals[0])
    read = n_calls * 2 + S * (n_sites + 1) * 4 + n_sites
    written = n_rec * (A.CONT_LOCUS_DT.itemsize + S * A.CONT_SAMPLE_DT.itemsize) + (n_sites + 1) * 4
    gbs = read / (best * 1e-3) / 1e9
    print(f"{name:5s} S={S} sites={n_sites} calls={n_calls} records={n_rec}: {best:.3f} ms, {read / 1e6:.1f} MB read, {written / 1e6:.1f} MB written, "
          f"{gbs:.0f} GB/s read = {100 * gbs / 3350:.1f} % of 3.35 TB/s")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {card}")
    ctx = api.Context(0)
    for S in (1, 2, 3):
        run(ctx, "mito", 16569, 5000.0, S, args.reps)
    run(ctx, "cfg2", 200000, 30.0, 1, args.reps)
    ctx.close()


if __name__ == "__main__":
    main()
