"""The K6b leg: K6's records of two samples, resident in HBM, regrouped into K5b's per-locus read lists (sx_link_indel_reads_dev), alone and
followed by K5b (sx_somatic_indel_from_records_dev).  Records shaped like the cfg2 window workload: ~84 records per locus over both
samples.  What is timed is a CALL: CUDA events around everything the entry point enqueues, which includes its two small host round
trips (the scratch size, then the output totals) -- the stage cannot be enqueued back to back without them, so that is the time a
caller sees.  Median over repeated calls after a warm-up.  The algorithmic bytes are counted here from the batch.  Needs a CUDA device:
there is no fallback.

    python tools/indel_reads_leg.py [--loci 1000000] [--reps 5]"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def algorithmic_bytes(normal, tumor, loci, totals, n_pairs):
    """What one pass must move: every record slot in use once (32 B), the per-read arrays once, every entry once (24 B), the table rows,
    the offsets, and the (read id, record, read, order) scratch written and read once."""
    b = 0
    for s in (normal, tumor):
        b += int(s.n_rec[: s.n_reads].sum()) * 32 + s.n_reads * (4 + 4 + 2 + 2 + 1 + (4 if s.read_id is not None else 0)) + s.n_keys * 4
    b += int(totals[0]) * 24 + int(totals[1]) * 32 + loci.n_loci * (4 + 3 * 4 + 4)
    b += n_pairs * 4 * 4 * 2
    return b


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--loci", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        sys.exit("indel_reads_leg: no CUDA device (this leg is only measured on one)")
    import indel_reads_gen as G
    from strelka_b200 import _abi as A
    from strelka_b200.api import Context, DevIndelLoci, DevIndelReadsSample, DevSomaticIndelChain

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    n_gid = int(args.loci / 0.8)
    # ~1.7 scored records per read on a listed locus; depth chosen so both samples together hold ~84 record slots in use per locus
    normal, tumor, loci = G.synthetic_case(1, n_gid=n_gid, n_regions=n_gid // 3, depth=36.0, max_width=8, locus_frac=0.8, sub_frac=0.1)
    ctx = Context(0)
    dn, dt, dl = DevIndelReadsSample(ctx, normal), DevIndelReadsSample(ctx, tumor), DevIndelLoci(ctx, loci)
    cr, ca = G.caps(normal, tumor, loci)
    out = ctx.link_indel_reads_dev(dn, dt, dl, cr, ca)  # warm-up, and the totals
    n_pairs = sum(int(np.isin(G.entries_of(s)[0], loci.gid).sum()) for s in (normal, tumor))
    nbytes = algorithmic_bytes(normal, tumor, loci, out.totals, n_pairs)
    n_records = int(normal.n_rec.sum()) + int(tumor.n_rec.sum())

    from strelka_b200.api import DeviceArray
    import ctypes as C

    d = {k: DeviceArray(ctx, getattr(out, k).nbytes + 64) for k in ("alt_off", "alts", "read_off", "reads", "status", "totals")}
    c = A.SxIndelReadsOut(d["alt_off"].ptr, d["alts"].ptr, d["read_off"].ptr, d["reads"].ptr, d["status"].ptr, d["totals"].ptr, ca, cr)
    totals = np.zeros(2, np.uint32)
    link_ms = []
    for _ in range(args.reps + 1):
        ctx._chk(ctx.lib.sx_link_indel_reads_dev(ctx.h, C.byref(dn.c), C.byref(dt.c), C.byref(dl.c), C.byref(c), totals.ctypes.data))
        link_ms.append(ctx.timing().kernel_ms)  # CUDA events around the stage's launches, read after the stream is synchronised
    chain = DevSomaticIndelChain(ctx, dn, dt, loci)
    chain_ms = []
    for _ in range(args.reps + 1):
        chain.run()
        chain_ms.append(ctx.timing().kernel_ms)
    ctx.synchronize()
    link, both = float(np.median(link_ms[1:])), float(np.median(chain_ms[1:]))
    print(f"card: {card}")
    print(f"batch: {loci.n_loci} loci, {n_records} records in use, {n_pairs} entries scattered, {int(out.totals[0])} entries and {int(out.totals[1])} alternates written, "
          f"{int((out.status != 0).sum())} loci flagged")
    print(f"link alone (call time, two round trips inside):  median {link:.2f} ms of {args.reps} (min {min(link_ms[1:]):.2f}, max {max(link_ms[1:]):.2f}); algorithmic bytes {nbytes / 1e9:.3f} GB "
          f"-> {nbytes / link / 1e6:.1f} GB/s achieved (HBM-bound stage: no arithmetic; H100 SXM data sheet 3350 GB/s at 700 W)")
    print(f"link + K5b (call time):  median {both:.2f} ms of {args.reps} (min {min(chain_ms[1:]):.2f}, max {max(chain_ms[1:]):.2f}); K5b is bound by its serial fp64 "
          f"per-read sums, not by bytes")
    ctx.close()


if __name__ == "__main__":
    main()
