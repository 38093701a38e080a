#!/usr/bin/env python
"""Times K4m (pile-up scoring metrics) on cfg2 windows: python tools/pileup_metrics_leg.py [--cells 50000] [--steps 5] [--warmup 2]

One cfg2-shaped window (bench.py's whole-path configuration: 50,000 cells a window, 20 windows a 1M-locus step) through
sx_process_window_metrics_dev in each mode.  The metrics stage's device time comes from the pass's own stage events (CUDA events on the
compute stream); the K4 pile-up stage of the same pass is printed beside it.  One JSON line."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import window_workload as WW  # noqa: E402
from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200.api import Context, DevWindow  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=50_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    windows_per_step = 1_000_000 // args.cells
    w = WW.make_window(WW.load_synth(), args.cells, args.seed)
    ctx = Context(0)
    res = {"cells": args.cells, "windows_per_cfg2_step": windows_per_step, "reads": w.n_reads, "sites": w.n_sites}
    for name, mode in (("mapq", A.SX_PM_MAPQ), ("germline", A.SX_PM_GERMLINE), ("somatic", A.SX_PM_SOMATIC)):
        dw = DevWindow(ctx, w, keep_outputs=False, metrics=mode)
        for _ in range(args.warmup):
            dw.run()
        st = [dw.run() for _ in range(args.steps)]
        dw.free()
        m = float(np.median([s["k4m_metrics"] for s in st]))
        k4 = float(np.median([s["k4_pileup"] for s in st]))
        res[name] = {"metrics_ms_per_window": m, "k4_pileup_ms_per_window": k4, "metrics_ms_per_cfg2_step": m * windows_per_step}
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
