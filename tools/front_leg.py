#!/usr/bin/env python
"""The front of the window pass on one cfg2 window: sx_process_window_dev after a warm-up, the per-stage device times of
sx_last_window_timing (the median of several passes) for the per-read stages at the front (prep, K7g gates, K7a keys, K7b link,
K9 choose) beside the rest, and the step's total.  Prints one JSON line.

    python tools/front_leg.py [--cells 50000] [--runs 7] [--warmup 2] [--profile DIR]

--profile DIR: one more pass under torch.profiler (CUDA activities) in a run of its own; the Chrome trace goes to DIR and the JSON line
gains each front-end stage's kernels (device ms of one pass, by kernel name).  The timed passes are taken with the profiler off."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200.api import Context, DevWindow  # noqa: E402
import window_workload as WW  # noqa: E402

FRONT = ("prep", "k7g_gates", "k7a_keys", "k7b_link", "k9_choose")
# the kernels of each front-end stage, by a prefix of their (mangled or plain) names
FRONT_KERNELS = {"prep": ("sxp_prep", "sx_read_index"), "k7g_gates": ("k7g_", "sxp_submapped"), "k7a_keys": ("k7a_", "k7_active"), "k7b_link": ("k8_",),
                 "k9_choose": ("k9_",)}


def gpu_name() -> dict:
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power, clock = (x.strip() for x in q.strip().splitlines()[0].split(","))
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"name": "unknown", "error": str(e)}


def profile_pass(dw: DevWindow, out_dir: str) -> dict:
    import torch
    from torch.profiler import ProfilerActivity, profile

    os.makedirs(out_dir, exist_ok=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        dw.run()
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(out_dir, "front_leg.pt.trace.json"))
    per_kernel = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if t > 0:
            per_kernel[e.key] = per_kernel.get(e.key, 0.0) + t / 1e3
    by_stage = {s: {} for s in FRONT}
    for k, ms in per_kernel.items():
        plain = k.replace("(anonymous namespace)::", "").replace("void ", "").split("(")[0].split("<")[0]
        for s, pre in FRONT_KERNELS.items():
            if any(p in plain for p in pre):
                by_stage[s][plain[:80]] = round(by_stage[s].get(plain[:80], 0.0) + ms, 4)
    top = sorted(per_kernel.items(), key=lambda kv: -kv[1])[:25]
    short = lambda k: k.replace("(anonymous namespace)::", "").replace("void ", "").split("(")[0].split("<")[0][:80]  # noqa: E731
    return {"front_kernels_ms": by_stage, "top_kernels_ms": {short(k): round(v, 4) for k, v in top}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=50_000, help="candidate loci of the window (cfg2: 50k)")
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    ap.add_argument("--profile", metavar="DIR", default="")
    args = ap.parse_args()
    import torch

    torch.cuda.init()
    ctx = Context(0)
    w = WW.make_window(WW.load_synth(), args.cells, args.seed, tile=0, qual_bits=4)
    dw = DevWindow(ctx, w, keep_outputs=False)
    for _ in range(args.warmup):
        dw.run()
    runs = [dw.run() for _ in range(args.runs)]
    med = {k: float(np.median([r[k] for r in runs])) for k in A.SX_WIN_STAGE_NAMES}
    res = {"leg": "front", "gpu": gpu_name(), "cells": args.cells, "reads": w.n_reads, "runs": args.runs, "stage_ms_median": {k: round(v, 4) for k, v in med.items()},
           "front_ms": round(sum(med[k] for k in FRONT), 4), "front4_ms": round(sum(med[k] for k in ("prep", "k7g_gates", "k7a_keys", "k9_choose")), 4),
           "pass_ms": round(sum(med.values()), 4)}
    if args.profile:
        res.update(profile_pass(dw, args.profile))
    dw.free()
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
