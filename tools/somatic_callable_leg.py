#!/usr/bin/env python
"""K2b's callable mode (isComputeNonSomatic, strelka2 --outputCallableRegions) against the default mode, on the GPU:
  k2b     sx_site_gl_somatic_dev and sx_site_gl_somatic_callable_dev on tools/site_legs.py's k2b workload (cfg3: 500k tumor/normal sites,
          60x / 30x), resident in HBM; then sx_somatic_callable_regions_dev on the callable-mode records
  window  sx_process_somatic_window_dev in both modes on one cfg2-shaped two-sample window (tools/somatic_window_leg.py's), and the region
          stage on the pass's site_snv
Every time is a CUDA-event time on the context's compute stream, the median of --reps after a warm-up.  Each pair of outputs is compared: the
callable-mode records equal the default mode's wherever the default computed them (and on the window, the SNV records), but for
nonsomatic_qphred.  The card's name and power limit are read in the same run.
Usage: python tools/somatic_callable_leg.py [--reps 10] [--cells 50000]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import somatic_window_leg as SWL  # noqa: E402
import window_workload as WW  # noqa: E402
from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200 import batch as B  # noqa: E402
from strelka_b200.api import Context, DeviceArray, DevPileupBatch, DevSomaticWindow  # noqa: E402


def med(x):
    return float(np.median(x))


def same_but_nqss(callable_rec: np.ndarray, default_rec: np.ndarray) -> bool:
    """the callable-mode records equal the default mode's where the default computed a record, but for nonsomatic_qphred"""
    m = default_rec["is_computed"] == 1
    a = callable_rec[m].copy()
    a["nonsomatic_qphred"] = 0
    return a.tobytes() == default_rec[m].tobytes()


def k2b(ctx, reps, n=500_000):
    synth = WW.load_synth()
    thr = max(1, len(os.sched_getaffinity(0)))

    def pile(depth, mode):  # (tools/site_legs.py's k2b inputs)
        off = np.zeros(n + 1, np.uint32)
        nc = synth.synth_pileups(n, C.c_double(depth), mode, C.c_uint64(5), thr, C.c_void_p(off.ctypes.data), None, None)
        calls, ref = np.zeros(nc + 8, np.uint16), np.zeros(n, np.uint8)
        synth.synth_pileups(n, C.c_double(depth), mode, C.c_uint64(5), thr, C.c_void_p(off.ctypes.data), C.c_void_p(calls.ctypes.data), C.c_void_p(ref.ctypes.data))
        return off, calls, ref

    noff, ncalls, ref = pile(30.0, 1)
    toff, tcalls, _ = pile(60.0, 2)
    dn, dt = DevPileupBatch(ctx, B.PileupBatch(noff, ncalls, ref)), DevPileupBatch(ctx, B.PileupBatch(toff, tcalls, ref))
    outs = {m: DeviceArray(ctx, n * A.SSNV_RESULT_DT.itemsize + 64) for m in ("default", "callable")}
    run = {"default": ctx.site_gl_somatic_dev, "callable": ctx.site_gl_somatic_callable_dev}
    ms = {m: [] for m in run}
    for i in range(reps + 2):
        for m, f in run.items():
            f(dn, dt, None, outs[m])
            if i >= 2:
                ms[m].append(ctx.timing().kernel_ms)
    got = {m: outs[m].download(A.SSNV_RESULT_DT, n) for m in run}
    cap = (n + 1) // 2
    rb, re = DeviceArray(ctx, 4 * cap + 64), DeviceArray(ctx, 4 * cap + 64)
    rms = []
    for i in range(reps + 2):
        n_reg = ctx.somatic_callable_regions_dev(outs["callable"], n, 0, rb, re, cap)
        if i >= 2:
            rms.append(ctx.timing().kernel_ms)
    wb, we = B.somatic_callable_regions(got["callable"], 0)
    regions_same = bool(np.array_equal(rb.download(np.int32, n_reg), wb) and np.array_equal(re.download(np.int32, n_reg), we))
    for x in list(outs.values()) + [rb, re] + list(dn.bufs.values()) + list(dt.bufs.values()):
        x.free()
    c, d = got["callable"], got["default"]
    return {"what": f"K2b on {n} tumor/normal sites (cfg3: 60x / 30x), resident in HBM", "default_ms": med(ms["default"]), "callable_ms": med(ms["callable"]),
            "callable_over_default": med(ms["callable"]) / med(ms["default"]), "regions_ms": med(rms), "n_regions": int(n_reg),
            "computed": {"default": int(d["is_computed"].sum()), "callable": int(c["is_computed"].sum())},
            "callable_positions": int((~((c["qphred"] < 15) & (c["nonsomatic_qphred"] < 15))).sum()),
            "records_same_but_nqss": same_but_nqss(c, d), "regions_equal_host_builder": regions_same}


def window(ctx, reps, cells, seed=7):
    w = WW.make_window(WW.load_synth(), cells, seed)
    normal, tumor, loci, key_gid, forced = SWL.two_sample_window(w, seed)
    opts = A.default_sindel_opts()
    opts.useTier2Evidence = 0
    sw = {m: DevSomaticWindow(ctx, normal, tumor, loci, [key_gid, key_gid], snv_forced=forced, opts=opts, records_only=True, compute_nonsomatic=(m == "callable"))
          for m in ("default", "callable")}
    ms = {m: [] for m in sw}
    k2b_ms = {m: [] for m in sw}
    rms = []
    for i in range(reps + 2):
        for m, x in sw.items():
            ctx.timer_mark(0)
            st = x.run()
            ctx.timer_mark(1)
            if i >= 2:
                ms[m].append(ctx.timer_elapsed_ms())
                k2b_ms[m].append(st["k2b_site_snv"])
        reg = sw["callable"].callable_regions()
        if i >= 2:
            rms.append(ctx.timing().kernel_ms)
    got = {m: x.download() for m, x in sw.items()}
    a = got["callable"]["snv_calls"].copy()
    a["r"]["nonsomatic_qphred"] = 0
    same = a.tobytes() == got["default"]["snv_calls"].tobytes() and got["callable"]["indel_calls"].tobytes() == got["default"]["indel_calls"].tobytes()
    for x in sw.values():
        x.free()
    return {"what": f"somatic window pass, one cfg2-shaped window ({normal.n_reads} + {tumor.n_reads} reads, {normal.n_sites} positions)",
            "default_ms": med(ms["default"]), "callable_ms": med(ms["callable"]), "k2b_stage_default_ms": med(k2b_ms["default"]),
            "k2b_stage_callable_ms": med(k2b_ms["callable"]), "regions_ms": med(rms), "n_regions": int(reg[0].size),
            "callable_positions": int((reg[1] - reg[0]).sum()), "records_same_but_nqss": bool(same)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--cells", type=int, default=50_000)
    args = ap.parse_args()
    ctx = Context(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    out = {"gpu": q[0] if q else "unknown", "k2b": k2b(ctx, args.reps), "window": window(ctx, args.reps, args.cells)}
    ctx.close()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
