"""K3 global_align by launch route: sx_global_align_dev on the route batches of tests/k3_routes.py and on the bench's K3 batch, each timed
with CUDA events after warm-up; prints one JSON line with the median time per batch, the card's name and power limit.

The bench's K3 batch (tools/synth.cpp synth_ga: R 30-100, Q up to about 124) runs entirely in the group kernel, so the bench cannot show a
change to the warp kernel.  These batches can:
  warp4, warp2, warp1   the warp-kernel batches (4, 2 and 1 warps per CTA; some group-kernel problems ride along) under the production scores
  group_open-4097       the group-kernel shapes with open = -4097, past the group kernel's score limit: the warp kernel's register strips
  bench                 the K3 batch of bench.py's cfg2 step (3 haplotypes for half of 1M loci): the group kernel

    python tools/k3_leg.py [--reps R] [--warmup W] [--bench-loci N]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import bench  # noqa: E402
import k3_routes as K  # noqa: E402
from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200 import batch as B  # noqa: E402
from strelka_b200.api import Context, DevGaBatch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        name, pl = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
        return name, pl
    except Exception:
        return "unknown", "unknown"


def route_batch(pairs) -> B.GaBatch:
    return B.GaBatch([q for q, _ in pairs], [r for _, r in pairs], max_ops=max(len(q) + len(r) for q, r in pairs) + 2)


def bench_batch(n_loci: int, seed: int = 1) -> B.GaBatch:
    """bench.py's K3 batch (whole-path step, rank 0): synth_ga over 3 haplotypes for half of the loci, 24 cigar slots each"""
    synth = bench.load_synth()
    threads = os.cpu_count() or 8
    n = (n_loci // 2) * 3
    q_off, r_off = np.zeros(n + 1, np.uint32), np.zeros(n + 1, np.uint32)
    tot = synth.synth_ga(n, C.c_uint64(seed), threads, C.c_void_p(q_off.ctypes.data), C.c_void_p(r_off.ctypes.data), None, None)
    query, ref = np.zeros((tot & 0xFFFFFFFF) + 16, np.uint8), np.zeros((tot >> 32) + 16, np.uint8)
    synth.synth_ga(n, C.c_uint64(seed), threads, C.c_void_p(q_off.ctypes.data), C.c_void_p(r_off.ctypes.data), C.c_void_p(query.ctypes.data), C.c_void_p(ref.ctypes.data))
    gb = B.GaBatch.__new__(B.GaBatch)
    gb.n, gb.query, gb.ref, gb.query_off, gb.ref_off, gb.max_ops = n, query, ref, q_off, r_off, 24
    gb.c = A.SxGaBatch(n, A.ptr(query), A.ptr(ref), A.ptr(q_off), A.ptr(r_off), gb.max_ops)
    return gb


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--bench-loci", type=int, default=bench.WHOLE_PATH["cfg2"][0])
    a = ap.parse_args()
    optin = int(torch.cuda.get_device_properties(0).shared_memory_per_block_optin)
    routes = K.route_batches(optin)
    prod, big = K.score_set("active_region-ins1-del1"), K.score_set("open-4097-ins1-del1")
    runs = {name: (prod, route_batch(routes[name])) for name in ("warp4", "warp2", "warp1")}
    runs["group_open-4097"] = (big, route_batch(routes["group"]))
    runs["bench"] = (prod, bench_batch(a.bench_loci))
    ctx = Context(0)
    out = {}
    for name, (sc, gb) in runs.items():
        db = DevGaBatch(ctx, gb)
        for _ in range(a.warmup):
            ctx.global_align_dev(sc, db)
        ms = []
        for _ in range(a.reps):
            ctx.global_align_dev(sc, db)  # CUDA events around the call's launches on the compute stream
            ms.append(ctx.timing().kernel_ms)
        out[name] = {"problems": gb.n, "ms_median": float(np.median(ms)), "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms))}
        for b in list(db.bufs.values()) + [db.res, db.cigar]:
            b.free()
    ctx.close()
    name, pl = card()
    print(json.dumps({"leg": "k3_routes", "reps": a.reps, "warmup": a.warmup, "batches": out, "gpu": name, "power_limit": pl}))


if __name__ == "__main__":
    main()
