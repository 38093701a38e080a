"""Leg: K6's records of one cfg2-shaped window pass -> germline indel genotype likelihoods.

The device route is sx_indel_gl_from_records_dev (DevGermlineIndelChain): the K6g link and K5 on the records the window pass left in HBM, timed
with CUDA events on the compute stream.  The host route is what a caller does without it: download the records, build K5's batch with the
host builder (batch.link_allele_groups) and call K5's host entry; it is timed on the wall clock.  Both give the same bytes (checked).  The
groups are formed from the window's entries: every INDEL entry alone, and each pair of overlapping INDEL entries with the next entry as its
contrast.  The bytes floor counts what the link must move at least: every record slot read once, each named id's triples written and read
(12 bytes), each supporting read's A+1 floats and 5 bytes written.  The card's name and power limit are read in the same run.

  python tools/germline_indel_leg.py [--cells 20000] [--steps 5] [--warmup 2] [--seed 7]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

from strelka_b200 import _abi as A  # noqa: E402
from strelka_b200 import batch as B  # noqa: E402

import somatic_window_leg as SW  # noqa: E402


def window_groups(w: B.WindowBatch, seed: int) -> B.AlleleGroups:
    """every INDEL entry of the window as a singleton group, and every pair of consecutive INDEL entries whose deleted ranges overlap (or that
    sit at one position) as a two-allele group with the entry after them as contrast; ploidy 2, every fifth group 1.  Ids are window entry
    indices (key_gid = arange)."""
    keys = w.a["keys"][: w.n_keys]
    ind = np.nonzero(keys["type"] == A.SX_INDEL_TYPE_INDEL)[0]
    al = [[int(k)] for k in ind]
    co = [[] for _ in ind]
    for i in range(ind.size - 1):
        a, b = ind[i], ind[i + 1]
        if keys["pos"][b] <= keys["pos"][a] + max(int(keys["del_len"][a]), 0):
            al.append([int(a), int(b)])
            co.append([int(ind[i + 2])] if i + 2 < ind.size else [])
    ploidy = np.where(np.arange(len(al)) % 5 == 4, 1, 2).astype(np.uint8)
    gid_key = keys if keys.size else np.zeros(1, A.INDEL_KEY_DT)
    return B.AlleleGroups.from_lists(al, co, ploidy, gid_key)


def host_sample(w: B.WindowBatch, recs, n_rec) -> B.IndelReadsSample:
    """the window's sample on the host, with the records its pass wrote"""
    sb = SimpleNamespace(n_regions=w.n_regions, n_reads=w.n_reads, n_keys=w.n_keys, non_ambig=SW.non_ambig_of(w),
                         **{k: w.a[k] for k in ("region_read_off", "region_key_off", "rec_off", "read_len", "read_flags")})
    return B.IndelReadsSample(sb, recs, np.append(n_rec, 0).astype(np.uint32), np.arange(w.n_keys, dtype=np.uint32))


def host_route(ctx, dw, groups: B.AlleleGroups):
    """download + host builder + K5's host entry: (results, status)"""
    w = dw.w
    recs = dw.obufs["recs"].download(A.READ_INDEL_SCORE_DT, dw.n_slots + 1)
    n_rec = dw.obufs["n_rec"].download(np.uint32, w.n_reads)
    linked = B.link_allele_groups(host_sample(w, recs, n_rec), groups)
    res = ctx.indel_gl(linked.batch())
    st = linked.status[: groups.n_groups].copy()
    res[st != 0] = np.zeros(1, A.INDEL_RESULT_DT)
    return res, st, linked


def bytes_floor(dw, groups: B.AlleleGroups, linked: B.AlleleGroupReadsOut) -> int:
    """record slots read once, named ids' triples written and read, the output written"""
    w = dw.w
    recs = dw.obufs["recs"].download(A.READ_INDEL_SCORE_DT, dw.n_slots + 1)
    n_rec = dw.obufs["n_rec"].download(np.uint32, w.n_reads)
    s = host_sample(w, recs, n_rec)
    n_records = int(n_rec.sum())
    named = np.unique(np.concatenate([groups.allele_gid, groups.contrast_gid]))
    cnt_total = 0
    if named.size:
        import indel_reads_gen as G

        g, _ = G.entries_of(s)
        cnt_total = int(np.isin(g, named).sum())
    out = int(linked.totals[1]) * 4 + int(linked.totals[0]) * 5 + groups.n_groups * 13
    return n_records * A.READ_INDEL_SCORE_DT.itemsize + 2 * 12 * cnt_total + out


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip()
    except Exception as e:  # (the numbers stay unlabelled rather than wrong)
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, default=20_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=7)
    args = ap.parse_args()
    import window_workload as WW
    from strelka_b200.api import Context, DevGermlineIndelChain, DevIndelReadsSample, DevWindow

    w = WW.make_window(WW.load_synth(), args.cells, args.seed)
    groups = window_groups(w, args.seed)
    ctx = Context(0)
    dw = DevWindow(ctx, w)
    dw.run()
    sample = DevIndelReadsSample.from_window(ctx, dw, np.arange(w.n_keys, dtype=np.uint32), None, SW.non_ambig_of(w))
    chain = DevGermlineIndelChain(ctx, sample, groups)
    for _ in range(args.warmup):
        chain.run()
        host_route(ctx, dw, groups)
    dev_ms, host_ms = [], []
    for _ in range(args.steps):
        ctx.timer_mark(0)
        chain.run()
        ctx.timer_mark(1)
        dev_ms.append(ctx.timer_elapsed_ms())
        t0 = time.perf_counter()
        want, want_st, linked = host_route(ctx, dw, groups)
        host_ms.append(1e3 * (time.perf_counter() - t0))
    got, st = chain.download()
    assert got.tobytes() == want.tobytes() and st.tobytes() == want_st.tobytes(), "device chain and host route differ"
    floor = bytes_floor(dw, groups, linked)
    med = float(np.median(dev_ms))
    print(json.dumps({"leg": "germline_indel", "card": card(), "cells": args.cells, "reads": w.n_reads, "records": int(dw.obufs["n_rec"].download(np.uint32, w.n_reads).sum()),
                      "groups": groups.n_groups, "supporting_reads": int(linked.totals[0]), "device_ms": [round(x, 3) for x in dev_ms],
                      "host_route_ms": [round(x, 1) for x in host_ms], "bytes_floor": floor, "device_GBps_of_floor": round(floor / (med * 1e6), 2) if med else None,
                      "identical": True}))
    dw.free()
    ctx.close()


if __name__ == "__main__":
    main()
