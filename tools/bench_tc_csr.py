#!/usr/bin/env python3
"""One-shot triangle count of a host undirected CSR (graph_b200.triangle_count_csr / gb_triangle_count_csr_u32)
against the twin path and the bus.

The CSR of an R-MAT graph (Sorted, seed 42; the twin's csr()) is copied to pinned host arrays, then three
things are run in one process, alternated, after warm-up runs:
  upload    a plain H2D copy of the offsets and targets (4(n+1) + 4m bytes), timed with CUDA events;
  one-shot  triangle_count_csr(offsets, targets): offsets first, targets in row-aligned chunks, each chunk
            checked and counted as soon as it has landed;
  twin      Graph.from_csr(offsets, targets) + global_triangle_count(): the full upload and checks, then the
            first count, which checks the row order once and counts in one launch.
Wall times (time.perf_counter around each call, device synchronised) are reported as best / median, with the
device times the calls report (CUDA events): the one-shot's upload and total, the twin's count.  The counts of
both paths must be equal.  Prints one JSON line.

    python tools/bench_tc_csr.py [--scale 22] [--runs 5] [--warmup 2] [--json out.json]
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import bench  # noqa: E402  (pinned host arrays)
import graph_b200 as gb  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0), out


def stats(ts):
    return {"best_ms": min(ts), "median_ms": statistics.median(ts), "runs": len(ts)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=22)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tc_csr needs a CUDA device")
    g = gb.Graph.rmat(args.scale, seed=42, layout=gb.Layout.Sorted)
    off_src, tgt_src = g.csr()
    n, m = len(off_src) - 1, len(tgt_src)
    keep_off, off = bench.pinned_empty(n + 1, np.uint32)
    keep_tgt, tgt = bench.pinned_empty(m, np.uint32)
    off[:], tgt[:] = off_src, tgt_src
    del g, off_src, tgt_src
    d_off = torch.empty(n + 1, dtype=torch.int32, device="cuda")
    d_tgt = torch.empty(m, dtype=torch.int32, device="cuda")
    h_off, h_tgt = torch.from_numpy(off.view(np.int32)), torch.from_numpy(tgt.view(np.int32))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    dev = {"upload": [], "one_shot_upload": [], "one_shot_total": [], "twin_count": []}
    counts = {}

    def upload():
        ev[0].record()
        d_off.copy_(h_off, non_blocking=True)
        d_tgt.copy_(h_tgt, non_blocking=True)
        ev[1].record()
        ev[1].synchronize()
        dev["upload"].append(ev[0].elapsed_time(ev[1]))

    def one_shot():
        r = gb.triangle_count_csr(off, tgt)
        dev["one_shot_upload"].append(r.info["upload_ms"])
        dev["one_shot_total"].append(r.info["total_ms"])
        counts["one_shot"] = r.triangles
        return r

    twin_parts = {"from_csr": [], "count": []}

    def twin():
        t0 = time.perf_counter()
        tg = gb.Graph.from_csr(off, tgt)
        t1 = time.perf_counter()
        counts["twin"] = tg.global_triangle_count().triangles
        t2 = time.perf_counter()
        twin_parts["from_csr"].append(1e3 * (t1 - t0))
        twin_parts["count"].append(1e3 * (t2 - t1))
        dev["twin_count"].append(tg.last_timing()["total_ms"])
        del tg

    paths = {"upload": upload, "one_shot": one_shot, "twin": twin}
    for _ in range(args.warmup):
        for fn in paths.values():
            fn()
    for v in list(dev.values()) + list(twin_parts.values()):
        v.clear()
    times = {k: [] for k in paths}
    info = None
    for _ in range(args.runs):  # alternated
        for k, fn in paths.items():
            t, out = wall(fn)
            times[k].append(t)
            if k == "one_shot":
                info = out.info
    res = {"card": card(), "scale": args.scale, "n": n, "m": m, "bytes": 4 * (n + 1) + 4 * m,
           "wall": {k: stats(v) for k, v in times.items()},
           "device": {k: stats(v) for k, v in dev.items()},
           "twin_parts": {k: stats(v) for k, v in twin_parts.items()},
           "chunks": info["chunks"], "chunk_entries": info["chunk_entries"],
           "sorted_chunks": info["sorted_chunks"], "list_chunks": info["list_chunks"],
           "triangles": counts["one_shot"], "counts_equal": counts["one_shot"] == counts["twin"]}
    print(json.dumps(res))
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(res, indent=1))
    if not res["counts_equal"]:
        sys.exit("the one-shot and twin counts differ")


if __name__ == "__main__":
    main()
