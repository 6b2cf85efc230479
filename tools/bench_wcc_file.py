#!/usr/bin/env python3
"""WCC of a graph file in one pass (graph_b200.wcc_file / gb_wcc_file_u32) against load + wcc on the same file.

For each R-MAT scale (seed 42, 16 edges per node) a Graph500 file is written to a local directory and read once to
warm the page cache.  Two paths are then run in one process, alternated, after warm-up runs:
  one-pass   wcc_file(path): the file streams through the pinned ring and every chunk's edges are linked on the
             device as they are decoded; no edge array or CSR is built;
  load+wcc   DiGraph.load(path) + wcc(): the device edge arrays, both CSRs (Unsorted build), then Afforest.
Wall times (time.perf_counter around each synchronised call) are reported as best / median, with the file's GB/s at
the best time, the one-pass call's H2D bytes and peak device bytes (wcc_file_info) and whether the labels are
bit-equal.  The card name and power limit are read in the same run, since they are part of every number.

    python tools/bench_wcc_file.py [--scales 24 26] [--runs 5] [--warmup 2] [--dir /local/disk] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import graph_b200 as gb  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def stats(ts):
    return {"best_ms": 1e3 * min(ts), "median_ms": 1e3 * statistics.median(ts), "runs": len(ts)}


def write_rmat_graph500(path, scale):
    """The RMAT-`scale` edges written in slices, so that the host never holds more than one slice."""
    m = 16 << scale
    step = 1 << 26
    src = np.empty(min(step, m), np.uint32)
    dst = np.empty(min(step, m), np.uint32)
    raw = np.empty(12 * len(src), np.uint8)
    with open(path, "wb") as f:
        for first in range(0, m, step):
            k = min(step, m - first)
            gb.check(gb.lib.gb_rmat_edges(0, scale, 42, first, k, gb._ptr(src), gb._ptr(dst)))
            gb.check(gb.lib.gb_graph500_encode(gb._ptr(src), gb._ptr(dst), k, gb._ptr(raw)))
            f.write(raw[:12 * k].tobytes())


def warm(path):
    with open(path, "rb") as f:
        while f.read(1 << 26):
            pass


def measure(path, runs, warmup):
    size = os.path.getsize(path)
    warm(path)
    one = lambda: gb.wcc_file(path).components()  # noqa: E731

    def two():
        g = gb.DiGraph.load(path)
        out = g.wcc().components()
        del g
        return out
    for _ in range(warmup):
        one()
        two()
    t_one, t_two = [], []
    for _ in range(runs):
        t, a = wall(one)
        t_one.append(t)
        info = gb.wcc_file_info()
        t, b = wall(two)
        t_two.append(t)
    s1, s2 = stats(t_one), stats(t_two)
    return {"file_bytes": size, "node_count": info["node_count"], "edges": info["edges"],
            "chunks": info["chunks"], "h2d_bytes": info["h2d_bytes"], "device_bytes": info["device_bytes"],
            "device_ms": info["total_ms"], "one_pass": s1, "load_wcc": s2,
            "one_pass_file_GBps": size / (s1["best_ms"] * 1e6), "load_wcc_file_GBps": size / (s2["best_ms"] * 1e6),
            "labels_equal": bool(a.tobytes() == b.tobytes())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[24, 26])
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--dir", default=None, help="a local directory for the files (default: a temporary one)")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    out = {"card": card(), "scales": {}}
    print(f"card: {out['card']}")
    with tempfile.TemporaryDirectory(dir=a.dir) as d:
        for scale in a.scales:
            path = os.path.join(d, f"rmat{scale}.graph500")
            write_rmat_graph500(path, scale)
            r = measure(path, a.runs, a.warmup)
            os.unlink(path)
            out["scales"][scale] = r
            print(f"RMAT-{scale}: {r['file_bytes'] / 1e9:.2f} GB, n {r['node_count']}, m {r['edges']}, "
                  f"{r['chunks']} chunks\n"
                  f"  one-pass  {r['one_pass']['best_ms']:9.1f} / {r['one_pass']['median_ms']:9.1f} ms  "
                  f"{r['one_pass_file_GBps']:6.2f} GB/s  h2d {r['h2d_bytes'] / 1e9:.2f} GB  "
                  f"peak device {r['device_bytes'] / 1e9:.3f} GB  device {r['device_ms']:.1f} ms\n"
                  f"  load+wcc  {r['load_wcc']['best_ms']:9.1f} / {r['load_wcc']['median_ms']:9.1f} ms  "
                  f"{r['load_wcc_file_GBps']:6.2f} GB/s\n"
                  f"  labels equal: {r['labels_equal']}", flush=True)
    if a.json:
        Path(a.json).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
