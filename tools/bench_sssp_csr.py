#!/usr/bin/env python3
"""One-shot SSSP of a host weighted out-CSR (graph_b200.sssp_csr / gb_sssp_csr_u32) against the twin path and the
bus.

Inputs (SURVEY.md §8d): R-MAT edges (oracle.rmat_edges) with f32 weights (oracle.rmat_weights), seed 42, built into
a Sorted out-CSR on the device and read back; delta = 0.1 x the mean weight; the start is the vertex of largest
out-degree.  The arrays are held twice on the host, page-locked and pageable.  Then, alternated after warm-up runs:
  floor     a plain H2D copy of the offsets, targets and weights (4(n+1) + 8m bytes) from page-locked memory,
            timed with CUDA events;
  pinned    sssp_csr on the page-locked arrays: the chunks go out at once and the bucket loop runs as they land;
  pageable  sssp_csr on the pageable arrays: synchronous copies, one chunk per relax pass;
  twin      DiGraph.from_csr(out-CSR, its transpose, weights) + delta_stepping: what a caller without the one-shot
            call runs.  The host transpose (oracle.csr_build, one thread) is timed once and reported on its own, as
            it does not change between runs; the twin's time per run is from_csr + delta_stepping.
Wall times (time.perf_counter around each call, device synchronised) are reported as best / median, with the device
times the calls report (CUDA events) and the one-shot call's info fields.  All distances must be bit-equal.  Prints
one JSON line per scale.

    python tools/bench_sssp_csr.py [--scales 22 24] [--runs 3] [--warmup 1] [--json out.json]
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
import oracle  # noqa: E402


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


def inputs(scale):
    s, d = oracle.rmat_edges(scale, seed=42)
    w = oracle.rmat_weights(42, 0, len(s))
    n = 1 << scale
    g = gb.DiGraph.from_numpy(np.stack([s, d], 1), layout=gb.Layout.Sorted, weights=w, node_count=n)
    off, tgt = g.csr("out")
    ow = g.out_weights()
    del g, s, d
    return n, np.array(off), np.array(tgt), ow, float(np.float32(0.1) * np.float32(w.mean()))


def one_scale(scale, runs, warmup):
    n, off, tgt, w, delta = inputs(scale)
    m = len(tgt)
    start = int(np.argmax(np.diff(off.astype(np.int64))))
    pinned = []
    keep = []
    for a in (off, tgt, w):
        t, p = bench.pinned_empty(len(a), a.dtype.type)
        p[:] = a
        keep.append(t)
        pinned.append(p)
    t0 = time.perf_counter()
    src = np.repeat(np.arange(n, dtype=np.uint32), np.diff(off.astype(np.int64)))
    io, it = oracle.csr_build(src, tgt, n, oracle.INCOMING, oracle.SORTED)
    transpose_ms = 1e3 * (time.perf_counter() - t0)
    del src
    d_buf = [torch.empty(len(a), dtype=torch.int32, device="cuda") for a in pinned]
    h_buf = [torch.from_numpy(a.view(np.int32)) for a in pinned]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    dev = {"floor": [], "pinned_upload": [], "pinned_total": [], "pageable_upload": [], "pageable_total": [],
           "twin_sssp": []}
    infos, dists = {}, {}

    def floor():
        ev[0].record()
        for d_, h_ in zip(d_buf, h_buf):
            d_.copy_(h_, non_blocking=True)
        ev[1].record()
        ev[1].synchronize()
        dev["floor"].append(ev[0].elapsed_time(ev[1]))

    def one_shot(kind, arrays):
        r = gb.sssp_csr(*arrays, start_node=start, delta=delta)
        dev[f"{kind}_upload"].append(r.info["upload_ms"])
        dev[f"{kind}_total"].append(r.info["total_ms"])
        infos[kind], dists[kind] = r.info, r.distances()

    def twin():
        g = gb.DiGraph.from_csr(off, tgt, io, it, out_weights=w)
        r = g.delta_stepping(start_node=start, delta=delta)
        dev["twin_sssp"].append(g.last_timing()["total_ms"])
        dists["twin"] = r.distances()
        del g

    paths = {"floor": floor, "pinned": lambda: one_shot("pinned", pinned),
             "pageable": lambda: one_shot("pageable", (off, tgt, w)), "twin": twin}
    for _ in range(warmup):
        for fn in paths.values():
            fn()
    for v in dev.values():
        v.clear()
    times = {k: [] for k in paths}
    for _ in range(runs):  # alternated
        for k, fn in paths.items():
            times[k].append(wall(fn)[0])
    equal = all(dists[k].tobytes() == dists["twin"].tobytes() for k in ("pinned", "pageable"))
    return {"card": card(), "scale": scale, "n": n, "m": m, "delta": delta, "start": start,
            "bytes": 4 * (n + 1) + 8 * m, "twin_bytes": 8 * (n + 1) + 12 * m,
            "reached": int((dists["twin"] < np.finfo(np.float32).max).sum()),
            "wall": {k: stats(v) for k, v in times.items()}, "device": {k: stats(v) for k, v in dev.items()},
            "host_transpose_ms": transpose_ms, "info": infos, "distances_equal": equal}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[22, 24])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_sssp_csr needs a CUDA device")
    out = []
    for scale in args.scales:
        res = one_scale(scale, args.runs, args.warmup)
        print(json.dumps(res), flush=True)
        out.append(res)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(out, indent=1))
    if not all(r["distances_equal"] for r in out):
        sys.exit("the one-shot and twin distances differ")


if __name__ == "__main__":
    main()
