#!/usr/bin/env python3
"""One-shot WCC of a host out-CSR (graph_b200.wcc_csr / gb_wcc_csr_u32) against the resident twin and the bus.

For each R-MAT scale (Sorted, seed 42) the CSRs are copied to pinned host arrays, then three paths are run in
one process, alternated, after warm-up runs:
  floor     a plain H2D copy of the out offsets and out targets (4(n+1) + 4m bytes), the least any one-shot
            path must move;
  one-shot  wcc_csr(out_offsets, out_targets): offsets first, targets streamed in chunks and linked as they land;
  twin      DiGraph.from_csr(out..., in...) + wcc(): both CSRs uploaded (8(n+1) + 8m bytes), then Afforest.
Wall times (time.perf_counter around each call, device synchronised) are reported as best / median.  Also:
the time after the last byte lands (one-shot minus floor), the one-shot from pageable arrays, whether every
path's labels are bit-equal, a sweep of the chunk size (GB_WCC_FEED_EDGES) at one scale and on a path graph
linked in reverse id order (the deepest parent chains), and the device timeline of one one-shot call at that
scale (torch.profiler: summed kernel and copy times).

    python tools/bench_wcc_csr.py [--scales 22 24 26] [--runs 5] [--sweep-scale 24] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import bench  # noqa: E402  (pinned host arrays, host CSR copies)
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
    return time.perf_counter() - t0, out


def stats(ts):
    return {"best_ms": 1e3 * min(ts), "median_ms": 1e3 * statistics.median(ts), "runs": len(ts)}


def fmt(s):
    return f"{s['best_ms']:8.2f} / {s['median_ms']:8.2f} ms"


def with_env(name, value, fn):
    old = os.environ.get(name)
    os.environ[name] = str(value)
    try:
        return fn()
    finally:
        if old is None:
            del os.environ[name]
        else:
            os.environ[name] = old


def timed_runs(fn, runs, warmup):
    for _ in range(warmup):
        fn()
    return [wall(fn)[0] for _ in range(runs)]


def measure_scale(scale, runs, warmup):
    g = gb.DiGraph.rmat(scale, seed=42, layout=gb.Layout.Sorted)
    n, m = g.node_count(), g.edge_count()
    (oo, ot, io, it), keep = bench.host_csr_from_device(g)
    del g
    torch.cuda.empty_cache()
    d_off = torch.empty(n + 1, dtype=torch.int32, device="cuda")
    d_tgt = torch.empty(m, dtype=torch.int32, device="cuda")
    h_off, h_tgt = torch.from_numpy(oo.view(np.int32)), torch.from_numpy(ot.view(np.int32))

    def floor():
        d_off.copy_(h_off, non_blocking=True)
        d_tgt.copy_(h_tgt, non_blocking=True)

    parts = {"upload": [], "wcc": []}

    def twin():
        t0 = time.perf_counter()
        tg = gb.DiGraph.from_csr(oo, ot, io, it)
        t1 = time.perf_counter()
        comp = tg.wcc().components()
        t2 = time.perf_counter()
        parts["upload"].append(t1 - t0)
        parts["wcc"].append(t2 - t1)
        del tg
        return comp

    times = {"floor": [], "one_shot": [], "twin": []}
    for _ in range(warmup):
        floor(), gb.wcc_csr(oo, ot), twin()
    parts["upload"].clear(), parts["wcc"].clear()
    labels = {}
    for _ in range(runs):  # alternated
        times["floor"].append(wall(floor)[0])
        t, labels["one_shot"] = wall(lambda: gb.wcc_csr(oo, ot).components())
        times["one_shot"].append(t)
        t, labels["twin"] = wall(twin)
        times["twin"].append(t)
    del d_off, d_tgt
    torch.cuda.empty_cache()
    po, pt = np.array(oo), np.array(ot)  # pageable copies
    gb.wcc_csr(po, pt)
    pageable = []
    for _ in range(max(3, runs // 2)):
        t, labels["pageable"] = wall(lambda: gb.wcc_csr(po, pt).components())
        pageable.append(t)
    equal = all(v.tobytes() == labels["twin"].tobytes() for v in labels.values())
    res = {"scale": scale, "n": n, "m": m,
           "bytes": {"floor": 4 * (n + 1) + 4 * m, "one_shot": 4 * (n + 1) + 4 * m,
                     "twin": 8 * (n + 1) + 8 * m},
           "floor": stats(times["floor"]), "one_shot": stats(times["one_shot"]), "twin": stats(times["twin"]),
           "twin_upload": stats(parts["upload"]), "twin_wcc": stats(parts["wcc"]),
           "pageable_one_shot": stats(pageable), "labels_bit_equal": equal}
    res["after_last_byte_ms"] = res["one_shot"]["best_ms"] - res["floor"]["best_ms"]
    res["floor_gb_s"] = res["bytes"]["floor"] / (res["floor"]["best_ms"] * 1e-3) / 1e9
    print(f"RMAT-{scale}: n={n} m={m}  (best / median of {runs})")
    for k in ("floor", "one_shot", "twin"):
        print(f"  {k:9s} {fmt(res[k])}   {res['bytes'][k] / 1e9:6.3f} GB")
    print(f"  twin parts: from_csr {fmt(res['twin_upload'])}, wcc {fmt(res['twin_wcc'])}")
    print(f"  after the last byte: {res['after_last_byte_ms']:.2f} ms;  floor {res['floor_gb_s']:.1f} GB/s;  "
          f"pageable one-shot {fmt(res['pageable_one_shot'])};  labels bit-equal: {equal}")
    return res, (oo, ot, keep)


def sweep(oo, ot, runs, warmup, name, values, tag):
    out = {}
    for v in values:
        ts = with_env(name, v, lambda: timed_runs(lambda: gb.wcc_csr(oo, ot), runs, warmup))
        out[str(v)] = stats(ts)
        print(f"  {tag} {name}={v:<10} {fmt(out[str(v)])}")
    return out


def timeline(oo, ot):
    """Summed device time per kernel and per copy kind of one one-shot call (CUPTI via torch.profiler)."""
    from torch.profiler import ProfilerActivity, profile
    gb.wcc_csr(oo, ot)
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t, _ = wall(lambda: gb.wcc_csr(oo, ot))
    rows = {e.key: (e.self_device_time_total / 1e3, e.count) for e in prof.key_averages()
            if getattr(e, "self_device_time_total", 0) > 0}
    print(f"  timeline of one one-shot call ({1e3 * t:.2f} ms wall; device time summed per kernel / copy kind):")
    for k, (ms, cnt) in sorted(rows.items(), key=lambda kv: -kv[1][0]):
        print(f"    {ms:9.3f} ms  x{cnt:<4d} {k[:90]}")
    return {"wall_ms": 1e3 * t, "device_ms": {k: v[0] for k, v in rows.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[22, 24, 26])
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--sweep-scale", type=int, default=24, help="scale of the chunk-size sweep and the timeline (0: none)")
    ap.add_argument("--feeds", type=int, nargs="+", default=[1 << 20, 1 << 22, 1 << 24, 1 << 25])
    ap.add_argument("--path-log2", type=int, default=24, help="reversed path graph of 2^k nodes (0: none)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    report = {"card": card(), "torch": torch.__version__, "scales": [], "sweeps": {}}
    print("card (name, power limit, max SM clock):", report["card"])
    for scale in args.scales:
        res, (oo, ot, keep) = measure_scale(scale, args.runs, args.warmup)
        report["scales"].append(res)
        if scale == args.sweep_scale:
            report["sweeps"]["feed_edges"] = sweep(oo, ot, args.runs, args.warmup, "GB_WCC_FEED_EDGES", args.feeds,
                                                   f"RMAT-{scale}")
            report["timeline"] = timeline(oo, ot)
        del oo, ot, keep
    if args.path_log2:
        n = 1 << args.path_log2
        t_off, off = bench.pinned_empty(n + 1, np.uint32)
        t_tgt, tgt = bench.pinned_empty(n - 1, np.uint32)
        off[0] = 0
        off[1:] = np.arange(n, dtype=np.uint32)
        tgt[:] = np.arange(n - 1, dtype=np.uint32)  # row i links i - 1
        assert (gb.wcc_csr(off, tgt).components() == 0).all()
        report["sweeps"]["path_feed_edges"] = sweep(off, tgt, args.runs, args.warmup, "GB_WCC_FEED_EDGES",
                                                    args.feeds, f"path-2^{args.path_log2}")
    print("card (name, power limit, max SM clock):", report["card"])
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
