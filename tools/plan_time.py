"""plan_time.py — wall time of the JACOBI layout build (gb_page_rank_plan_reset + rebuild), several reps,
and the high-water mark of the device memory pool during each build (resident graph included)."""
import argparse, ctypes as C, json, sys, time
from pathlib import Path
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
ap = argparse.ArgumentParser(); ap.add_argument("--scale", type=int, default=26); ap.add_argument("--reps", type=int, default=3)
a = ap.parse_args()
import torch, graph_b200 as gb
from graph_b200._capi import lib, check
from bench_load import Pool
g = gb.DiGraph.rmat(a.scale, 16, 42, gb.Layout.Sorted)
pool = Pool()
ts, peaks = [], []
for _ in range(a.reps):
    check(lib.gb_page_rank_plan_reset(g._g)); torch.cuda.synchronize()
    pool.reset()
    t0 = time.perf_counter(); info = g.page_rank_plan_info(); torch.cuda.synchronize(); ts.append((time.perf_counter() - t0) * 1e3)
    peaks.append(pool.high())
print(json.dumps({"scale": a.scale, "plan_build_ms": [round(t, 2) for t in ts], "peak_device_bytes": peaks,
                  "device_bytes": info["device_bytes"]}))
