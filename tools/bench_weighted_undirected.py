"""Weighted undirected graphs (UndirectedCsrGraph<u32, (), f32>): what keeping the f32 values costs against the
unweighted twin of the same edges.

    python tools/bench_weighted_undirected.py [--scales 22,24] [--runs 5] [--load-scale 18] [--json out.json]

Workloads (each run once as a warm-up, then --runs times; medians of host wall time around calls that return
only once the device work is done):
  - build: gb_graph_from_weighted_edges_u32 against gb_graph_from_edges_u32 on the undirected RMAT edges of each
    scale (edge factor 16, host arrays, so the upload is included), Unsorted and Sorted;
  - to_undirected: gb_to_undirected_weighted against gb_to_undirected on DiGraph.rmat(scale, weights=True);
  - load: Graph.load_weighted against Graph.load of one weighted text edge list of at least 64 MiB (RMAT
    --load-scale edges), which takes the streamed device path.
Peak device bytes: each build runs in a fresh process; the peak of the default memory pool (cudaMemPoolAttrUsedMemHigh)
is read beside the figure computed from the build's allocations (peak_model_bytes), gb_graph_info.device_bytes of
the result and the drop in cudaMemGetInfo's free bytes (the pool keeps freed blocks, so that drop covers the peak).
The card's name and power limit are read in the same run."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import graph_b200 as gb  # noqa: E402
from graph_b200 import _capi  # noqa: E402

LAYOUTS = {"Unsorted": gb.Layout.Unsorted, "Sorted": gb.Layout.Sorted}
POOL_USED_HIGH = 8  # cudaMemPoolAttrUsedMemHigh


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.splitlines()[0]
    name, power, clock = (x.strip() for x in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def rmat_host(scale: int, seed: int = 42):
    m = 16 << scale
    src = np.empty(m, np.uint32)
    dst = np.empty(m, np.uint32)
    _capi.check(_capi.lib.gb_rmat_edges(0, scale, seed, 0, m, src.ctypes.data_as(C.c_void_p),
                                        dst.ctypes.data_as(C.c_void_p)))
    w = np.random.default_rng(seed).random(m, dtype=np.float32)
    return src, dst, w


def timed(fn, runs: int) -> tuple[float, object]:
    fn()  # warm-up
    times, last = [], None
    for _ in range(runs):
        last = None  # the previous graph is freed before the next build
        t0 = time.perf_counter()
        last = fn()
        times.append(time.perf_counter() - t0)
    return statistics.median(times) * 1e3, last


def peak_model_bytes(n: int, m: int, layout: str, weighted: bool) -> int:
    """The buffers a host-edge undirected build holds at its peak (graph.cu: graph_from_host_edges, build_graph_csrs,
    build_csr_device), cub's temporary storage left out: the uploaded edges (8m, + 4m values), both passes' rows and
    columns (16m), the sort's keys (Unsorted: rows copy, alternate keys, index and alternate index, 4 x 8m; Sorted:
    2 x 16m of 64-bit keys, + 2 x 8m of index payload with values), and the result (4(n + 1) offsets, 8m + 32 targets,
    + 8m + 32 values)."""
    edges = 8 * m + (4 * m if weighted else 0)
    passes = 16 * m
    if layout == "Unsorted":
        sort = 32 * m
    else:
        sort = 32 * m + (16 * m if weighted else 0)
    result = 4 * (n + 1) + 8 * m + 32 + ((8 * m + 32) if weighted else 0)
    return edges + passes + sort + result


def peak_child(scale: int, layout: str, weighted: bool) -> dict:
    """Runs in a fresh process: one build, with the pool's peak and cudaMemGetInfo around it."""
    cudart = C.CDLL("libcudart.so.12")
    src, dst, w = rmat_host(scale)
    pool = C.c_void_p()
    assert cudart.cudaDeviceGetDefaultMemPool(C.byref(pool), 0) == 0
    free0, total = C.c_size_t(), C.c_size_t()
    assert cudart.cudaMemGetInfo(C.byref(free0), C.byref(total)) == 0
    zero = C.c_uint64(0)
    assert cudart.cudaMemPoolSetAttribute(pool, POOL_USED_HIGH, C.byref(zero)) == 0
    edges = np.stack([src, dst], 1)
    g = gb.Graph.from_numpy(edges, LAYOUTS[layout], node_count=1 << scale, weights=w if weighted else None)
    high, free1 = C.c_uint64(), C.c_size_t()
    assert cudart.cudaMemPoolGetAttribute(pool, POOL_USED_HIGH, C.byref(high)) == 0
    assert cudart.cudaMemGetInfo(C.byref(free1), C.byref(total)) == 0
    m = len(src)
    return {"scale": scale, "layout": layout, "weighted": weighted, "pool_peak_bytes": int(high.value),
            "mem_get_info_drop_bytes": int(free0.value - free1.value), "device_bytes": g.device_bytes(),
            "peak_model_bytes": peak_model_bytes(1 << scale, m, layout, weighted), "edges": m}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--scales", default="22,24")
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--load-scale", type=int, default=18)
    ap.add_argument("--peak-scale", type=int, default=22)
    ap.add_argument("--json", default=None)
    ap.add_argument("--peak-child", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.peak_child:
        scale, layout, weighted = a.peak_child.split(":")
        print(json.dumps(peak_child(int(scale), layout, weighted == "1")))
        return
    if gb.device_count() == 0:
        raise SystemExit("no CUDA device: these timings need an H100")
    out = {"card": card(), "runs": a.runs, "build": [], "to_undirected": [], "load": [], "peak": []}
    print(json.dumps(out["card"]), flush=True)

    for scale in (int(s) for s in a.scales.split(",")):
        src, dst, w = rmat_host(scale)
        edges = np.stack([src, dst], 1)
        n = 1 << scale
        for name, lay in LAYOUTS.items():
            t_plain, _ = timed(lambda: gb.Graph.from_numpy(edges, lay, node_count=n), a.runs)
            t_w, g = timed(lambda: gb.Graph.from_numpy(edges, lay, node_count=n, weights=w), a.runs)
            row = {"scale": scale, "layout": name, "edges": len(src), "unweighted_ms": t_plain, "weighted_ms": t_w,
                   "ratio": t_w / t_plain, "weighted_device_bytes": g.device_bytes()}
            out["build"].append(row)
            print("build", json.dumps(row), flush=True)
        del edges, src, dst, w
        d = gb.DiGraph.rmat(scale, weights=True, layout=gb.Layout.Sorted)
        for name, lay in LAYOUTS.items():
            t_plain, _ = timed(lambda: d.to_undirected(lay), a.runs)
            t_w, _ = timed(lambda: d.to_undirected(lay, weights=True), a.runs)
            row = {"scale": scale, "layout": name, "unweighted_ms": t_plain, "weighted_ms": t_w,
                   "ratio": t_w / t_plain}
            out["to_undirected"].append(row)
            print("to_undirected", json.dumps(row), flush=True)
        del d

    with tempfile.TemporaryDirectory() as tmp:
        p = Path(tmp) / f"rmat{a.load_scale}.wel"
        src, dst, w = rmat_host(a.load_scale)
        np.savetxt(p, np.column_stack([src, dst, w]), fmt=["%d", "%d", "%.6f"], delimiter=" ")
        size = p.stat().st_size
        assert size >= 64 << 20, f"{size} bytes: use a larger --load-scale for the streamed path"
        for name, lay in LAYOUTS.items():
            t_plain, _ = timed(lambda: gb.Graph.load(p, lay, gb.FileFormat.EdgeList), a.runs)
            t_w, g = timed(lambda: gb.Graph.load_weighted(p, lay), a.runs)
            row = {"file_bytes": size, "layout": name, "chunks": g.load_info()["chunks"], "unweighted_ms": t_plain,
                   "weighted_ms": t_w, "ratio": t_w / t_plain}
            out["load"].append(row)
            print("load", json.dumps(row), flush=True)

    for name in LAYOUTS:
        for weighted in (False, True):
            r = subprocess.run([sys.executable, __file__, "--peak-child", f"{a.peak_scale}:{name}:{int(weighted)}"],
                               capture_output=True, text=True, check=True)
            row = json.loads(r.stdout.splitlines()[-1])
            out["peak"].append(row)
            print("peak", json.dumps(row), flush=True)

    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
