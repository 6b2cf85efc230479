"""Adjacency-list graphs on one GPU: the build against the CSR build, add_edges batches against a full CSR rebuild,
the snapshot's rate, and the build's peak pool bytes against its model (DESIGN.md §10).

    python tools/bench_al.py [--runs 5]

Every figure is the median of `runs` after one warm-up.  Edges are R-MAT (seed 42; batches from seeds 43, 44, ...).
- build: DirectedALGraph.from_torch against DiGraph.from_torch on the same device edges at directed RMAT-22, wall
  time of the call (it ends in a device synchronise).
- batches: add_edges from device tensors of 1, 10^3, 10^5 and 10^7 uniformly random edges, Unsorted and Sorted, at
  RMAT-18 and RMAT-22.  The graph gets one batch of each size before the timed ones, so that the rows a batch
  touches are no longer at cap = len; the time is gb_algraph_batch_info's CUDA-event time without compactions, which
  are counted and timed apart.  The rebuild column is what a user without adjacency lists does: a DiGraph build of
  all m + b edges from device tensors.
- snapshot: to_graph() CUDA-event time and GB/s over its compulsory bytes: read len, start and the targets of both
  lists, write their offsets and targets.
- peak: one Unsorted directed build at RMAT-22 from device edges in a fresh process; the default pool's
  cudaMemPoolAttrUsedMemHigh against peak_model_bytes.
The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import graph_b200 as gb  # noqa: E402

POOL_USED_HIGH = 8  # cudaMemPoolAttrUsedMemHigh


def card() -> dict:
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [x.strip() for x in r.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def rmat_device(scale: int, seed: int, count: int | None = None):
    import torch
    m = count if count is not None else 16 << scale
    s = np.empty(m, np.uint32)
    d = np.empty(m, np.uint32)
    gb._capi.check(gb.lib.gb_rmat_edges(0, scale, seed, 0, m, gb._ptr(s), gb._ptr(d)))
    return torch.from_numpy(s.view(np.int32)).cuda(), torch.from_numpy(d.view(np.int32)).cuda()


def uniform_device(n: int, b: int, seed: int):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randint(0, n, (b,), device="cuda", generator=g, dtype=torch.int32),
            torch.randint(0, n, (b,), device="cuda", generator=g, dtype=torch.int32))


def median(xs):
    return float(np.median(xs))


def timed(fn, runs: int):
    fn()  # warm-up
    out = []
    for _ in range(runs):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return median(out)


def peak_model_bytes(n: int, m: int) -> int:
    """A directed Unsorted build from device edges at its peak, the in-list's radix sort: the caller's edges are not
    counted (they are not the pool's); the out-list (pool of 1.25 m + 2^16 targets, start/len/cap per row), and
    build_csr_device's row copy, alternate keys, two index arrays, targets and offsets."""
    out_list = 4 * (m + m // 4 + (1 << 16)) + 16 * n
    build = 16 * m + 4 * m + 4 * (n + 1)
    return out_list + build


def peak_child(scale: int) -> dict:
    import torch
    s, d = rmat_device(scale, 42)
    torch.cuda.synchronize()
    cudart = C.CDLL("libcudart.so.12")
    pool = C.c_void_p()
    assert cudart.cudaDeviceGetDefaultMemPool(C.byref(pool), 0) == 0
    zero = C.c_uint64(0)
    assert cudart.cudaMemPoolSetAttribute(pool, POOL_USED_HIGH, C.byref(zero)) == 0
    g = gb.DirectedALGraph.from_torch(s, d, node_count=1 << scale, layout=gb.Layout.Unsorted)
    high = C.c_uint64(0)
    assert cudart.cudaMemPoolGetAttribute(pool, POOL_USED_HIGH, C.byref(high)) == 0
    m = 16 << scale
    return {"scale": scale, "pool_peak_bytes": int(high.value), "peak_model_bytes": peak_model_bytes(1 << scale, m),
            "device_bytes": g.device_bytes()}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--scales", default="18,22")
    ap.add_argument("--sizes", default="1,1000,100000,10000000")
    ap.add_argument("--peak-child", type=int, default=0, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.peak_child:
        print(json.dumps(peak_child(a.peak_child)))
        return
    import torch
    out = {"card": card(), "runs": a.runs}
    print("card", json.dumps(out["card"]), flush=True)

    s, d = rmat_device(22, 42)
    n = 1 << 22
    out["build_rmat22"] = {
        "al_ms": {name: timed(lambda: gb.DirectedALGraph.from_torch(s, d, node_count=n, layout=lay), a.runs)
                  for name, lay in (("Unsorted", gb.Layout.Unsorted), ("Sorted", gb.Layout.Sorted))},
        "csr_ms": {name: timed(lambda: gb.DiGraph.from_torch(s, d, node_count=n, layout=lay), a.runs)
                   for name, lay in (("Unsorted", gb.Layout.Unsorted), ("Sorted", gb.Layout.Sorted))}}
    print("build", json.dumps(out["build_rmat22"]), flush=True)
    del s, d

    out["batches"], out["snapshot"] = [], []
    seed = 43
    for scale in map(int, a.scales.split(",")):
        n = 1 << scale
        s, d = rmat_device(scale, 42)
        m = len(s)
        for name, lay in (("Unsorted", gb.Layout.Unsorted), ("Sorted", gb.Layout.Sorted)):
            g = gb.DirectedALGraph.from_torch(s, d, node_count=n, layout=lay)
            for b in map(int, a.sizes.split(",")):
                bs, bd = uniform_device(n, b, seed)
                seed += 1
                g.add_edges(bs, bd)  # warm-up: the rows it touches get slack
                times, comp_ms, comps = [], [], 0
                for _ in range(a.runs):
                    bs, bd = uniform_device(n, b, seed)
                    seed += 1
                    g.add_edges(bs, bd)
                    info = g.last_batch()
                    comps += info["compactions"]
                    if info["compactions"]:
                        comp_ms.append(info["compaction_ms"])
                    times.append(info["total_ms"] - info["compaction_ms"])
                allsrc, alldst = torch.cat([s, bs]), torch.cat([d, bd])
                rebuild = timed(lambda: gb.DiGraph.from_torch(allsrc, alldst, node_count=n, layout=lay), a.runs)
                row = {"scale": scale, "m": m, "layout": name, "batch": b, "add_edges_ms": median(times),
                       "compactions": comps, "compaction_ms": comp_ms, "rebuild_ms": rebuild,
                       "graph_edges": g.edge_count()}
                out["batches"].append(row)
                print("batch", json.dumps(row), flush=True)
            snaps = []
            for _ in range(a.runs + 1):
                snap = g.to_graph()
                snaps.append(snap.last_timing()["total_ms"])
            me = g.edge_count()
            # per list: len (4n) + start (8n) + targets (4 me) read, offsets (4 (n + 1)) + targets (4 me) written
            compulsory = 2 * (12 * n + 8 * me + 4 * (n + 1))
            ms = median(snaps[1:])
            row = {"scale": scale, "layout": name, "edges": me, "snapshot_ms": ms, "compulsory_bytes": compulsory,
                   "gb_per_s": compulsory / ms / 1e6}
            out["snapshot"].append(row)
            print("snapshot", json.dumps(row), flush=True)
            del g, snap
        del s, d
        torch.cuda.empty_cache()

    r = subprocess.run([sys.executable, __file__, "--peak-child", "22"], capture_output=True, text=True)
    out["peak"] = json.loads(r.stdout.strip().splitlines()[-1]) if r.returncode == 0 else {"error": r.stderr[-2000:]}
    print("peak", json.dumps(out["peak"]), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
