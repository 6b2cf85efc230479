#!/usr/bin/env python3
"""One-shot PageRank of a host CSR on one device and over the devices of a communicator.

For each R-MAT scale (Sorted, seed 42) the in-CSR and the out offsets are copied to pinned host arrays, then
these calls (20 JACOBI sweeps, tolerance 0) are run in one process, alternated, after warm-up runs:
  page_rank_csr_u32   gb_page_rank_csr_u32 on device 0: one device, the targets classified as they land;
  comm[0] csr         Comm([0]).page_rank_csr (gb_page_rank_csr_multi_u32 with one part);
  comm[0] twin        DiGraph.for_page_rank + Comm([0]).page_rank: the twin path it replaces;
  comm[0..P-1] csr / twin   the same over devices 0..P-1 for P = 2, 4, 8 where the box has them (the twin path
                      uploads a full twin to every device).
Wall times (time.perf_counter around each call, every device synchronised) are reported as best / median.  Also
per device: the H2D bytes each path moves, computed from the split (pr_split, graph_b200/csrc/csr_split.h), and the peak
device bytes of one call: the high-water mark of the device's default memory pool (cudaMemPoolAttrUsedMemHigh,
which holds every buffer of the one-device paths) plus, with several parts, the cudaMalloc'd part and offset
buffers computed from the split.  The communicator's score vectors, the same for both comm paths, are not
counted.  Finally whether the ranks of all comm calls are bit-equal.  The card's name, power limit and max SM
clock are read in the same run.

    python tools/bench_pr_csr_multi.py [--scales 22 24 26] [--runs 5] [--warmup 2] [--json f]
"""
import argparse
import ctypes as C
import json
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
from graph_b200._capi import PR_JACOBI, PageRankConfig, check, lib  # noqa: E402

MAXIT = 20


def cards():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines() if q.returncode == 0 and q.stdout.strip() else ["unknown"]


def sync_all():
    for d in range(torch.cuda.device_count()):
        torch.cuda.synchronize(d)


def wall(fn):
    sync_all()
    t0 = time.perf_counter()
    out = fn()
    sync_all()
    return time.perf_counter() - t0, out


def stats(ts):
    return {"best_ms": 1e3 * min(ts), "median_ms": 1e3 * statistics.median(ts), "runs": len(ts)}


class Pools:
    """High-water marks of the devices' default memory pools (libcudart is shared with the library)."""

    def __init__(self, ndev):
        self.rt = C.CDLL("libcudart.so.12")
        self.pools = []
        for d in range(ndev):
            p = C.c_void_p()
            assert self.rt.cudaDeviceGetDefaultMemPool(C.byref(p), d) == 0
            self.pools.append(p)

    def reset(self):
        for p in self.pools:
            zero = C.c_uint64(0)
            self.rt.cudaMemPoolSetAttribute(p, 8, C.byref(zero))  # cudaMemPoolAttrUsedMemHigh

    def high(self):
        out = []
        for p in self.pools:
            v = C.c_uint64(0)
            self.rt.cudaMemPoolGetAttribute(p, 8, C.byref(v))
            out.append(int(v.value))
        return out


def split_rows(off, parts):
    """R_0 .. R_U of pr_split (csr_split.h; monotone offsets)"""
    m, n = int(off[-1]), len(off) - 1
    cuts = [0] + [int(np.searchsorted(off, m * u // parts, side="left")) for u in range(1, parts)] + [n]
    for i in range(1, len(cuts)):
        cuts[i] = min(max(cuts[i], cuts[i - 1]), n)
    return cuts


def part_bytes(io, p):
    """per device of a p-device comm: (H2D bytes of its part, cudaMalloc'd bytes of its part + full offsets)"""
    n = len(io) - 1
    R = split_rows(io, p)
    h2d = [8 * (R[u + 1] - R[u] + 1) + 4 * (int(io[R[u + 1]]) - int(io[R[u]])) for u in range(p)]
    malloc = [b + 8 * (n + 1) for b in h2d] if p > 1 else [0]
    return h2d, malloc


def measure_scale(scale, runs, warmup, comms, pools):
    g = gb.DiGraph.rmat(scale, seed=42, layout=gb.Layout.Sorted)
    n, m = g.node_count(), g.edge_count()
    (oo, _, io, it), keep = bench.host_csr_from_device(g, out_targets=False)
    del g
    torch.cuda.empty_cache()
    cfg = PageRankConfig(MAXIT, 0.0, 0.85, PR_JACOBI)

    def single():
        scores = np.empty(n, np.float32)
        itc, err = C.c_uint64(0), C.c_double(0.0)
        check(lib.gb_page_rank_csr_u32(0, n, io.ctypes.data_as(C.c_void_p), it.ctypes.data_as(C.c_void_p),
                                       oo.ctypes.data_as(C.c_void_p), C.byref(cfg), scores.ctypes.data_as(C.c_void_p),
                                       C.byref(itc), C.byref(err)))
        return scores

    def twin_path(comm):
        graphs = []
        for d in comm.devices:
            gb.set_device(d)
            graphs.append(gb.DiGraph.for_page_rank(io, it, oo))
        gb.set_device(0)
        return comm.page_rank(graphs, max_iterations=MAXIT, tolerance=0.0).scores()

    calls = {"page_rank_csr_u32": single}
    for p, c in comms.items():
        name = "comm[0]" if p == 1 else f"comm[0..{p - 1}]"
        calls[f"{name} csr"] = lambda c=c: c.page_rank_csr(io, it, oo, max_iterations=MAXIT, tolerance=0.0).scores()
        calls[f"{name} twin"] = lambda c=c: twin_path(c)
    times = {name: [] for name in calls}
    ranks = {}
    for i in range(warmup + runs):  # alternated
        for name, fn in calls.items():
            t, s = wall(fn)
            if i >= warmup:
                times[name].append(t)
                ranks[name] = s.tobytes()
    peaks = {}
    for name, fn in calls.items():  # one more call each, for the pools' high-water marks
        sync_all()
        pools.reset()
        fn()
        sync_all()
        peaks[name] = pools.high()
    comm_ranks = {v for k, v in ranks.items() if k.startswith("comm")}
    res = {"scale": scale, "n": n, "m": m, "comm_ranks_bit_equal": len(comm_ranks) == 1,
           "calls": {k: stats(ts) for k, ts in times.items()}, "devices": {}}
    print(f"RMAT-{scale}: n={n} m={m}  (best / median of {runs})")
    for k, s in res["calls"].items():
        print(f"  {k:22s} {s['best_ms']:9.2f} / {s['median_ms']:9.2f} ms")
    for p in comms:
        name = "comm[0]" if p == 1 else f"comm[0..{p - 1}]"
        h2d, malloc = part_bytes(io, p)
        twin_bytes = 4 * m + 8 * (n + 1)
        dev = {"h2d_bytes_csr": h2d, "h2d_bytes_twin": [twin_bytes] * p,
               "peak_bytes_csr": [peaks[f"{name} csr"][d] + malloc[d] if p > 1 else peaks[f"{name} csr"][d]
                                  for d in range(p)],
               "peak_bytes_twin": peaks[f"{name} twin"][:p]}
        res["devices"][name] = dev
        print(f"  {name}: H2D GB per device csr {[round(b / 1e9, 3) for b in h2d]}, twin {twin_bytes / 1e9:.3f}; "
              f"peak GB per device csr {[round(b / 1e9, 3) for b in dev['peak_bytes_csr']]}, "
              f"twin {[round(b / 1e9, 3) for b in dev['peak_bytes_twin']]}")
    print(f"  page_rank_csr_u32 peak GB on device 0: {peaks['page_rank_csr_u32'][0] / 1e9:.3f}")
    res["peak_bytes_single"] = peaks["page_rank_csr_u32"][0]
    print(f"  ranks of all comm calls bit-equal: {res['comm_ranks_bit_equal']}")
    del keep
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[22, 24, 26])
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    ndev = torch.cuda.device_count()
    comms = {p: gb.Comm(list(range(p))) for p in (1, 2, 4, 8) if p <= ndev}
    pools = Pools(ndev)
    report = {"cards": cards(), "devices": ndev, "torch": torch.__version__, "scales": []}
    print("cards (name, power limit, max SM clock):", report["cards"])
    for scale in args.scales:
        report["scales"].append(measure_scale(scale, args.runs, args.warmup, comms, pools))
    if ndev < 2:
        print("one device: the multi-device rows are not measured")
    print("cards (name, power limit, max SM clock):", report["cards"])
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
