#!/usr/bin/env python3
"""One-shot WCC of a host out-CSR on one device and over the devices of a communicator.

For each R-MAT scale (Sorted, seed 42) the out-CSR is copied to pinned host arrays, then these calls are run
in one process, alternated, after warm-up runs:
  wcc_csr          graph_b200.wcc_csr on device 0 (gb_wcc_csr_u32);
  comm[0]          Comm([0]).wcc_csr: the multi-part path with one part, which should cost what wcc_csr costs;
  comm[0] xV       Comm([0]).wcc_csr with GB_WCC_MULTI_PARTS=V: V virtual parts on one device (the split,
                   row slices and merge rounds, without more buses);
  comm[0..P-1]     Comm(devices 0..P-1).wcc_csr for P = 2, 4, 8 where the box has them.
Each call runs with a pinned `out` and with out=None (labels into fresh pageable memory).  Wall times
(time.perf_counter around each call, every device synchronised) are reported as best / median.  Also: the
per-device H2D floor, a plain copy of 1/P of the bytes the call moves (4(n+1) + 4m) from pinned memory to
device 0, and whether every call's labels are bit-equal.  The card's name, power limit and max SM clock are
read in the same run.

    python tools/bench_wcc_csr_multi.py [--scales 22 24 26] [--runs 5] [--warmup 2] [--virtual 2 4] [--json f]
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


def fmt(s):
    return f"{s['best_ms']:8.2f} / {s['median_ms']:8.2f} ms"


def with_parts(v, fn):
    old = os.environ.get("GB_WCC_MULTI_PARTS")
    os.environ["GB_WCC_MULTI_PARTS"] = str(v)
    try:
        return fn()
    finally:
        if old is None:
            del os.environ["GB_WCC_MULTI_PARTS"]
        else:
            os.environ["GB_WCC_MULTI_PARTS"] = old


def measure_scale(scale, runs, warmup, virtual, comms):
    g = gb.DiGraph.rmat(scale, seed=42, layout=gb.Layout.Sorted)
    n, m = g.node_count(), g.edge_count()
    (oo, ot, _, _), keep = bench.host_csr_from_device(g)
    del g
    torch.cuda.empty_cache()
    t_out, out = bench.pinned_empty(n, np.uint32)
    nbytes = 4 * (n + 1) + 4 * m

    calls = {"wcc_csr": lambda o: gb.wcc_csr(oo, ot, out=o).components()}
    calls["comm[0]"] = lambda o: comms[1].wcc_csr(oo, ot, out=o).components()
    for v in virtual:
        calls[f"comm[0] x{v}"] = lambda o, v=v: with_parts(v, lambda: comms[1].wcc_csr(oo, ot, out=o).components())
    for p, c in comms.items():
        if p > 1:
            calls[f"comm[0..{p - 1}]"] = lambda o, c=c: c.wcc_csr(oo, ot, out=o).components()
    # the per-device floor: 1/P of the bytes, pinned -> device 0
    h = torch.from_numpy(ot.view(np.int32))
    d = torch.empty(m, dtype=torch.int32, device="cuda:0")
    floors = {}
    for p in (1, 2, 4, 8):
        k = min(m, (n + 1 + m) // p)  # 1/P of the offsets' and targets' u32 entries
        floors[p] = lambda k=k: d[:k].copy_(h[:k], non_blocking=True)

    times = {(name, kind): [] for name in calls for kind in ("pinned", "pageable")}
    ftimes = {p: [] for p in floors}
    labels = {}
    for i in range(warmup + runs):  # alternated
        for p, f in floors.items():
            t, _ = wall(f)
            if i >= warmup:
                ftimes[p].append(t)
        for name, fn in calls.items():
            for kind in ("pinned", "pageable"):
                t, lab = wall(lambda: fn(out if kind == "pinned" else None))
                if i >= warmup:
                    times[(name, kind)].append(t)
                    labels[(name, kind)] = lab.tobytes()
    del d
    torch.cuda.empty_cache()
    equal = len(set(labels.values())) == 1
    res = {"scale": scale, "n": n, "m": m, "bytes": nbytes, "labels_bit_equal": equal,
           "floor": {str(p): stats(ts) for p, ts in ftimes.items()},
           "calls": {f"{name} / {kind} out": stats(ts) for (name, kind), ts in times.items()}}
    print(f"RMAT-{scale}: n={n} m={m}  {nbytes / 1e9:.3f} GB  (best / median of {runs})")
    for p, s in res["floor"].items():
        print(f"  H2D floor, 1/{p} of the bytes  {fmt(s)}")
    for k, s in res["calls"].items():
        print(f"  {k:32s} {fmt(s)}")
    print(f"  labels bit-equal: {equal}")
    del t_out, keep
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="+", default=[22, 24, 26])
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--virtual", type=int, nargs="*", default=[2, 4], help="GB_WCC_MULTI_PARTS on Comm([0])")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    ndev = torch.cuda.device_count()
    comms = {p: gb.Comm(list(range(p))) for p in (1, 2, 4, 8) if p <= ndev}
    report = {"cards": cards(), "devices": ndev, "torch": torch.__version__, "scales": []}
    print("cards (name, power limit, max SM clock):", report["cards"])
    for scale in args.scales:
        report["scales"].append(measure_scale(scale, args.runs, args.warmup, args.virtual, comms))
    if ndev < 2:
        print("one device: the multi-device rows are not measured")
    print("cards (name, power limit, max SM clock):", report["cards"])
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
