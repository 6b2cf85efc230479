"""Save and load time of binary graph files (Graph.serialize / DiGraph.load with FileFormat.Binary, csrc/load.cu)
next to the Graph500 load of the same graph and the pread floor of each file (bench_load.py's protocol: 4
threads read the file into pinned memory in 64 MiB pieces, nothing else).

    python tools/bench_binary.py [--scales 20,24] [--runs 3] [--json out.json]

Per scale: an RMAT Graph500 file (device generator + write_graph500) is loaded as a Sorted DiGraph, which is
serialized to a binary file (8m + 8n + 54 bytes).  Files live in a temporary directory removed on exit and are
read once before timing, so the page cache is warm: the numbers are not disk numbers.  One warm-up of each
path, then --runs timed runs alternating the paths; the reloaded CSRs are compared byte for byte and the best
run is reported.  Saves include the write into the page cache, not a flush to disk."""
from __future__ import annotations

import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))
import graph_b200 as gb  # noqa: E402
from bench_load import pread_floor, same_csr  # noqa: E402


def warm(path):
    with open(path, "rb") as f:
        while f.read(1 << 26):
            pass


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="20,24")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card, "page_cache": "warm (every file is read once before timing)"}), flush=True)
    pinned = torch.empty(4 * (64 << 20), dtype=torch.uint8, pin_memory=True)
    out = {"card": card, "page_cache": "warm", "results": []}
    tmp = Path(tempfile.mkdtemp(prefix="bench_binary_"))
    try:
        for s in [int(x) for x in args.scales.split(",") if x]:
            m = 16 << s
            src = np.empty(m, np.uint32)
            dst = np.empty(m, np.uint32)
            gb.check(gb.lib.gb_rmat_edges(0, s, 42, 0, m, gb._ptr(src), gb._ptr(dst)))
            g500, binf = tmp / f"rmat{s}.graph500", tmp / f"rmat{s}.bin"
            gb.write_graph500(g500, src, dst)
            del src, dst
            load500 = lambda: gb.DiGraph.load(g500, layout=gb.Layout.Sorted)  # noqa: E731
            loadbin = lambda: gb.DiGraph.load(binf, file_format=gb.FileFormat.Binary)  # noqa: E731
            g = load500()
            g.serialize(binf)  # warm-up of the save
            warm(g500)
            warm(binf)
            h = loadbin()
            res = {"workload": f"RMAT-{s} directed, Sorted", "graph500_bytes": os.path.getsize(g500),
                   "binary_bytes": os.path.getsize(binf), "csr_byte_equal": same_csr(g, h, False),
                   "binary_chunks": h.load_info()["chunks"]}
            del h
            floor500, floorbin, save, l500, lbin = [], [], [], [], []
            for _ in range(args.runs):
                floor500.append(pread_floor(g500, pinned))
                floorbin.append(pread_floor(binf, pinned))
                save.append(timed(lambda: g.serialize(binf))[0])
                for fn, acc in ((load500, l500), (loadbin, lbin)):
                    t, x = timed(fn)
                    acc.append(t)
                    del x
            res.update({"pread_floor_graph500_s": min(floor500), "pread_floor_binary_s": min(floorbin),
                        "save_s": min(save), "load_graph500_s": min(l500), "load_binary_s": min(lbin),
                        "save_runs_s": save, "load_binary_runs_s": lbin, "load_graph500_runs_s": l500})
            res["binary_over_floor"] = res["load_binary_s"] / res["pread_floor_binary_s"]
            print(json.dumps(res), flush=True)
            out["results"].append(res)
            del g
            os.unlink(g500)
            os.unlink(binf)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.json:
        Path(args.json).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
