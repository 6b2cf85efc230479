"""Node-labelled graphs: LabelStats, NodeLabelIndex and NeighborLabelFrequencies on the device (csrc/labels.cu),
and DotGraph (.graph) loads, beside the numpy restatement of the reference the tests compare them with
(tests/dotgraph_restatement.py).  That restatement is vectorised numpy (its reader a Python loop), not the
reference's Rust, so its times are a CPU point of comparison, not the reference's numbers.

    python tools/bench_labels.py [--runs 5] [--nlf-scales 22,24] [--cpu-max-scale 22] [--load-only] [--json out.json]

Workloads:
  - label_stats and node_label_index on the graph of the reference's Criterion bench
    (crates/builder/benches/dotgraph.rs): edges([(0, n - 1)]) with labels uniform in 0..42, at n = 1e3, 1e4,
    1e5 (the reference's sizes), 2^24 and 2^26;
  - neighbor_label_frequencies on undirected Sorted RMAT graphs (edge factor 16) with labels uniform in 0..42;
  - .graph loads of an RMAT-18 file (below 64 MiB, so read by the host reader unless GB_LOAD_CHUNK_BYTES selects
    the device parser) and of an RMAT-20 file (parsed on the device);
  - the same two graphs saved with serialize_labeled and loaded back with load_labeled(file_format=Binary): the
    RMAT-18 file on the host path and the streamed path, the RMAT-20 file (above 64 MiB) on the streamed path, beside
    the pread floor of the file (tools/bench_load.py: 4 threads reading it into pinned memory, no device work).
Times: each structure reports the CUDA-event time of its device work (gb_graph_last_timing: first kernel to last,
the copies of the results to the host excluded) and the host time of the whole call; the achieved bandwidth of
neighbor_label_frequencies is computed over the device time from the compulsory bytes
4(n+1) offsets + 4E targets + 4E gathered labels + 4(n+1) pair offsets + 8 * pairs written, E = target_count.
Each workload runs once as a warm-up, then --runs times; the median is reported.  The device results are
compared with the restatement wherever it is run."""
from __future__ import annotations

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

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tests"))
import graph_b200 as gb  # noqa: E402
import oracle  # noqa: E402
import dotgraph_restatement as dot  # noqa: E402
from bench_load import pread_floor  # noqa: E402


def timed(fn, runs):
    """(last result, median host ms) of `runs` calls after one warm-up"""
    fn()
    out, times = None, []
    for _ in range(runs):
        t0 = time.perf_counter()
        out = fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return out, statistics.median(times)


def device_timed(g, fn, runs):
    """(last result, median CUDA-event ms of the call's device work, median host ms of the whole call)"""
    fn()
    out, dev, host = None, [], []
    for _ in range(runs):
        t0 = time.perf_counter()
        out = fn()
        host.append((time.perf_counter() - t0) * 1e3)
        dev.append(g.last_timing()["total_ms"])
    return out, statistics.median(dev), statistics.median(host)


def emit(rows, row):
    rows.append(row)
    print(json.dumps(row), flush=True)


def bench_stats(rows, runs, sizes, cpu_max):
    rng = np.random.default_rng(42)
    for n in sizes:
        labels = rng.integers(0, 42, n).astype(np.uint32)
        g = gb.Graph.from_numpy(np.array([[0, n - 1]], np.uint32), node_values=labels)
        st, st_dev, st_call = device_timed(g, g.label_stats, runs)
        idx, idx_dev, idx_call = device_timed(g, g.node_label_index, runs)
        row = {"bench": "label_stats+node_label_index", "n": n, "label_stats_device_ms": st_dev,
               "label_stats_call_ms": st_call, "node_label_index_device_ms": idx_dev,
               "node_label_index_call_ms": idx_call}
        if n <= cpu_max:
            off, tgt = g.csr()
            want, row["numpy_label_stats_ms"] = timed(lambda: dot.label_stats(off, tgt, labels), runs)
            (w_off, w_nodes), row["numpy_node_label_index_ms"] = timed(lambda: dot.node_label_index(labels), runs)
            row["match"] = (st.label_frequency == want["label_frequency"] and st.max_degree == want["max_degree"]
                            and idx.offsets.tolist() == w_off.tolist() and idx._nodes.tobytes() == w_nodes.tobytes())
        else:
            row["numpy_label_stats_ms"] = row["numpy_node_label_index_ms"] = "not measured"
        emit(rows, row)


def bench_nlf(rows, runs, scales, cpu_max_scale):
    for scale in scales:
        n = 1 << scale
        src, dst = oracle.rmat_edges(scale, seed=42)
        labels = np.random.default_rng(scale).integers(0, 42, n).astype(np.uint32)
        g = gb.Graph.from_numpy(np.stack([src, dst], axis=1), layout=gb.Layout.Sorted, node_values=labels)
        del src, dst
        E = int(g._info.target_count)
        g.neighbor_label_frequencies()
        call_ms, dev_ms, res = [], [], None
        for _ in range(runs):
            res = g.neighbor_label_frequencies()
            call_ms.append(res.micros / 1e3)
            dev_ms.append(res.device_ms)
        pairs = int(res.offsets[-1])
        compulsory = 8 * (n + 1) + 8 * E + 8 * pairs
        row = {"bench": "neighbor_label_frequencies", "scale": scale, "n": n, "target_count": E, "pairs": pairs,
               "device_ms": statistics.median(dev_ms), "call_ms": statistics.median(call_ms),
               "compulsory_bytes": compulsory, "gb_per_s": compulsory / statistics.median(dev_ms) / 1e6}
        if scale <= cpu_max_scale:
            off, tgt = g.csr()
            t0 = time.perf_counter()
            w_off, w_lab, w_cnt = dot.neighbor_label_frequencies(off, tgt, labels)
            row["numpy_ms"] = (time.perf_counter() - t0) * 1e3
            row["match"] = (res.offsets.tobytes() == w_off.tobytes() and res.labels.tobytes() == w_lab.tobytes()
                            and res.counts.tobytes() == w_cnt.tobytes())
        else:
            row["numpy_ms"] = "not measured"
        emit(rows, row)
        del g, res


def write_dotgraph(path, scale):
    src, dst = oracle.rmat_edges(scale, seed=3)
    n = 1 << scale
    labels = np.random.default_rng(scale).integers(0, 42, n)
    with open(path, "wb") as f:
        f.write(dot.write(labels, list(zip(src.tolist(), dst.tolist()))))
    return n, len(src)


def bench_load(rows, runs, tmp, pinned):
    for scale, paths in ((18, ("host", "device")), (20, ("device",))):
        path = Path(tmp) / f"rmat{scale}.graph"
        n, m = write_dotgraph(path, scale)
        size = path.stat().st_size
        path.read_bytes()  # warm page cache: these are not disk numbers
        for which in paths:
            if which == "device" and size < (64 << 20):
                os.environ["GB_LOAD_CHUNK_BYTES"] = str(64 << 20)
            else:
                os.environ.pop("GB_LOAD_CHUNK_BYTES", None)
            g, ms = timed(lambda: gb.Graph.load_labeled(path, layout=gb.Layout.Sorted), runs)
            os.environ.pop("GB_LOAD_CHUNK_BYTES", None)
            row = {"bench": "load_labeled", "scale": scale, "path": which, "file_bytes": size, "edges": m,
                   "ms": ms, "file_gb_per_s": size / ms / 1e6, "chunks": g.load_info()["chunks"]}
            if which == paths[0]:
                t0 = time.perf_counter()
                want = dot.read(path.read_bytes())
                row["python_read_ms"] = (time.perf_counter() - t0) * 1e3
                row["match"] = g.node_values().tobytes() == want.labels.tobytes()
            emit(rows, row)
            if which != paths[-1]:
                del g
        bench_binary(rows, runs, path.with_suffix(".bin"), g, scale, paths, pinned)
        del g


def bench_binary(rows, runs, path, g, scale, paths, pinned):
    """save_labeled of the DotGraph twin g, then load_labeled of that binary file on each path"""
    _, save_ms = timed(lambda: g.serialize_labeled(path), runs)
    size = path.stat().st_size
    emit(rows, {"bench": "save_labeled", "scale": scale, "file_bytes": size, "ms": save_ms,
                "file_gb_per_s": size / save_ms / 1e6})
    path.read_bytes()  # warm page cache
    floor = min(pread_floor(path, pinned) for _ in range(runs)) * 1e3
    for which in paths:
        if which == "device" and size < (64 << 20):
            os.environ["GB_LOAD_CHUNK_BYTES"] = str(64 << 20)
        else:
            os.environ.pop("GB_LOAD_CHUNK_BYTES", None)
        h, ms = timed(lambda: gb.Graph.load_labeled(path, file_format=gb.FileFormat.Binary), runs)
        os.environ.pop("GB_LOAD_CHUNK_BYTES", None)
        info = h.load_info()
        emit(rows, {"bench": "load_labeled binary", "scale": scale, "path": which, "file_bytes": size,
                    "ms": ms, "file_gb_per_s": size / ms / 1e6, "pread_floor_ms": floor, "over_floor": ms / floor,
                    "chunks": info["chunks"], "h2d_bytes": info["h2d_bytes"],
                    "match": (h.node_values().tobytes() == g.node_values().tobytes()
                              and all(a.tobytes() == b.tobytes() for a, b in zip(h.csr(), g.csr())))})
        del h
    path.unlink()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--nlf-scales", default="22,24")
    ap.add_argument("--cpu-max-scale", type=int, default=22, help="largest RMAT scale the numpy restatement runs")
    ap.add_argument("--cpu-max-nodes", type=int, default=1 << 24, help="largest stats workload the numpy code runs")
    ap.add_argument("--skip-load", action="store_true")
    ap.add_argument("--load-only", action="store_true", help="only the DotGraph and binary file rows")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if gb.device_count() == 0:
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU fallback")
    info = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    rows = []
    emit(rows, {"device": info})
    if not a.load_only:
        bench_stats(rows, a.runs, [1000, 10000, 100000, 1 << 24, 1 << 26], a.cpu_max_nodes)
        bench_nlf(rows, a.runs, [int(s) for s in a.nlf_scales.split(",") if s], a.cpu_max_scale)
    if not a.skip_load:
        import torch  # the pinned buffer of the pread floor
        pinned = torch.empty(4 * (64 << 20), dtype=torch.uint8, pin_memory=True)
        with tempfile.TemporaryDirectory() as tmp:
            bench_load(rows, a.runs, tmp, pinned)
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps(rows, indent=1))


if __name__ == "__main__":
    main()
