#!/usr/bin/env python3
"""Secondary configs of BASELINE.json (WCC scale-24, triangle count scale-22, SSSP) timed on one GPU
next to the oracle's multi-threaded CPU port.  One JSON line per algorithm.
  python tools/bench_algos.py [--wcc-scale 24] [--tc-scale 22] [--sssp-scale 22] [--cpu]"""
import argparse, json, sys, time
from pathlib import Path
import numpy as np
ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import graph_b200 as gb

PEAK = 3350.0  # GB/s, H100 SXM data sheet
try:
    PEAK = float(json.loads((ROOT / "MEASURED_PEAKS.json").read_text())["hbm_gbs"])
except Exception:
    pass


def timed(fn, reps=3, warm=1):
    for _ in range(warm):
        out = fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter(); out = fn(); ts.append(time.perf_counter() - t0)
    return out, min(ts), float(np.mean(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--wcc-scale", type=int, default=24)
    ap.add_argument("--tc-scale", type=int, default=22)
    ap.add_argument("--sssp-scale", type=int, default=22)
    ap.add_argument("--cpu", action="store_true")
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    want = set(a.only.split(",")) if a.only else {"wcc", "tc", "sssp"}
    if "wcc" in want:
        s = a.wcc_scale; n = 1 << s; m = 16 * n
        g = gb.DiGraph.rmat(s, seed=42, layout=gb.Layout.Sorted)
        res, best, mean = timed(lambda: g.wcc())
        dev_ms = g.last_timing()["total_ms"]
        byts = 8 * m + 16 * n + 8
        line = {"algo": "wcc_afforest", "scale": s, "device_ms": dev_ms, "call_ms_best": best * 1e3,
                "edges_per_s": m / (dev_ms * 1e-3), "effective_GBps": byts / (dev_ms * 1e-3) / 1e9,
                "frac_of_hbm_peak": byts / (dev_ms * 1e-3) / 1e9 / PEAK,
                "components": int(len(np.unique(res.components())))}
        if a.cpu:
            import oracle
            oo, ot = g.csr("out"); io, it = g.csr("in")
            oracle.wcc_afforest(oo, ot, io, it, threads=0)
            t0 = time.perf_counter(); c = oracle.wcc_afforest(oo, ot, io, it, threads=0); dt = time.perf_counter() - t0
            line["cpu_ms"] = dt * 1e3; line["cpu_threads"] = oracle.hardware_threads()
            line["bit_exact_vs_cpu"] = bool((c == res.components()).all())
        print(json.dumps(line), flush=True)
        del g
    if "tc" in want:
        s = a.tc_scale; n = 1 << s; m = 16 * n
        ug = gb.Graph.rmat(s, seed=42, layout=gb.Layout.Sorted)
        res, best, mean = timed(lambda: ug.global_triangle_count(), reps=1, warm=0)
        dev_ms = ug.last_timing()["total_ms"]
        t0 = time.perf_counter(); ug.make_degree_ordered(); relabel_s = time.perf_counter() - t0
        res2, best2, _ = timed(lambda: ug.global_triangle_count(), reps=2, warm=0)
        dev_ms2 = ug.last_timing()["total_ms"]
        byts = 8 * m + 4 * (n + 1)
        line = {"algo": "global_triangle_count", "scale": s, "triangles_sorted": res.triangles, "device_ms_sorted": dev_ms,
                "relabel_ms": relabel_s * 1e3, "triangles_degree_ordered": res2.triangles, "device_ms_degree_ordered": dev_ms2,
                "compulsory_GBps_degree_ordered": byts / (dev_ms2 * 1e-3) / 1e9}
        if a.cpu:
            import oracle
            off, tgt = ug.csr()
            t0 = time.perf_counter(); c = oracle.triangle_count(off, tgt, threads=0); dt = time.perf_counter() - t0
            line["cpu_ms_degree_ordered"] = dt * 1e3; line["cpu_threads"] = oracle.hardware_threads()
            line["bit_exact_vs_cpu"] = bool(c == res2.triangles)
        print(json.dumps(line), flush=True)
        del ug
    if "sssp" in want:
        s = a.sssp_scale; n = 1 << s; m = 16 * n
        g = gb.DiGraph.rmat(s, seed=42, layout=gb.Layout.Sorted, weights=True)
        off, _ = g.csr("out")
        start = int(np.argmax(np.diff(off.astype(np.int64))))
        delta = 0.05
        res, best, mean = timed(lambda: g.delta_stepping(start_node=start, delta=delta), reps=2)
        dev_ms = g.last_timing()["total_ms"]
        d = res.distances()
        byts = 8 * m + 4 * (n + 1) + 8 * n
        line = {"algo": "delta_stepping", "scale": s, "delta": delta, "device_ms": dev_ms, "launches": g.last_timing()["kernel_launches"],
                "reached": int((d < np.finfo(np.float32).max).sum()), "edges_per_s": m / (dev_ms * 1e-3),
                "frac_of_hbm_peak": byts / (dev_ms * 1e-3) / 1e9 / PEAK}
        if a.cpu:
            import oracle
            off, tgt = g.csr("out"); w = g.out_weights()
            t0 = time.perf_counter(); c = oracle.sssp_delta_stepping(off, tgt, w, start, delta); dt = time.perf_counter() - t0
            line["cpu_ms_single_thread"] = dt * 1e3
            line["bit_exact_vs_cpu"] = bool(c.tobytes() == d.tobytes())
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
