#!/usr/bin/env python3
"""The reference's end-to-end walk-through (crates/algos/examples/usage-demo.rs and
crates/mate/notebooks/usage-demo.ipynb) against graph_b200: load a Graph500 file, PageRank, WCC,
to_undirected, make_degree_ordered, triangle count.  Needs an H100.

  python examples/usage_demo.py [path.graph500]      # default: synthetic RMAT scale-20 written to /tmp
"""
import sys
import time
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import graph_mate as gm  # noqa: E402  (the reference's module name, bound to graph_b200)
import graph_b200 as gb  # noqa: E402


def timed(label, fn):
    t0 = time.perf_counter()
    out = fn()
    print(f"{label}: {1e3 * (time.perf_counter() - t0):.1f} ms")
    return out


def main():
    if len(sys.argv) > 1:
        path = sys.argv[1]
    else:
        # no dataset at hand: emit a synthetic R-MAT graph in the reference's own input format
        path = "/tmp/rmat_scale20.graph500"
        tmp = gb.DiGraph.rmat(20, seed=42)
        off, tgt = tmp.csr("out")
        src = np.repeat(np.arange(tmp.node_count(), dtype=np.uint32), np.diff(off.astype(np.int64)))
        gb.write_graph500(path, src, tgt)
        del tmp
    g = timed("load (Deduplicated)", lambda: gm.DiGraph.load(path, layout=gm.Layout.Deduplicated))
    print(g)

    pr = timed("page_rank", lambda: g.page_rank())
    s = pr.scores()
    print(pr)
    print(f"size = {len(s)}  min = {s.min():.3e}  max = {s.max():.3e}  mean = {s.mean():.3e}  median = {np.median(s):.3e}")

    wcc = timed("wcc", lambda: g.wcc())
    print(f"component count = {len(np.unique(wcc.components()))}")

    ug = timed("to_undirected (Deduplicated)", lambda: g.to_undirected(gm.Layout.Deduplicated))
    del g  # the undirected graph is a full copy, not a view
    timed("make_degree_ordered", ug.make_degree_ordered)
    tc = timed("global_triangle_count", ug.global_triangle_count)
    print(f"TC: found {tc.triangles} triangles.")


if __name__ == "__main__":
    main()
