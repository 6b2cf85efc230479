#!/usr/bin/env python3
"""Compare the PageRank sweep of two source trees on one GPU: a base tree and the tree under test, each built
in place, run one after the other on the same card.

  python tools/ab_pagerank.py --base DIR --test DIR --out DIR [--repeats 3]

What it runs, alternating the trees wherever a number is compared:
  * the card's name, power limit and max SM clock (nvidia-smi, read only);
  * bench.py --steps 5 --warmup 3 at RMAT-26, `repeats` times per tree, with --dump-outputs;
  * one GB_PR_TRACE=1 bench run per tree at RMAT-26 and at RMAT-25 (per-kernel times of every sweep), the
    RMAT-25 one with --dump-outputs;
  * bench.py at RMAT-22 and RMAT-24 (the SELL path), once per tree;
and writes every bench line, the trace lines and a summary (OUT/ab.json): the GTEPS and e2e of every run, the
kernel times, and whether the two trees' dumped scores are bit-identical at each scale (if not, their largest
relative difference)."""
from __future__ import annotations

import argparse
import json
import os
import re
import subprocess
import sys
from pathlib import Path

import numpy as np


def sh(cmd, cwd, env=None, log=None):
    p = subprocess.run(cmd, cwd=cwd, env={**os.environ, **(env or {})}, capture_output=True, text=True)
    if log:
        Path(log).write_text(f"$ {' '.join(cmd)}\n[exit {p.returncode}]\n--- stdout\n{p.stdout}\n--- stderr\n{p.stderr}")
    return p


def bench(tree, out, tag, args, env=None):
    p = sh([sys.executable, "bench.py", "--gpus", "1", *args], tree, env, log=out / f"{tag}.log")
    line = None
    for l in p.stdout.splitlines():
        if l.startswith("{"):
            line = json.loads(l)
    trace = [l for l in p.stderr.splitlines() if "[gb trace]" in l]
    rec = {"tag": tag, "exit": p.returncode, "trace": trace}
    if line:
        rec.update(value=line.get("value"), e2e=(line.get("e2e") or {}).get("value"), verified=line.get("verified"))
    print(json.dumps({k: rec[k] for k in rec if k != "trace"} | ({"trace": trace[-1:]} if trace else {})),
          flush=True)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True)
    ap.add_argument("--test", required=True)
    ap.add_argument("--out", required=True)
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    out = Path(a.out).resolve()  # bench runs from each tree
    out.mkdir(parents=True, exist_ok=True)
    trees = {"base": Path(a.base).resolve(), "test": Path(a.test).resolve()}
    card = sh(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], ".").stdout
    print(card, flush=True)
    for name, tree in trees.items():
        p = sh([sys.executable, "-c", "import __graft_entry__ as e; e.build()"], tree, log=out / f"build_{name}.log")
        assert p.returncode == 0, f"build of {name} failed: see {out}/build_{name}.log"
    runs = []
    for i in range(a.repeats):
        for name, tree in trees.items():
            runs.append(bench(tree, out, f"s26_{name}_{i}", ["--steps", "5", "--warmup", "3", "--dump-outputs",
                                                            str(out / f"dump26_{name}")]) | {"tree": name})
    for scale, extra in ((26, []), (25, ["--dump-outputs"])):
        for name, tree in trees.items():
            args = ["--scale", str(scale), "--steps", "2", "--warmup", "1", "--no-cpu"]
            if extra:
                args += [extra[0], str(out / f"dump{scale}_{name}")]
            runs.append(bench(tree, out, f"trace{scale}_{name}", args, {"GB_PR_TRACE": "1"}) | {"tree": name})
    for scale in (22, 24):
        for name, tree in trees.items():
            runs.append(bench(tree, out, f"s{scale}_{name}", ["--scale", str(scale), "--steps", "5", "--warmup", "3",
                                                              "--no-cpu"]) | {"tree": name})
    same = {}
    for scale in (26, 25):
        try:
            x, y = (np.load(out / f"dump{scale}_{t}" / "scores.npy") for t in trees)
            same[scale] = bool(np.array_equal(x, y))
            if not same[scale]:  # reordered sums: how far apart, relative to the base tree's scores
                same[scale] = {"max_rel_diff": float(np.max(np.abs(y.astype(np.float64) - x) / np.abs(x)))}
        except OSError as e:
            same[scale] = f"missing: {e}"
    kern = {}
    for r in runs:
        for l in r["trace"]:
            m = re.search(r"k_pr_cb ([\d.]+)\s+pass A ([\d.]+)\s+pass B ([\d.]+)\s+k_pr_finish ([\d.]+)", l)
            if m:  # k_pr_cb and pass A as two launches
                kern[r["tag"]] = dict(zip(("k_pr_cb", "pass_a", "pass_b", "k_pr_finish"), map(float, m.groups())))
            m = re.search(r"k_pr_cb with pass A ([\d.]+)\s+pass B ([\d.]+)\s+k_pr_finish ([\d.]+)", l)
            if m:  # pass A inside k_pr_cb's tasks
                kern[r["tag"]] = dict(zip(("k_pr_cb_with_pass_a", "pass_b", "k_pr_finish"), map(float, m.groups())))
    summary = {"card": card.strip(), "bit_identical_scores": same, "kernel_ms": kern,
               "runs": [{k: r.get(k) for k in ("tag", "tree", "exit", "value", "e2e", "verified")} for r in runs]}
    (out / "ab.json").write_text(json.dumps(summary, indent=1))
    print(json.dumps({"bit_identical_scores": same, "kernel_ms": kern}, indent=1))


if __name__ == "__main__":
    main()
