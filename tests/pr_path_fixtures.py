"""Graphs that steer the JACOBI PageRank layout (graph_b200/csrc/pagerank.cu, build_pr_plan) onto its less
common paths, and the path each is meant to reach.  Shared by the CPU check against the layout model
(test_pr_path_model.py) and the GPU tests (test_gpu_pr_paths.py), so that a retuned default that moves a
graph off its path fails on the CPU already instead of silently thinning the GPU coverage."""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import layout_model as lm  # noqa: E402

import oracle  # noqa: E402

TAIL_R = (1, 2, 3, 5, 33)
# every environment knob of the plan build and the sweep (graph_b200/csrc/pagerank.cu)
KNOBS = ("GB_PR_BLOCK", "GB_PR_TAU", "GB_PR_MIN_BLOCK", "GB_PR_MEGA", "GB_PR_CHUNK", "GB_PR_TASK_CHUNKS",
         "GB_PR_DUAL", "GB_PR_DEBUG", "GB_PR_FIN_U", "GB_PR_FIN_SPLIT", "GB_PR_FEED_CHUNKS", "GB_PR_FEED_MIN_EDGES")


def tail_block(r):
    """n = 8 * 1024 + r.  Every vertex sends two edges to hub 0 (kept by Sorted), one along a random
    permutation (every in-degree >= 1) and n/8 more at random, so that the last block in the internal
    order (in-degree 1, out-degree 3: the last ids) is hot for the hub row and holds r entries: the scalar
    tail of the block load (r <= 3: no bulk copy at all)."""
    rng = np.random.default_rng(100 + r)
    n = 8 * 1024 + r
    v = np.arange(1, n, dtype=np.uint32)
    src = np.concatenate([v, v, np.arange(n, dtype=np.uint32), rng.integers(0, n, n // 8).astype(np.uint32)])
    dst = np.concatenate([np.zeros(2 * (n - 1), np.uint32), rng.permutation(n).astype(np.uint32),
                          rng.integers(0, n, n // 8).astype(np.uint32)])
    return src, dst, n


def equal_degrees(n=20001, d=32):
    """every in- and out-degree is d (a union of d random permutations): the degree keys all tie and the
    staircase is a rectangle; n is odd, so the last SELL slice and the last finish group are partial"""
    rng = np.random.default_rng(5)
    src = np.tile(np.arange(n, dtype=np.uint32), d)
    dst = np.concatenate([rng.permutation(n).astype(np.uint32) for _ in range(d)])
    return src, dst, n


def star_in(n=200003):
    """every vertex points to hub 0: one row of ~2e5 in-edges (the sort path of the layout build at the
    default threshold) whose block segments are cut by chunk boundaries at the default knobs"""
    v = np.arange(1, n, dtype=np.uint32)
    return v, np.zeros(n - 1, np.uint32), n


def repeated_source(reps=50000):
    """row 5's in-list is source 77 repeated `reps` times, on an RMAT-15 background"""
    src, dst = oracle.rmat_edges(15, seed=9)
    src = np.concatenate([src, np.full(reps, 77, np.uint32)])
    dst = np.concatenate([dst, np.full(reps, 5, np.uint32)])
    return src, dst, 1 << 15


def few_active(rows=20, blocks=150):
    """only `rows` rows have in-edges (fewer than one 32-row group), from sources in `blocks` blocks of
    1024: the hub group of k_pr_finish is partial and there is no tail"""
    n = blocks * 1024 + 7
    v = np.arange(n, dtype=np.uint32)
    targets = (np.arange(rows, dtype=np.uint32) * 7001 + 3) % n
    return v, targets[v % rows], n


def rmat18():
    """RMAT-18 (seed 7) at GB_PR_BLOCK=1024: 148 hot blocks and 6 hub groups in k_pr_finish"""
    src, dst = oracle.rmat_edges(18, seed=7)
    return src, dst, 1 << 18


def capped_finish(n_reg=586 * 1024 - 1, d=16, thin_blocks=70):
    """~6e5 rows with segments in 6 blocks and one hub row with segments in 76: at GB_PR_FIN_U=2 the finish
    grid is capped (every warp walks several row groups), and GB_PR_FIN_SPLIT=1 splits it anyway.
    Internal order: hub, the n_reg rows of in-degree d, 6 blocks of heavy sources, thin_blocks blocks of
    sources with one edge each to the hub."""
    rng = np.random.default_rng(11)
    heavy0 = 1 + n_reg
    thin0 = heavy0 + 6 * 1024
    n = thin0 + thin_blocks * 1024
    rows = np.repeat(np.arange(1, heavy0, dtype=np.uint32), d)
    src = np.concatenate([rng.integers(heavy0, thin0, len(rows)).astype(np.uint32),
                          np.arange(thin0, n, dtype=np.uint32)])
    dst = np.concatenate([rows, np.zeros(n - thin0, np.uint32)])
    return src, dst, n


# name -> (builder, GB_PR_BLOCK or None for the default)
FIXTURES = {
    **{f"tail_r{r}": (lambda r=r: tail_block(r), 1024) for r in TAIL_R},
    "equal_degrees": (equal_degrees, 1024),
    "star_in": (star_in, None),
    "repeated_source": (repeated_source, None),
    "few_active": (few_active, 1024),
    "rmat18": (rmat18, 1024),
    "capped_finish": (capped_finish, 1024),
}

_CACHE: dict = {}


def set_knobs(monkeypatch, name, **env):
    """every knob unset except the fixture's GB_PR_BLOCK and `env`"""
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    block = FIXTURES[name][1] if name in FIXTURES else None
    if block:
        monkeypatch.setenv("GB_PR_BLOCK", str(block))
    for k, v in env.items():
        monkeypatch.setenv(k, str(v))


def graph(name):
    """(src, dst, n, out CSR, in CSR) of a fixture, Sorted layout (duplicates kept), cached"""
    if name not in _CACHE:
        src, dst, n = FIXTURES[name][0]()
        out = oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED)
        inc = oracle.csr_build(src, dst, n, oracle.INCOMING, oracle.SORTED)
        _CACHE.clear()   # keep one graph at a time: the large ones hold ~100 MB
        _CACHE[name] = (src, dst, n, out, inc)
    return _CACHE[name]


def model(name, P=1, p=0, sms=lm.H100_SMS, **knobs):
    """the layout model's plan, launch shape and layout statistics for a fixture at its knobs"""
    _, _, n, out, inc = graph(name)
    B = lm.clamp_block(FIXTURES[name][1] or lm.CB_BLOCK_DEFAULT)
    plan = lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)), B, lm.CB_TAU_DEFAULT,
                        P=P, p=p)
    return plan, lm.launch_shape(plan, sms=sms, **knobs), lm.layout_counts(plan, inc[0], inc[1])


def check_path(name, plan, shape):
    """the path each fixture was built for; returns a one-line description (AssertionError otherwise)"""
    n = plan["n"]
    if name.startswith("tail_r"):
        r = int(name[6:])
        assert n % plan["B"] == r and shape["last_hot_block"] == plan["nblk"] - 1, "the partial last block is hot"
        return f"last block {plan['nblk'] - 1} hot with {r} entries ({r & ~3} by bulk copy)"
    if name == "equal_degrees":
        assert n % 32 and n % 2 and (plan["nrows"] == plan["nrows"][0]).all() and shape["n_fin"] == n
        return f"rectangular staircase: {shape['hot_blocks']} blocks x {plan['nrows'][0]} rows, n_fin {shape['n_fin']}"
    if name == "star_in":
        assert shape["n_mega"] == 1 and shape["n_cb"] == 1 and shape["hot_blocks"] > 1
        return f"one mega row across {shape['hot_blocks']} blocks"
    if name == "repeated_source":
        assert shape["n_mega"] >= 1
        return f"{shape['n_mega']} mega rows, one of them a single source repeated"
    if name == "few_active":
        assert plan["n_active"] < 32 and shape["hot_blocks"] >= 100 and shape["n_fin_warp"] == shape["n_fin"] < 32
        return f"{plan['n_active']} active rows over {shape['hot_blocks']} hot blocks: one partial hub group"
    if name == "rmat18":
        assert shape["n_fin_warp"] > 0 and shape["hot_blocks"] > lm.FIN_CTA_BLOCKS
        assert shape["fin_u"] == 2 and shape["fin_hub_ctas"] == 0 and not shape["grid_capped"]
        return (f"{shape['n_fin_warp'] // 32} hub groups, {shape['hot_blocks']} blocks, n_fin {shape['n_fin']}, "
                f"fin_u 2, no split")
    if name == "capped_finish":
        assert shape["fin_u"] == 4 and shape["n_fin_warp"] == 32 and not shape["grid_capped"]
        return f"fin_u 4 at {shape['grid_fin']} finish CTAs; n_fin {shape['n_fin']}"
    raise KeyError(name)
