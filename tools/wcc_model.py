"""wcc_model.py — a CPU replay of gb_wcc (wcc_impl in graph_b200/csrc/wcc.cu), phase by phase.

k_cc_sample + k_cc_compress leave every vertex pointing at the minimum id of its component in the subgraph
of the first `rounds` out-edges of each vertex (of each vertex in [vb, ve) on a shard); `rounds` is the
config's u64 neighbor_rounds clamped to 0xFFFFFFFF.  most_frequent_label draws min(sampling_size, 2^20)
vertices with splitmix64 from the seed 0x5DEECE66D, reads their sampled roots, and takes the label of the
first longest run of the sorted draws: the smallest label among tied counts.  k_cc_link_remaining sees
each vertex as one of
  * dead: nothing past its first `rounds` out-edges and no in-edge;
  * skip: live, but its sampled root is the label (it drops out; a vertex hooked under the label while
    the kernel runs may drop out too, which the replay cannot know and the labels do not depend on);
  * lane: live with at most LANE_WORK remaining entries, linked by its own lane;
  * warp: live with more, served by the whole warp in 32-entry strides over the out-remainder and the
    in-list.
The final labels are the minimum id of each component of the sampled forest plus every edge a live,
unskipped vertex links; `keep_out` / `keep_in` cut the out-remainder or the in-list of some vertices to
their first k entries, so that a test can show which endpoint and which entry a bridge depends on.
Components are found with numpy alone: roots hooked under the lowest root they share an edge with, then
full pointer jumping, until no edge joins two roots.  LANE_WORK is read from wcc.cu.
Run: python tools/wcc_model.py   (also exercised by tests/test_wcc_model.py)."""
from __future__ import annotations

import re
from dataclasses import dataclass
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
LANE_WORK = int(re.search(r"const bool small = live && work <= (\d+);",
                          (ROOT / "graph_b200" / "csrc" / "wcc.cu").read_text()).group(1))
SEED = 0x5DEECE66D
MAX_SAMPLES = 1 << 20
MAX_ROUNDS = 0xFFFFFFFF
DEAD, SKIP, LANE, WARP = "dead", "skip", "lane", "warp"


def clamp_rounds(neighbor_rounds: int) -> int:
    return min(int(neighbor_rounds), MAX_ROUNDS)


def min_label(n: int, a, b) -> np.ndarray:
    """the minimum vertex id of every component of the undirected graph with the edges (a[i], b[i])"""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    p = np.arange(n, dtype=np.int64)          # p[x] <= x, and p[x] == x only at a root
    while True:
        ra, rb = p[a], p[b]                   # every p[x] is a root here
        join = ra != rb
        if not join.any():
            return p.astype(np.uint32)        # each root is the smallest id below it
        np.minimum.at(p, np.maximum(ra, rb)[join], np.minimum(ra, rb)[join])
        while True:
            pp = p[p]
            if (pp == p).all():
                break
            p = pp


def _rows(off, vb: int, ve: int):
    off = np.asarray(off, np.int64)
    return off[vb:ve], off[vb + 1:ve + 1]


def _expand(begin, end, rows):
    """(row, entry index) of every entry in [begin[i], end[i]) of every row rows[i]"""
    lens = end - begin
    row = np.repeat(rows, lens)
    idx = np.arange(lens.sum()) - np.repeat(np.cumsum(lens) - lens, lens) + np.repeat(begin, lens)
    return row, idx


def first_round_edges(off, tgt, rounds: int, vb: int = 0, ve: int | None = None):
    """the edges k_cc_sample links: (u, tgt[i]) for the first `rounds` entries of every row u in [vb, ve)"""
    ve = len(off) - 1 if ve is None else ve
    b, e = _rows(off, vb, ve)
    lim = np.minimum(e, b + clamp_rounds(rounds))
    u, i = _expand(b, lim, np.arange(vb, ve))
    return u, np.asarray(tgt, np.int64)[i]


def sampled_forest(off, tgt, rounds: int, vb: int = 0, ve: int | None = None) -> np.ndarray:
    """parent[] after k_cc_init, k_cc_sample over [vb, ve) and k_cc_compress"""
    u, v = first_round_edges(off, tgt, rounds, vb, ve)
    return min_label(len(off) - 1, u, v)


def sample_draws(n: int, sampling_size: int) -> np.ndarray:
    """the vertices k_cc_sample_labels reads: parent[z % n] for the i-th splitmix64 output z"""
    count = min(int(sampling_size), MAX_SAMPLES)
    with np.errstate(over="ignore"):
        z = np.uint64(SEED) + np.uint64(0x9E3779B97F4A7C15) * np.arange(1, count + 1, dtype=np.uint64)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z ^= z >> np.uint64(31)
    return (z % np.uint64(n)).astype(np.int64)


def sample_counts(forest, sampling_size: int):
    """(labels ascending, how often each was drawn)"""
    if len(forest) == 0 or sampling_size == 0:
        return np.zeros(0, np.uint32), np.zeros(0, np.int64)
    return np.unique(np.asarray(forest)[sample_draws(len(forest), sampling_size)], return_counts=True)


def sample_label(forest, sampling_size: int):
    """(label, found) of most_frequent_label: the first longest run of the sorted draws"""
    labels, counts = sample_counts(forest, sampling_size)
    if len(labels) == 0:
        return 0, False
    return int(labels[np.argmax(counts)]), True


def kernel_launches(rounds: int, found: bool) -> int:
    """init, sample (rounds > 0), compress, sample labels (a label was drawn), link_remaining, compress"""
    return 2 + (clamp_rounds(rounds) > 0) + bool(found) + 2


@dataclass
class Classes:
    cls: np.ndarray        # DEAD / SKIP / LANE / WARP per vertex of the range
    out_len: np.ndarray    # the out-remainder: entries past the first `rounds`
    in_len: np.ndarray


def classify(out_off, in_off, forest, rounds: int, label: int, found: bool, vb: int = 0,
             ve: int | None = None) -> Classes:
    """what k_cc_link_remaining does with every vertex of [vb, ve), the skip test taken on the forest
    the kernel starts from"""
    ve = len(out_off) - 1 if ve is None else ve
    ob, oe = _rows(out_off, vb, ve)
    ib, ie = _rows(in_off, vb, ve)
    out_len = np.maximum(oe - ob - clamp_rounds(rounds), 0)
    in_len = ie - ib
    live = (out_len > 0) | (in_len > 0)
    skip = live & found & (np.asarray(forest)[vb:ve] == label)
    cls = np.where(~live, DEAD, np.where(skip, SKIP, np.where(out_len + in_len <= LANE_WORK, LANE, WARP)))
    return Classes(cls, out_len, in_len)


def _keep(b, e, keep):
    """cut the rows v of `keep` to their first keep[v] entries"""
    if keep:
        v = np.fromiter(keep, np.int64)
        e = e.copy()
        e[v] = np.minimum(e[v], b[v] + np.fromiter(keep.values(), np.int64))
    return e


def remaining_edges(out_off, out_tgt, in_off, in_tgt, rounds: int, linking, keep_out=None, keep_in=None):
    """the edges k_cc_link_remaining links for the vertices where `linking` holds; keep_out / keep_in:
    {v: k} links only the first k entries of v's out-remainder / in-list"""
    n = len(out_off) - 1
    u = np.flatnonzero(linking)
    b, e = _rows(out_off, 0, n)
    b = np.minimum(e, b + clamp_rounds(rounds))
    e = _keep(b, e, keep_out)
    u1, i1 = _expand(b[u], e[u], u)
    b, e = _rows(in_off, 0, n)
    e = _keep(b, e, keep_in)
    u2, i2 = _expand(b[u], e[u], u)
    return (np.concatenate([u1, u2]),
            np.concatenate([np.asarray(out_tgt, np.int64)[i1], np.asarray(in_tgt, np.int64)[i2]]))


@dataclass
class Replay:
    forest: np.ndarray
    label: int
    found: bool
    classes: Classes
    labels: np.ndarray
    launches: int


def replay(out_off, out_tgt, in_off, in_tgt, neighbor_rounds: int = 2, sampling_size: int = 1024,
           keep_out=None, keep_in=None) -> Replay:
    n = len(out_off) - 1
    forest = sampled_forest(out_off, out_tgt, neighbor_rounds)
    label, found = sample_label(forest, sampling_size)
    c = classify(out_off, in_off, forest, neighbor_rounds, label, found)
    u, v = remaining_edges(out_off, out_tgt, in_off, in_tgt, neighbor_rounds, (c.cls == LANE) | (c.cls == WARP),
                           keep_out, keep_in)
    labels = min_label(n, np.concatenate([np.arange(n), u]), np.concatenate([forest, v]))
    return Replay(forest, label, found, c, labels, kernel_launches(neighbor_rounds, found))


if __name__ == "__main__":
    import sys
    sys.path.insert(0, str(ROOT))
    import oracle
    src, dst = oracle.rmat_edges(12, seed=42)
    out = oracle.csr_build(src, dst, 1 << 12, oracle.OUTGOING, oracle.SORTED)
    inc = oracle.csr_build(src, dst, 1 << 12, oracle.INCOMING, oracle.SORTED)
    r = replay(*out, *inc)
    kinds, counts = np.unique(r.classes.cls, return_counts=True)
    print("label", r.label, "launches", r.launches, dict(zip(kinds.tolist(), counts.tolist())),
          "labels == oracle:", bool((r.labels == oracle.wcc_min_label(*out)).all()))
