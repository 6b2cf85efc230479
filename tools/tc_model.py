"""tc_model.py — a one-thread replay of gb_triangle_count (graph_b200/csrc/tc.cu), item by item.

Rows are checked for order the way k_tc_rows_unsorted does: a descent inside a row makes them unsorted, one
across a row boundary does not.  Sorted rows replay k_tc: one item per CSR entry (u, v) with v <= u; both
lists are cut to values <= v with the kernel's upper bound, the item is live when both cuts are non-empty,
the walked list is N(u) when lu * bitlen(lv) < lv * bitlen(lu) (by_u) and N(v) otherwise (by_v), a walk of
at most TC_SHORT entries stays in one lane ("short") and a longer one goes to the warp in steps of 32
("long").  The by_u side counts a value at its first occurrence only; on the warp path that is the
tgt[j-1] != w test, which reads across a 32-entry step when a run of equal values straddles one.  Every
binary search is the kernel's own (bisect is the same lower / upper bound), so the replay gives what the
kernel gives even on rows it was not written for.  Unsorted rows replay k_tc_cut + k_tc_list: the
reference loop in list order.

The replay also tallies which (direction, short/long) classes the items reach, the walk lengths, and the
runs of repeated values on long by_u walks, so that a test can check on the CPU that a fixture still
reaches the path it is named for after TC_SHORT (read from tc.cu) or the direction rule changes.
Run: python tools/tc_model.py   (also exercised by tests/test_tc_model.py)."""
from __future__ import annotations

import re
from bisect import bisect_left, bisect_right
from collections import Counter
from dataclasses import dataclass, field
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
TC_SHORT = int(re.search(r"constexpr uint32_t TC_SHORT = (\d+);",
                         (ROOT / "graph_b200" / "csrc" / "tc.cu").read_text()).group(1))
STEP = 32   # entries a warp walks per step


def rows_sorted(off, tgt) -> bool:
    """k_tc_rows_unsorted: no tgt[i-1] > tgt[i] where entry i does not begin a row"""
    off = np.asarray(off, np.int64)
    tgt = np.asarray(tgt, np.int64)
    if len(tgt) < 2:
        return True
    begins = np.zeros(len(tgt), bool)
    begins[off[:-1][off[:-1] < len(tgt)]] = True
    return not ((tgt[1:] < tgt[:-1]) & ~begins[1:]).any()


def by_u_rule(lu: int, lv: int) -> bool:
    """k_tc's direction: walk N(u) when that costs fewer lookups; ties go to N(v)"""
    return lu * lv.bit_length() < lv * lu.bit_length()


@dataclass
class SortedReplay:
    count: int = 0
    classes: Counter = field(default_factory=Counter)   # (direction, "short" | "long") -> live items
    walks: Counter = field(default_factory=Counter)     # (direction, walk length) -> live items
    runs: Counter = field(default_factory=Counter)      # (offset in the walk, length) of repeated values, long by_u
    crossings: int = 0                                  # of those runs, the ones that straddle a 32-entry step


def replay_sorted(off, tgt) -> SortedReplay:
    """k_tc on (off, tgt), entry by entry"""
    off = [int(x) for x in off]
    t = [int(x) for x in tgt]
    n = len(off) - 1
    r = SortedReplay()
    for u in range(n):
        ub, ue_row = off[u], off[u + 1]
        for i in range(ub, ue_row):
            v = t[i]
            if v > u:
                continue
            vb = off[v]
            ve = bisect_right(t, v, vb, off[v + 1])
            ue = bisect_right(t, v, ub, ue_row)
            if not (ve > vb and ue > ub):
                continue
            lu, lv = ue - ub, ve - vb
            by_u = by_u_rule(lu, lv)
            walk_b, walk_e, find_b, find_e = (ub, ue, vb, ve) if by_u else (vb, ve, ub, ue)
            walk = walk_e - walk_b
            direction = "by_u" if by_u else "by_v"
            is_short = walk <= TC_SHORT
            r.classes[(direction, "short" if is_short else "long")] += 1
            r.walks[(direction, walk)] += 1
            for j in range(walk_b, walk_e):
                w = t[j]
                if by_u:
                    if j == walk_b or t[j - 1] != w:   # first occurrence (the lane's `prev` is the same test)
                        lo = bisect_left(t, w, find_b, find_e)
                        r.count += bisect_right(t, w, lo, find_e) - lo
                else:
                    p = bisect_left(t, w, find_b, find_e)
                    r.count += 1 if p < find_e and t[p] == w else 0
            if by_u and not is_short:
                j = walk_b
                while j < walk_e:
                    k = j
                    while k + 1 < walk_e and t[k + 1] == t[j]:
                        k += 1
                    if k > j:
                        a, b = j - walk_b, k - walk_b
                        r.runs[(a, b - a + 1)] += 1
                        r.crossings += a // STEP != b // STEP
                    j = k + 1
    return r


def row_cut(off, tgt) -> list:
    """k_tc_cut: the first index of row u whose target is > u, else off[u + 1]"""
    off = np.asarray(off, np.int64)
    tgt = np.asarray(tgt, np.int64)
    n = len(off) - 1
    rows = np.repeat(np.arange(n), np.diff(off))
    over = np.flatnonzero(tgt > rows)
    cut = off[1:].copy()
    np.minimum.at(cut, rows[over], over)
    return cut.tolist()


def replay_list_order(off, tgt) -> int:
    """k_tc_cut + k_tc_list: one item per entry i < cut[u], a put-back cursor over N(u), list order"""
    off = [int(x) for x in off]
    t = [int(x) for x in tgt]
    cut = row_cut(off, t)
    total = 0
    for u in range(len(off) - 1):
        ue = off[u + 1]
        for i in range(off[u], cut[u]):
            v = t[i]
            it = off[u]
            for j in range(off[v], cut[v]):
                w = t[j]
                while it < ue and t[it] < w:
                    it += 1
                if it == ue:
                    break
                total += t[it] == w
    return total


def triangle_count(off, tgt) -> int:
    """what gb_triangle_count returns for this CSR"""
    return replay_sorted(off, tgt).count if rows_sorted(off, tgt) else replay_list_order(off, tgt)


if __name__ == "__main__":
    import sys
    sys.path.insert(0, str(ROOT))
    import oracle
    for scale in (8, 10):
        s, d = oracle.rmat_edges(scale, seed=42)
        for name, lay in (("Unsorted", oracle.UNSORTED), ("Sorted", oracle.SORTED)):
            o, g = oracle.csr_build(s, d, 1 << scale, oracle.UNDIRECTED, lay)
            rs = replay_sorted(o, g)
            print(f"RMAT-{scale} {name}: rows sorted {rows_sorted(o, g)}, oracle {oracle.triangle_count(o, g)}, "
                  f"model {triangle_count(o, g)}, k_tc alone {rs.count}, classes {dict(rs.classes)}")
