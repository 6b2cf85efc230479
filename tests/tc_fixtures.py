"""Undirected CSRs that drive gb_triangle_count (graph_b200/csrc/tc.cu) onto each of its paths: k_tc's walk
lengths around TC_SHORT and the 32-entry warp step in both directions, repeated values on either list, self
loops, the row search at empty and crowded rows, and rows that are not sorted (the list-order path).
Shared by the CPU replay of the kernel (test_tc_model.py) and the GPU tests (test_gpu_tc.py).

Most fixtures put one live item (u, v) on the two highest ids and give u and v their other neighbours
among the low ids, so that every neighbour counts toward the `<= v` prefixes: lu = |N(u)| (v included,
through the edge u-v) and lv = |N(v)| (u excluded).  A list four times longer on the other side forces the
direction (k_tc walks N(u) iff lu * bitlen(lv) < lv * bitlen(lu))."""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

import oracle

SHORT = 16   # TC_SHORT in tc.cu, as the fixture names assume it
WALKS = (1, 15, 16, 17, 31, 32, 33, 63, 64, 65)


@dataclass
class Fixture:
    off: np.ndarray
    tgt: np.ndarray
    edges: np.ndarray | None = None     # (m, 2) edge list whose `layout` build is (off, tgt); None: CSR only
    layout: str | None = None           # "Sorted" | "Unsorted"
    sorted_rows: bool = True            # no descent inside a row: k_tc, else the list-order path
    walks: set = field(default_factory=set)      # (direction, walk length) that some live item must reach
    classes: set = field(default_factory=set)    # (direction, "short" | "long") that some live item must reach
    runs: set = field(default_factory=set)       # (walk offset, length) of a repeated run on a long by_u walk
    crossing: bool = False              # some such run straddles a 32-entry step

    @property
    def n(self) -> int:
        return len(self.off) - 1


_LAYOUT = {"Sorted": oracle.SORTED, "Unsorted": oracle.UNSORTED}


def from_edges(src, dst, n, layout="Sorted", **expect) -> Fixture:
    src, dst = np.asarray(src, np.uint32), np.asarray(dst, np.uint32)
    off, tgt = oracle.csr_build(src, dst, n, oracle.UNDIRECTED, _LAYOUT[layout])
    return Fixture(off, tgt, np.stack([src, dst], 1), layout, **expect)


def from_csr(rows, **expect) -> Fixture:
    off = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.uint32)
    tgt = np.array([x for r in rows for x in r], np.uint32)
    return Fixture(off, tgt, **expect)


def pair(nu, nv, extra=(), **expect) -> Fixture:
    """the edge u-v on the two highest ids (v = T, u = T + 1, T above every low id), an edge u-x for every x
    of nu and v-x for every x of nv (a repeated x is a parallel edge), and `extra` edges among low ids"""
    low = list(nu) + list(nv) + [a for e in extra for a in e]
    t = max(low, default=-1) + 1
    u, v = t + 1, t
    src = [u] * len(nu) + [v] * len(nv) + [u] + [a for a, _ in extra]
    dst = list(nu) + list(nv) + [v] + [b for _, b in extra]
    return from_edges(src, dst, t + 2, **expect)


def kind(walk: int) -> str:
    return "short" if walk <= SHORT else "long"


# ---- walk lengths ---------------------------------------------------------------------------------------
def walk(direction: str, length: int) -> Fixture:
    """the item (u, v) walks `length` entries of N(u) (by_u) or N(v) (by_v); the other list is 4x longer and
    about half of the shorter one's low ids are shared, spread over the list"""
    lu, lv = (length, 4 * length) if direction == "by_u" else (4 * length, length)
    shared = (min(lu - 1, lv) + 1) // 2
    ids = np.random.default_rng(lu * 1000 + lv).permutation((lu - 1) + lv - shared)
    nu = np.sort(ids[:lu - 1])
    nv = np.sort(np.concatenate([ids[:shared], ids[lu - 1:]]))
    return pair(nu, nv, walks={(direction, length)}, classes={(direction, kind(length))})


# ---- repeated values --------------------------------------------------------------------------------------
def run_by_u(at: int, reps: int) -> Fixture:
    """long by_u walk with a run of `reps` copies of x = `at` starting at walk offset `at`; x is twice in N(v),
    so a value counted at every occurrence instead of its first would add 2 * (reps - 1)"""
    x = at
    nu = list(range(x)) + [x] * reps + list(range(x + 1, x + 13))
    lu = len(nu) + 1
    shared = [y for y in range(0, x + 13, 2) if y != x]
    nv = shared + [x, x]
    nv += list(range(x + 13, x + 13 + 4 * lu - len(nv)))
    crosses = at // 32 != (at + reps - 1) // 32
    return pair(nu, nv, classes={("by_u", "long")}, runs={(at, reps)}, crossing=crosses)


def repeated_w_in_v(long: bool) -> Fixture:
    """by_v walk over N(v) holding values 1-3 times each, all of them in N(u): every occurrence counts"""
    k = 20 if long else 6
    nv = [y for y in range(k) for _ in range(y % 3 + 1)]
    nu = list(range(k + 4 * len(nv)))
    return pair(nu, nv, walks={("by_v", len(nv))}, classes={("by_v", kind(len(nv)))})


def repeated_x_in_u() -> Fixture:
    """long by_v walk over 20 distinct values, each three times in N(u): each counts once"""
    nv = list(range(20))
    nu = [y for y in range(20) for _ in range(3)] + list(range(20, 101))
    return pair(nu, nv, walks={("by_v", 20)}, classes={("by_v", "long")})


def clique(k, base=0):
    a, b = np.triu_indices(k, 1)
    return (a + base).astype(np.uint32), (b + base).astype(np.uint32)


def self_loops(reps: int, with_clique: bool = True) -> Fixture:
    if with_clique:
        s, d = clique(6)
        loops = np.repeat(np.arange(6), reps)
        return from_edges(np.concatenate([s, loops]), np.concatenate([d, loops]), 6)
    loops = np.array([0, 1, 1, 3, 3, 3])
    return from_edges(loops, loops, 5)


# ---- the row search ----------------------------------------------------------------------------------------
def empty_rows() -> Fixture:
    """rows 0..23 and 41..63 are empty: a K8 on 24..31 and chords among 24..40"""
    s, d = clique(8, 24)
    rng = np.random.default_rng(11)
    cs, cd = rng.integers(24, 41, 30), rng.integers(24, 41, 30)
    return from_edges(np.concatenate([s, cs]), np.concatenate([d, cd]), 64)


def star_last_row() -> Fixture:
    """a star on row n-1 = 39 with the chords (2i, 2i+1), one of them twice"""
    leaves = np.arange(39)
    cs, cd = np.arange(0, 38, 2), np.arange(1, 38, 2)
    return from_edges(np.concatenate([np.full(39, 39), cs, [0]]), np.concatenate([leaves, cd, [1]]), 40)


def all_in_last_row() -> Fixture:
    """a CSR whose every entry is in row n-1 (not symmetric: from_csr does not ask for that)"""
    return from_csr([[]] * 19 + [[0, 2, 3, 3, 7, 19, 19]])


def single_vertex() -> Fixture:
    return from_edges([0, 0, 0], [0, 0, 0], 1)


def straddle() -> Fixture:
    """a K40 and random chords over 100 ids: 32-entry warps start in the middle of rows"""
    s, d = clique(40)
    rng = np.random.default_rng(12)
    cs, cd = rng.integers(0, 100, 25), rng.integers(0, 100, 25)
    return from_edges(np.concatenate([s, cs]), np.concatenate([d, cd]), 100,
                      classes={("by_u", "short"), ("by_u", "long"), ("by_v", "short"), ("by_v", "long")})


# ---- a total above 2^32 -----------------------------------------------------------------------------------
def multi_clique_edges(n: int, reps: int):
    """K_n with every edge `reps` times"""
    s, d = clique(n)
    return np.tile(s, reps), np.tile(d, reps)


def multi_clique_count(n: int, reps: int) -> int:
    """each triangle a > b > c is counted once per occurrence of b in N(a) and of c in N(b); the repeats of c
    in N(a) do not add"""
    return reps * reps * math.comb(n, 3)


# ---- rows out of order --------------------------------------------------------------------------------------
def rows_of(f: Fixture):
    return [f.tgt[f.off[u]:f.off[u + 1]].tolist() for u in range(f.n)]


def holes() -> Fixture:
    """sorted rows that drop at every row boundary: a clique on 0..12 without 6, and 6-2, 6-4.  Row 6 is
    [2, 4] and row 12 is the last one"""
    s, d = clique(13)
    keep = (s != 6) & (d != 6)
    return from_edges(np.concatenate([s[keep], [6, 6]]), np.concatenate([d[keep], [2, 4]]), 13)


def swap_in_row(rows, u, j) -> Fixture:
    rows = [list(r) for r in rows]
    rows[u][j], rows[u][j + 1] = rows[u][j + 1], rows[u][j]
    return from_csr(rows, sorted_rows=False)


def rmat_sorted_rows(scale=8):
    s, d = oracle.rmat_edges(scale, seed=42)
    return rows_of(from_edges(s, d, 1 << scale))


def shuffled_rows() -> Fixture:
    rng = np.random.default_rng(7)
    return from_csr([rng.permutation(r).tolist() for r in rmat_sorted_rows()], sorted_rows=False)


def descending_rows() -> Fixture:
    return from_csr([r[::-1] for r in rmat_sorted_rows()], sorted_rows=False)


def rmat_unsorted(scale: int) -> Fixture:
    s, d = oracle.rmat_edges(scale, seed=42)
    return from_edges(s, d, 1 << scale, layout="Unsorted", sorted_rows=False)


FIXTURES = {
    **{f"walk_{d}_{k}": (lambda d=d, k=k: walk(d, k)) for d in ("by_u", "by_v") for k in WALKS},
    **{f"run_by_u_at_{a}": (lambda a=a: run_by_u(a, 3)) for a in (30, 31, 32, 33)},
    "run_by_u_40": lambda: run_by_u(10, 40),
    "repeated_w_in_v_short": lambda: repeated_w_in_v(False),
    "repeated_w_in_v_long": lambda: repeated_w_in_v(True),
    "repeated_x_in_u_by_v": repeated_x_in_u,
    "self_loops": lambda: self_loops(1),
    "self_loops_x3": lambda: self_loops(3),
    "self_loops_only": lambda: self_loops(1, with_clique=False),
    "empty_rows": empty_rows,
    "star_last_row": star_last_row,
    "all_in_last_row": all_in_last_row,
    "single_vertex": single_vertex,
    "straddle": straddle,
    "boundary_drops": holes,
    "inversion_last_row": lambda: swap_in_row(rows_of(holes()), 12, 0),
    "inversion_row_of_2": lambda: swap_in_row(rows_of(holes()), 6, 0),
    "shuffled_rows": shuffled_rows,
    "descending_rows": descending_rows,
    "rmat8_unsorted": lambda: rmat_unsorted(8),
    "rmat10_unsorted": lambda: rmat_unsorted(10),
}
