"""One JACOBI PageRank sweep from a source vector of integers, restated exactly in numpy (shared by
test_gpu_pr_sweep_values.py and test_pr_sweep_values_model.py).

The vectors hold random integers in [0, K], K = floor((2^24 - 1) / max in-degree): every partial sum of a row is
an integer below 2^24, so every f32 / f64 summation order the sweep kernels use gives the same exact row sum S,
and the update of pr_update (pagerank.cu) can be restated with one rounding per operation.  Neighbouring
vertices of the internal order then hold different values, so a gather from the wrong source changes the bytes
of its row (the start vector init / outdeg gives tied vertices the same value and hides such a gather).  Every
source that no row of the shard gathers holds a quiet NaN whose payload names it: a sweep that reads one writes a
NaN."""
from __future__ import annotations

import numpy as np

import pr_path_fixtures as fx

lm = fx.lm

DAMPING = np.float32(0.85)
EXACT = (1 << 24) - 1
SENTINEL = np.uint32(0xFFC0DEAD)   # a negative quiet NaN: the bits of every entry a sweep must not write
NAN_BASE = 0x7FC00000              # quiet NaN; payload 1 + source % (2^22 - 1)


def nan_of(sources):
    return (NAN_BASE | (1 + np.asarray(sources, np.int64) % 0x3FFFFF)).astype(np.uint32).view(np.float32)


def internal(plan, out, inc):
    """the in-CSR with rows and sources in the plan's internal order: the original row offsets, the internal
    source of every entry, and the internal row / in-degree / out-degree of every vertex"""
    n = plan["n"]
    new_id = plan["new_id"].astype(np.uint32)
    indeg = np.diff(inc[0].astype(np.int64))
    outdeg = np.diff(out[0].astype(np.int64))
    return dict(n=n, n_active=plan["n_active"], off=inc[0].astype(np.int64), src=new_id[inc[1]], new_id=new_id,
                indeg=indeg, indeg_int=indeg[plan["order"]], outdeg_int=outdeg[plan["order"]])


def owned(n, n_active, P=1, p=0):
    """rank p's rows (internal order) under the cyclic deal of 32-row slices: active rows only"""
    r = np.arange(n)
    return (r < n_active) & ((r >> 5) % P == p)


def gathered(ic, mine):
    """the internal sources that the rows in `mine` gather"""
    rows = np.repeat(ic["new_id"], ic["indeg"])          # internal row of every entry
    g = np.zeros(ic["n"], bool)
    g[ic["src"][mine[rows]]] = True
    return g


def vector(ic, used, seed):
    """integers in [0, K] on the gathered sources, a NaN naming the source on every other one"""
    rng = np.random.default_rng(seed)
    K = EXACT // max(1, int(ic["indeg"].max()))
    x = rng.integers(0, K + 1, ic["n"]).astype(np.float32)
    x[~used] = nan_of(np.flatnonzero(~used))
    return x


def row_sums(ic, x, src=None):
    """exact row sums S (int64, internal order) of x over the in-CSR, and the rows that read a NaN"""
    src = ic["src"] if src is None else src
    n, off, nz = ic["n"], ic["off"], ic["indeg"] > 0
    bad_x = np.isnan(x)
    xi = np.where(bad_x, 0, x).astype(np.int64)
    assert (xi == np.where(bad_x, 0, x)).all(), "the vector holds integers"
    S, bad = np.zeros(n, np.int64), np.zeros(n, bool)
    if len(src):
        S[ic["new_id"][nz]] = np.add.reduceat(xi[src], off[:-1][nz])
        bad[ic["new_id"][nz]] = np.add.reduceat(bad_x[src].astype(np.int64), off[:-1][nz]) > 0
    assert S.max(initial=0) <= EXACT, "every partial sum is exact in f32"
    return S, bad


def start(n, d=DAMPING):
    """PrStart: (init, base) in f32"""
    return np.float32(1.0) / np.float32(n), (np.float32(1.0) - d) / np.float32(n)


def expected(ic, x, src=None, d=DAMPING):
    """(scores, x_next) of every row (internal order; meaningful on the active rows): pr_update in f32, one
    rounding per operation: score = base + d * S, x_next = score / outdeg"""
    S, bad = row_sums(ic, x, src)
    _, base = start(ic["n"], d)
    score = base + d * S.astype(np.float32)
    score[bad] = np.float32(np.nan)
    with np.errstate(divide="ignore", invalid="ignore"):
        xn = score / ic["outdeg_int"].astype(np.float32)
    return score.astype(np.float32), xn.astype(np.float32)


def error_share(ic, score, old, mine, sweep_no, p, d=DAMPING):
    """the rank's error share: sum of |f32(score - old)| over its rows, plus on sweep 1 rank 0's closed form for
    the rows without in-edges (first_sweep_err)"""
    e = float(np.abs((score[mine] - old[mine]).astype(np.float32)).astype(np.float64).sum())
    if sweep_no == 1 and p == 0:
        init, base = start(ic["n"], d)
        e += float(ic["n"] - ic["n_active"]) * abs(float(np.float32(base - init)))
    return e


def fill_inactive(ic, d=DAMPING):
    """k_pr_fill_inactive: base / outdeg on the rows without in-edges (+inf for the dangling ones)"""
    _, base = start(ic["n"], d)
    with np.errstate(divide="ignore"):
        return (base / ic["outdeg_int"][ic["n_active"]:].astype(np.float32)).astype(np.float32)


# ---- wrong gathers, stated on the in-CSR ---------------------------------------------------------------------
def tie_neighbours(ic):
    """every source moved to its neighbour in the internal order with the same (in-degree, out-degree) key (the
    next vertex, else the previous one; a vertex with no tied neighbour keeps its entries)"""
    n = ic["n"]
    key = ic["indeg_int"] * (1 << 32) + ic["outdeg_int"]
    to = np.arange(n)
    nxt = np.r_[key[1:] == key[:-1], False]
    prv = np.r_[False, key[1:] == key[:-1]]
    to[prv] -= 1
    to[nxt] = np.flatnonzero(nxt) + 1
    return to.astype(np.uint32)[ic["src"]]


def shift_block(ic, B, j):
    """the sources of block j (internal ids [jB, jB + B)) read one id further: a block base off by one (the
    block's last id reads the next block's first, or the first of its own when it is the last block)"""
    src = ic["src"].astype(np.int64)
    hit = src // B == j
    src[hit] += 1
    src[hit & (src == ic["n"])] = j * B
    return src.astype(np.uint32)


def busiest_block(ic, B):
    return int(np.bincount(ic["src"] // B).argmax())
