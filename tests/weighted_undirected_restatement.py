"""A numpy restatement of the reference's undirected build with f32 edge values (csr.rs:124-221 with
Direction::Undirected, EV = f32), and the value order this library gives it, for the tests.

Edge (s, t, w) puts Target(t, w) in row s and Target(s, w) in row t; a self-loop puts u into row u twice.
    Unsorted      the single-thread order: the outgoing pass, then the incoming pass, each in edge-list order
    Sorted        each row ascending by target; equal targets keep their Unsorted order
    Deduplicated  Sorted, then the first entry of each run of equal targets, and no self-loops (csr.rs:897-948)

`build` is the vectorised form the GPU tests compare with at size; `build_rows` is the same rule written row by
row, the way the reference fills its rows, and the CPU tests hold the two equal.
"""
import numpy as np

UNSORTED, SORTED, DEDUPLICATED = 0, 1, 2


def build(src, dst, w, n, layout):
    """(offsets u32[n + 1], targets u32[2m or fewer], values f32) of the undirected CSR."""
    src = np.asarray(src, np.uint32)
    dst = np.asarray(dst, np.uint32)
    w = np.asarray(w, np.float32)
    assert len(src) == len(dst) == len(w)
    rows = np.concatenate([src, dst])
    cols = np.concatenate([dst, src])
    vals = np.concatenate([w, w])
    if layout == UNSORTED:
        order = np.argsort(rows, kind="stable")
    else:
        order = np.lexsort((cols, rows))  # stable: equal (row, target) keys stay in Unsorted order
    rows, cols, vals = rows[order], cols[order], vals[order]
    if layout == DEDUPLICATED:
        first = np.ones(len(rows), bool)
        first[1:] = (rows[1:] != rows[:-1]) | (cols[1:] != cols[:-1])
        keep = first & (rows != cols)
        rows, cols, vals = rows[keep], cols[keep], vals[keep]
    off = np.zeros(n + 1, np.uint64)
    np.cumsum(np.bincount(rows, minlength=n)[:n], out=off[1:])
    return off.astype(np.uint32), cols.astype(np.uint32), vals.astype(np.float32)


def build_rows(src, dst, w, n, layout):
    """build() written as the reference fills rows: one list per row, appended to in the two passes."""
    rows = [[] for _ in range(n)]
    for s, t, x in zip(src, dst, np.asarray(w, np.float32)):
        rows[int(s)].append((int(t), x))
    for s, t, x in zip(src, dst, np.asarray(w, np.float32)):
        rows[int(t)].append((int(s), x))
    if layout != UNSORTED:
        rows = [sorted(r, key=lambda e: e[0]) for r in rows]  # sorted() is stable
    if layout == DEDUPLICATED:
        out = []
        for u, r in enumerate(rows):
            kept = []
            for t, x in r:
                if t != u and (not kept or kept[-1][0] != t):
                    kept.append((t, x))
            out.append(kept)
        rows = out
    off = np.zeros(n + 1, np.uint32)
    off[1:] = np.cumsum([len(r) for r in rows])
    tgt = np.array([t for r in rows for t, _ in r], np.uint32)
    val = np.array([x for r in rows for _, x in r], np.float32)
    return off, tgt, val


def rows_of(off, tgt, val, node):
    """[(target, value)] of one row, for the pinned examples."""
    b, e = int(off[node]), int(off[node + 1])
    return [(int(t), float(x)) for t, x in zip(tgt[b:e], val[b:e])]


def csr_edges(off, tgt, w):
    """The entries of a weighted out-CSR as (src, dst, value) arrays in CSR order: what to_undirected feeds."""
    off = np.asarray(off, np.int64)
    src = np.repeat(np.arange(len(off) - 1, dtype=np.uint32), np.diff(off))
    return src, np.asarray(tgt, np.uint32), np.asarray(w, np.float32)
