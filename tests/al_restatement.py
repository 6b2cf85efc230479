"""A plain restatement of the reference's adjacency lists (crates/builder/src/graph/adj_list.rs): AdjacencyList::from
run by one thread, and add_edge one call at a time with apply_layout done literally.  Each row is a list of
(target, value) pairs; value is None for EV = ().  The device twins (graph_b200.DirectedALGraph / UndirectedALGraph)
are tested against it bit for bit."""
from __future__ import annotations

import bisect

import numpy as np

UNSORTED, SORTED, DEDUPLICATED = 0, 1, 2


class MissingNode(ValueError):
    """crate::Error::MissingNode (lib.rs:300): `node "3" does not exist in the graph`"""

    def __init__(self, node: int):
        super().__init__(f'node "{node}" does not exist in the graph')
        self.node = str(node)


def _finish(rows, layout):
    """The per-row layout of AdjacencyList::from (adj_list.rs:250-268): a stable sort keeps equal targets in push
    order, which is the order this library pins (the reference's sort_unstable leaves it open); dedup keeps the first
    of each run and, unlike the CSR build, every self-loop."""
    if layout == UNSORTED:
        return rows
    out = []
    for row in rows:
        row = sorted(row, key=lambda e: e[0])
        if layout == DEDUPLICATED:
            row = [e for i, e in enumerate(row) if i == 0 or row[i - 1][0] != e[0]]
        out.append(row)
    return out


def adjacency_list(src, dst, values, node_count, direction, layout):
    """AdjacencyList::from((&edges, node_count, direction, layout)) (adj_list.rs:216-277), one thread: direction
    "out", "in" or "undirected"; rows of (target, value) pairs."""
    rows = [[] for _ in range(node_count)]
    vals = [None] * len(src) if values is None else [np.float32(v) for v in values]
    for s, t, v in zip(src, dst, vals):
        if direction in ("out", "undirected"):
            rows[int(s)].append((int(t), v))
        if direction in ("in", "undirected"):
            rows[int(t)].append((int(s), v))
    return _finish(rows, layout)


class ALGraph:
    """DirectedALGraph (lists out and inc) or UndirectedALGraph (one list)."""

    def __init__(self, src, dst, values=None, node_count=0, layout=UNSORTED, directed=True):
        src = [int(x) for x in src]
        dst = [int(x) for x in dst]
        if node_count == 0:
            if not src:
                raise ValueError("cannot infer node_count from an empty edge list")
            node_count = max(max(src), max(dst)) + 1  # max_node_id + 1 (adj_list.rs:414)
        self.n, self.layout, self.directed = node_count, layout, directed
        self.with_values = values is not None
        if directed:  # adj_list.rs:412-425
            self.out = adjacency_list(src, dst, values, self.n, "out", layout)
            self.inc = adjacency_list(src, dst, values, self.n, "in", layout)
        else:  # adj_list.rs:565-574
            self.out = self.inc = adjacency_list(src, dst, values, self.n, "undirected", layout)

    # Graph / degrees / neighbours
    def node_count(self):
        return self.n

    def edge_count(self):
        total = sum(len(r) for r in self.out)
        return total if self.directed else total // 2  # adj_list.rs:484-486

    def _check_bounds(self, node):  # adj_list.rs:71-78
        if node >= self.n:
            raise MissingNode(node)

    @staticmethod
    def _apply_layout(layout, row, target):  # adj_list.rs:81-94
        keys = [e[0] for e in row]
        if layout == UNSORTED:
            row.append(target)
        elif layout == SORTED:
            # binary_search leaves the place among equal targets open; the new entry goes after them
            row.insert(bisect.bisect_right(keys, target[0]), target)
        else:
            i = bisect.bisect_left(keys, target[0])
            if not (i < len(keys) and keys[i] == target[0]):
                row.insert(i, target)

    def add_edge(self, source, target, value=None):
        """add_edge_with_value (adj_list.rs:381-389 directed, :534-542 undirected)"""
        v = None if value is None else np.float32(value)
        self._check_bounds(source)
        self._check_bounds(target)
        self._apply_layout(self.layout, self.out[source], (target, v))
        self._apply_layout(self.layout, self.inc[target], (source, v))

    def add_edges(self, src, dst, values=None):
        """The batch contract: all or nothing, the first bad edge named (its source first)."""
        for k, (s, t) in enumerate(zip(src, dst)):
            for x in (s, t):
                if int(x) >= self.n:
                    raise MissingNode(int(x))
        for k, (s, t) in enumerate(zip(src, dst)):
            self.add_edge(int(s), int(t), None if values is None else values[k])

    # as arrays
    def rows(self, which="out"):
        return self.out if which == "out" else self.inc

    def csr(self, which="out"):
        """(offsets u32, targets u32, values f32 or None) of one list, compacted."""
        rows = self.rows(which)
        off = np.zeros(self.n + 1, np.uint32)
        off[1:] = np.cumsum([len(r) for r in rows], dtype=np.uint64).astype(np.uint32)
        tgt = np.array([e[0] for r in rows for e in r], np.uint32)
        val = np.array([e[1] for r in rows for e in r], np.float32) if self.with_values else None
        return off, tgt, val


def layout_entries(rows, tgt, val, n, layout):
    """Entries given in push order (rows, targets, values or None) as one list's CSR (offsets, targets, values).
    Pushing them one at a time through apply_layout, or building from them, gives these rows: Unsorted keeps push
    order within a row; Sorted orders by target, equal targets in push order (a new entry goes after the equal ones
    already there); Deduplicated keeps the first entry of each target.  test_al_cpu.py checks this against ALGraph."""
    rows = np.asarray(rows, np.int64)
    tgt = np.asarray(tgt, np.int64)
    seq = np.arange(len(rows))
    order = np.lexsort((seq, rows)) if layout == UNSORTED else np.lexsort((seq, tgt, rows))
    rows, tgt = rows[order], tgt[order]
    val = None if val is None else np.asarray(val, np.float32)[order]
    if layout == DEDUPLICATED and len(rows):
        keep = np.ones(len(rows), bool)
        keep[1:] = (rows[1:] != rows[:-1]) | (tgt[1:] != tgt[:-1])
        rows, tgt = rows[keep], tgt[keep]
        val = None if val is None else val[keep]
    off = np.zeros(n + 1, np.uint32)
    off[1:] = np.cumsum(np.bincount(rows, minlength=n)[:n], dtype=np.uint64).astype(np.uint32)
    return off, tgt.astype(np.uint32), val


class FastAL:
    """The same graph as ALGraph, held as one push-ordered entry stream per list, for graphs and batches too large
    for one-at-a-time inserts.  csr() lays the stream out with layout_entries."""

    def __init__(self, src, dst, values=None, node_count=0, layout=UNSORTED, directed=True):
        src = np.asarray(src, np.int64)
        dst = np.asarray(dst, np.int64)
        if node_count == 0:
            if not len(src):
                raise ValueError("cannot infer node_count from an empty edge list")
            node_count = int(max(src.max(), dst.max())) + 1
        self.n, self.layout, self.directed = node_count, layout, directed
        self.with_values = values is not None
        self.lists = {"out": ([], [], []), "in": ([], [], [])} if directed else {"out": ([], [], [])}
        self._push(src, dst, values)

    def _push(self, src, dst, values):
        w = np.zeros(len(src), np.float32) if values is None else np.asarray(values, np.float32)
        if self.directed:
            parts = {"out": (src, dst, w), "in": (dst, src, w)}
        else:  # edge k pushes (s, t) and then (t, s)
            r = np.empty(2 * len(src), np.int64)
            c = np.empty(2 * len(src), np.int64)
            r[0::2], r[1::2], c[0::2], c[1::2] = src, dst, dst, src
            parts = {"out": (r, c, np.repeat(w, 2))}
        for k, (r, c, v) in parts.items():
            # the stream is kept laid out: its order then stands for every earlier push
            off, tgt, val = self._layout(k, r, c, v)
            rows = np.repeat(np.arange(self.n), np.diff(off.astype(np.int64)))
            self.lists[k] = (rows, tgt.astype(np.int64), val)

    def _layout(self, k, r, c, v):
        rows, tgt, val = self.lists[k]
        return layout_entries(np.concatenate([np.asarray(rows, np.int64), r]),
                              np.concatenate([np.asarray(tgt, np.int64), c]),
                              np.concatenate([np.asarray(val, np.float32), v]), self.n, self.layout)

    def add_edges(self, src, dst, values=None):
        src = np.asarray(src, np.int64)
        dst = np.asarray(dst, np.int64)
        for k in range(len(src)):
            if src[k] >= self.n or dst[k] >= self.n:
                raise MissingNode(int(src[k] if src[k] >= self.n else dst[k]))
        self._push(src, dst, values)

    def edge_count(self):
        m = len(self.lists["out"][0])
        return m if self.directed else m // 2

    def csr(self, which="out"):
        rows, tgt, val = self.lists[which]
        off = np.zeros(self.n + 1, np.uint32)
        off[1:] = np.cumsum(np.bincount(rows, minlength=self.n)[:self.n], dtype=np.uint64).astype(np.uint32)
        return off, tgt.astype(np.uint32), (val.astype(np.float32) if self.with_values else None)
