"""A Python restatement of the reference's node-labelled graph support, written from its Rust source for the tests:
the DotGraph (.graph) reader and the three structures over a labelled undirected CSR.

    DotGraph::try_from(LineReader)      crates/builder/src/input/dotgraph.rs:136-203
    LabelStats::from_graph              dotgraph.rs:220-313
    NeighborLabelFrequencies            dotgraph.rs:367-427
    NodeLabelIndex::from_stats          dotgraph.rs:430-532

The reader is positional: it skips 2 bytes of every line unread, reads leading ASCII digits, skips exactly one
byte between numbers and stops after line 1 + N + M.  Where the reference panics or misreads, this restatement
raises ValueError with the message libgraph_b200 gives: a missing line, a number without digits, bytes after the
last number (a '\\r' included) and a number >= 2^32.
"""
from __future__ import annotations

import numpy as np

NO_DIGITS = "a number has no digits"
TRAILING = "bytes follow the last number"
WIDE = "a number does not fit 32 bits"


class DotGraph:
    """labels[N], src / dst[M] in file order, and what the reference's DotGraph also keeps: the declared
    max_degree (the file's degree column), max_label and the label_frequency map."""

    def __init__(self, labels, src, dst, max_degree):
        self.labels = np.asarray(labels, np.uint32)
        self.src = np.asarray(src, np.uint32)
        self.dst = np.asarray(dst, np.uint32)
        self.max_degree = max_degree
        values, counts = np.unique(self.labels, return_counts=True)
        self.label_frequency = dict(zip(values.tolist(), counts.tolist()))
        self.max_label = int(values[-1]) if len(values) else 0

    def label_count(self) -> int:
        """DotGraph::label_count (dotgraph.rs:108-110): max_label + 1, not the number of distinct labels."""
        return self.max_label + 1

    def max_label_frequency(self) -> int:
        return max(self.label_frequency.values(), default=0)


def _numbers(line: bytes, count: int, lineno: int):
    p, out = 2, []
    for k in range(count):
        if k:
            p += 1
        q = p
        while q < len(line) and 48 <= line[q] <= 57:
            q += 1
        if q == p:
            raise ValueError(f"DotGraph line {lineno}: {NO_DIGITS}")
        digits = line[p:q].lstrip(b"0") or b"0"  # leading zeros are allowed, however many
        if len(digits) > 10 or int(digits) > 0xFFFFFFFF:
            raise ValueError(f"DotGraph line {lineno}: {WIDE}")
        out.append(int(digits))
        p = q
    if p != len(line):
        raise ValueError(f"DotGraph line {lineno}: {TRAILING}")
    return out


def read(data: bytes) -> DotGraph:
    lines = data.split(b"\n")
    if lines and lines[-1] == b"":
        lines.pop()  # the bytes after the last '\n' are a line only when there are some
    if not lines:
        raise ValueError('DotGraph file is empty: the header line "t N M" is missing')
    n, m = _numbers(lines[0], 2, 1)
    if len(lines) < 1 + n + m:
        bad = next((i for i, ln in enumerate(lines[1:], 1) if _bad(ln, 3 if i <= n else 2, i + 1)), None)
        if bad is None:
            raise ValueError(f"DotGraph file ends after {len(lines)} lines; its header declares 1 + {n} node + "
                             f"{m} edge lines")
    labels, max_degree = [], 0
    for i in range(1, n + 1):
        _, label, degree = _numbers(lines[i], 3, i + 1)
        labels.append(label)
        max_degree = max(max_degree, degree)
    src, dst = [], []
    for i in range(n + 1, n + m + 1):
        s, d = _numbers(lines[i], 2, i + 1)
        src.append(s)
        dst.append(d)
    return DotGraph(labels, src, dst, max_degree)


def _bad(line: bytes, count: int, lineno: int) -> bool:
    _numbers(line, count, lineno)  # raises the line's error, which comes before the missing lines
    return False


def write(labels, edges, degrees=None, tag: bytes = b"v") -> bytes:
    """A well-formed .graph file; degrees default to 0 (the reader keeps only their maximum)."""
    labels = list(map(int, labels))
    degrees = [0] * len(labels) if degrees is None else list(map(int, degrees))
    out = [b"t %d %d\n" % (len(labels), len(edges))]
    out += [tag + b" %d %d %d\n" % (i, l, d) for i, (l, d) in enumerate(zip(labels, degrees))]
    out += [b"e %d %d\n" % (int(s), int(t)) for s, t in edges]
    return b"".join(out)


def label_stats(off, tgt, labels):
    """LabelStats: max_degree is the largest CSR degree, label_count the number of distinct labels."""
    off = np.asarray(off, np.int64)
    values, counts = np.unique(np.asarray(labels, np.uint32), return_counts=True)
    return {"max_degree": int(np.diff(off).max()) if len(off) > 1 else 0, "label_count": len(values),
            "max_label": int(values[-1]), "max_label_frequency": int(counts.max()),
            "label_frequency": dict(zip(values.tolist(), counts.tolist()))}


def node_label_index(labels):
    """(offsets[max_label + 2], nodes[n]): row l holds the nodes labelled l, ascending."""
    labels = np.asarray(labels, np.uint32)
    nodes = np.argsort(labels, kind="stable").astype(np.uint32)
    offsets = np.zeros(int(labels.max()) + 2, np.uint32)
    np.cumsum(np.bincount(labels, minlength=int(labels.max()) + 1), out=offsets[1:])
    return offsets, nodes


def neighbor_label_frequencies(off, tgt, labels):
    """The pair CSR (offsets[n + 1], labels, counts): node u's labels ascending, each with its count in u's row."""
    off = np.asarray(off, np.int64)
    n = len(off) - 1
    rows = np.repeat(np.arange(n, dtype=np.uint64), np.diff(off))
    keys = rows << np.uint64(32) | np.asarray(labels, np.uint32)[np.asarray(tgt, np.int64)].astype(np.uint64)
    uniq, counts = np.unique(keys, return_counts=True)
    pair_rows = (uniq >> np.uint64(32)).astype(np.int64)
    offsets = np.zeros(n + 1, np.uint32)
    np.cumsum(np.bincount(pair_rows, minlength=n), out=offsets[1:])
    return offsets, (uniq & np.uint64(0xFFFFFFFF)).astype(np.uint32), counts.astype(np.uint32)


def frequency_maps(offsets, labels, counts):
    """The pair CSR as the reference's Vec<FxHashMap<Label, usize>>."""
    return [dict(zip(labels[offsets[u]:offsets[u + 1]].tolist(), counts[offsets[u]:offsets[u + 1]].tolist()))
            for u in range(len(offsets) - 1)]


# A well-formed file, and malformed ones with the message both readers of the library give
GOOD = b"t 2 1\nv 0 4 1\nv 1 6 1\ne 0 1\n"
MALFORMED = [
    (b"", 'DotGraph file is empty: the header line "t N M" is missing'),
    (b"t 2 1\nv 0 4 1\nv 1 6 1\n", "DotGraph file ends after 3 lines; its header declares 1 + 2 node + 1 edge lines"),
    (b"t 2 1\nv 0 4 1\n", "DotGraph file ends after 2 lines; its header declares 1 + 2 node + 1 edge lines"),
    (b"t 2 1\nv 0 x 1\nv 1 6 1\ne 0 1\n", "DotGraph line 2: a number has no digits"),
    (b"t 2 1\nv 0 4 1\n\ne 0 1\n", "DotGraph line 3: a number has no digits"),
    (b"t 2 1\nv 0 4 1\nv 1 6\ne 0 1\n", "DotGraph line 3: a number has no digits"),
    (b"t 2 1\nv 0 4 1\r\nv 1 6 1\ne 0 1\n", "DotGraph line 2: bytes follow the last number"),
    (b"t 2 1\nv 0 4 1\nv 1 6 1\ne 0 1 \n", "DotGraph line 4: bytes follow the last number"),
    (b"t 2 1\nv 0 4294967296 1\nv 1 6 1\ne 0 1\n", "DotGraph line 2: a number does not fit 32 bits"),
    (b"t 2 1\nv 0 4 1\nv 1 6 1\ne 0 99999999999\n", "DotGraph line 4: a number does not fit 32 bits"),
    (b"t 4294967296 1\n", "DotGraph line 1: a number does not fit 32 bits"),
    (b"t 2 1\r\nv 0 4 1\nv 1 6 1\ne 0 1\n", "DotGraph line 1: bytes follow the last number"),
    (b"t 2\n", "DotGraph line 1: a number has no digits"),
    # a bad line before the end of the file is reported before the missing lines
    (b"t 3 1\nv 0 4 1\nv 1 6 1x\n", "DotGraph line 3: bytes follow the last number"),
    # headers that declare more lines than the file could hold: nothing is sized by N and M, the error is the same
    (b"t 4294967295 4294967295\n",
     "DotGraph file ends after 1 lines; its header declares 1 + 4294967295 node + 4294967295 edge lines"),
    (b"t 1000 0\nv 0 1 1\nv 1 2x 1\n", "DotGraph line 3: a number has no digits"),
    # header lines longer than a first read of the file
    (b"t 2 1" + b" " * 5000 + b"\nv 0 4 1\nv 1 6 1\ne 0 1\n", "DotGraph line 1: bytes follow the last number"),
    (b"t " + b"0" * 6000 + b"2 1\nv 0 4 1\nv 1 6\n", "DotGraph line 3: a number has no digits"),
]
