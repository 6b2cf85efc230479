"""Adjacency-list graphs on the device (graph_b200.DirectedALGraph / UndirectedALGraph): every constructor and
sequences of add_edges batches against the restatement (tests/al_restatement.py), bit for bit: offsets, targets and
value bits.  Then the snapshot (to_graph) against the CSR twin of the restatement's rows, the rejected batches, and
several threads on one handle."""
import threading

import numpy as np
import pytest

import al_restatement as ar
import graph_b200 as gb
import oracle

pytestmark = pytest.mark.gpu

LAYOUTS = [(gb.Layout.Unsorted, ar.UNSORTED), (gb.Layout.Sorted, ar.SORTED),
           (gb.Layout.Deduplicated, ar.DEDUPLICATED)]
LAYOUT_IDS = ["Unsorted", "Sorted", "Deduplicated"]


def _cls(directed):
    return gb.DirectedALGraph if directed else gb.UndirectedALGraph


def _same(g, ref, directed):
    """Every list of g equals the restatement's, and so does edge_count."""
    assert g.edge_count() == ref.edge_count()
    assert g.node_count() == ref.n
    for which in (("out", "in") if directed else ("out",)):
        want = ref.csr(which)
        got = g.csr(which, with_values=ref.with_values) if directed else g.csr(with_values=ref.with_values)
        assert got[0].tobytes() == want[0].tobytes(), f"{which} offsets differ"
        assert got[1].tobytes() == want[1].tobytes(), f"{which} targets differ"
        if ref.with_values:
            assert got[2].view(np.uint32).tobytes() == want[2].view(np.uint32).tobytes(), f"{which} values differ"


def _edges(seed, n, m):
    """Random edges with self-loops and duplicates; node n - 1 and a few others stay isolated when n is larger."""
    rng = np.random.default_rng(seed)
    src = rng.integers(0, n, m, dtype=np.uint32)
    dst = rng.integers(0, n, m, dtype=np.uint32)
    dst[::9] = src[::9]
    src[1::5], dst[1::5] = src[::5][:len(src[1::5])], dst[::5][:len(dst[1::5])]
    w = (rng.integers(-1000, 1000, m) / 8).astype(np.float32)
    return src, dst, w


@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
@pytest.mark.parametrize("directed", [True, False], ids=["directed", "undirected"])
@pytest.mark.parametrize("values", [False, True], ids=["plain", "values"])
def test_constructors(layout, directed, values):
    import torch
    lay, rl = layout
    cls = _cls(directed)
    src, dst, w = _edges(3, 300, 4000)
    ww = w if values else None
    for node_count in (0, 420):  # 420: isolated nodes past the largest id
        ref = ar.FastAL(src, dst, ww, node_count, rl, directed)
        _same(cls.from_numpy(np.stack([src, dst], 1), layout=lay, weights=ww, node_count=node_count), ref, directed)
        t = [torch.from_numpy(a.astype(np.int64)).cuda() for a in (src, dst)]
        tw = torch.from_numpy(w).cuda() if values else None
        _same(cls.from_torch(t[0], t[1], weights=tw, node_count=node_count, layout=lay), ref, directed)
    # an empty edge list with an explicit node count
    empty = cls.from_numpy(np.zeros((0, 2), np.uint32), layout=lay, weights=np.zeros(0, np.float32) if values else None,
                           node_count=5)
    assert (empty.node_count(), empty.edge_count()) == (5, 0)
    _same(empty, ar.FastAL([], [], np.zeros(0) if values else None, 5, rl, directed), directed)
    with pytest.raises(ValueError, match="empty edge list"):
        cls.from_numpy(np.zeros((0, 2), np.uint32), layout=lay)


@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
@pytest.mark.parametrize("directed", [True, False], ids=["directed", "undirected"])
def test_file_loads(layout, directed, golden_dir):
    lay, rl = layout
    cls = _cls(directed)
    for name in ("example.el", "test.el"):
        s, d = gb._read_edge_list(golden_dir / name)
        _same(cls.load(golden_dir / name, layout=lay, file_format=gb.FileFormat.EdgeList),
              ar.FastAL(s, d, None, 0, rl, directed), directed)
    for name in ("example.wel", "test.wel"):
        s, d, w = gb._read_edge_list(golden_dir / name, with_values=True)
        _same(cls.load_weighted(golden_dir / name, layout=lay), ar.FastAL(s, d, w, 0, rl, directed), directed)
    s, d, n = gb._read_graph500(golden_dir / "scale_8.graph500")
    g = cls.load(golden_dir / "scale_8.graph500", layout=lay)
    assert g.node_count() == n == len(s) // 16
    assert g.load_info()["edges"] == len(s)
    _same(g, ar.FastAL(s, d, None, n, rl, directed), directed)


def _rmat12():
    src, dst = oracle.rmat_edges(12, seed=42)
    return src.astype(np.uint32), dst.astype(np.uint32)


def _batches(n, seed):
    """batches of 0, 1, 1000 and 10^5 edges with duplicates inside and against existing rows, and self-loops"""
    rng = np.random.default_rng(seed)
    src0, dst0 = _rmat12()
    out = []
    for size in (0, 1, 1000, 100_000):
        s = rng.integers(0, n, size, dtype=np.uint32)
        d = rng.integers(0, n, size, dtype=np.uint32)
        if size >= 1000:
            k = size // 10
            pick = rng.integers(0, len(src0), k)
            s[:k], d[:k] = src0[pick], dst0[pick]      # edges the graph has
            s[k:2 * k], d[k:2 * k] = s[:k][::-1], d[:k][::-1]  # repeated in the batch
            d[2 * k:3 * k] = s[2 * k:3 * k]            # self-loops
        out.append((s, d, (rng.integers(0, 1 << 20, size) / 1024).astype(np.float32)))
    return out


@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
@pytest.mark.parametrize("directed", [True, False], ids=["directed", "undirected"])
@pytest.mark.parametrize("values", [False, True], ids=["plain", "values"])
def test_batches_on_rmat12(layout, directed, values):
    lay, rl = layout
    src, dst = _rmat12()
    n = 1 << 12
    w = (np.arange(len(src)) % 977).astype(np.float32) if values else None
    g = _cls(directed).from_numpy(np.stack([src, dst], 1), layout=lay, weights=w, node_count=n)
    ref = ar.FastAL(src, dst, w, n, rl, directed)
    _same(g, ref, directed)
    for s, d, bw in _batches(n, 11):
        g.add_edges(s, d, bw if values else None)
        ref.add_edges(s, d, bw if values else None)
        _same(g, ref, directed)
        info = g.last_batch()
        assert info["edges"] == len(s)
    # a star hub receiving 10^5 edges in one batch: it moves to the tail, past the first pool's free tail
    hub = np.full(100_000, 7, np.uint32)
    leaves = np.random.default_rng(5).integers(0, n, 100_000, dtype=np.uint32)
    hw = np.arange(100_000, dtype=np.float32) if values else None
    g.add_edges(hub, leaves, hw)
    ref.add_edges(hub, leaves, hw)
    _same(g, ref, directed)
    assert g.last_batch()["relocated_rows"] >= 1
    snap = g.to_graph()
    want = ref.csr("out")
    got = snap.csr()[0:2] if not directed else snap.csr("out")
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()


@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
@pytest.mark.parametrize("directed", [True, False], ids=["directed", "undirected"])
def test_compaction_and_growth(layout, directed):
    """Many batches into few rows: the pool is rebuilt compacted at least once, and every row stays right."""
    lay, rl = layout
    src, dst = _rmat12()
    n = 1 << 12
    g = _cls(directed).from_numpy(np.stack([src, dst], 1), layout=lay, node_count=n)
    ref = ar.FastAL(src, dst, None, n, rl, directed)
    rng = np.random.default_rng(9)
    for i in range(24):
        rows = rng.integers(0, 64, 20_000, dtype=np.uint32)  # hubs and tail rows grow by doubling
        tgt = rng.integers(0, n, 20_000, dtype=np.uint32)
        g.add_edges(rows, tgt)
        ref.add_edges(rows, tgt)
        if i % 6 == 5:
            _same(g, ref, directed)
    _same(g, ref, directed)
    assert g.last_batch()["total_compactions"] >= 1


@pytest.mark.parametrize("directed", [True, False], ids=["directed", "undirected"])
def test_sorted_rows_whose_middle_shifts(directed):
    for lay, rl in LAYOUTS[1:]:
        src = np.array([0, 0, 0, 0, 1], np.uint32)
        dst = np.array([10, 20, 30, 40, 20], np.uint32)
        w = np.array([1, 2, 3, 4, 5], np.float32)
        g = _cls(directed).from_numpy(np.stack([src, dst], 1), layout=lay, weights=w, node_count=64)
        ref = ar.ALGraph(src, dst, w, 64, rl, directed)
        bs = np.array([0, 0, 0, 0, 0], np.uint32)
        bd = np.array([25, 20, 15, 25, 45], np.uint32)
        bw = np.array([6, 7, 8, 9, 10], np.float32)
        g.add_edges(bs, bd, bw)
        ref.add_edges(bs, bd, bw)
        _same(g, ref, directed)
        t, v = g.out_neighbors_with_values(0) if directed else g.neighbors_with_values(0)
        assert t.tolist() == [x for x, _ in ref.out[0]]
        assert v.tolist() == [float(y) for _, y in ref.out[0]]


@pytest.mark.parametrize("directed", [True, False], ids=["directed", "undirected"])
def test_reference_add_edge_cases(directed):
    cls = _cls(directed)
    g = cls.from_numpy(np.array([[0, 2], [1, 2]]), layout=gb.Layout.Unsorted)
    row = g.out_neighbors if directed else g.neighbors
    g.add_edge(0, 1)
    assert row(0).tolist() == [2, 1]
    g.add_edge(0, 2)
    assert row(0).tolist() == [2, 1, 2]
    with pytest.raises(ValueError, match='node "3" does not exist in the graph'):
        g.add_edge(0, 3)
    with pytest.raises(ValueError, match='node "5" does not exist in the graph'):
        g.add_edge(5, 3)
    g = cls.from_numpy(np.array([[0, 2], [1, 2], [1, 3]]), layout=gb.Layout.Deduplicated)
    row = g.out_neighbors if directed else g.neighbors
    g.add_edge(0, 1)
    g.add_edge(0, 1)
    g.add_edge(0, 3)
    assert row(0).tolist() == [1, 2, 3]
    w = cls.from_numpy(np.array([[0, 2], [1, 2]]), weights=[4.2, 13.37])
    w.add_edge(0, 1, 19.84)
    t, v = w.out_neighbors_with_values(0) if directed else w.neighbors_with_values(0)
    assert t.tolist() == [2, 1] and v.tobytes() == np.array([4.2, 19.84], np.float32).tobytes()
    if directed:  # the crate doc-test (lib.rs:234-255)
        d = cls.from_numpy(np.array([[0, 1], [0, 2], [1, 2], [1, 3], [2, 3]]))
        assert (d.node_count(), d.edge_count(), d.out_degree(1), d.in_degree(1)) == (4, 5, 2, 1)
        d.add_edge(1, 0)
        assert d.edge_count() == 6 and d.out_neighbors(1).tolist() == [2, 3, 0]


@pytest.mark.parametrize("directed", [True, False], ids=["directed", "undirected"])
def test_rejected_batches_change_nothing(directed):
    src, dst = _rmat12()
    n = 1 << 12
    g = _cls(directed).from_numpy(np.stack([src, dst], 1), layout=gb.Layout.Sorted, node_count=n)
    ref = ar.FastAL(src, dst, None, n, ar.SORTED, directed)
    cases = [([1, n + 3, 2, 5], [2, 4, n + 9, 5], n + 3),   # a missing source first
             ([1, 2, n + 7], [2, n + 1, 3], n + 1),          # a missing target first
             ([1, n + 2], [2, n + 8], n + 2)]                # both: the source is named
    for s, d, missing in cases:
        with pytest.raises(ValueError, match=f'node "{missing}" does not exist in the graph'):
            g.add_edges(np.array(s, np.uint32), np.array(d, np.uint32))
        _same(g, ref, directed)


def test_entry_count_overflow_is_refused_before_any_allocation():
    g = gb.UndirectedALGraph.from_numpy(np.array([[0, 1]]), layout=gb.Layout.Unsorted)
    before = g.device_bytes()
    big = np.zeros(1 << 31, np.uint32)  # zero pages, never touched: 2^31 edges make 2^32 undirected entries
    with pytest.raises(ValueError, match="fewer than 2\\^32 - 1"):
        g.add_edges(big, big)
    assert g.edge_count() == 1 and g.device_bytes() == before
    assert g.last_batch()["edges"] == 0  # no batch ran


def _same_results(snap, twin, directed, weighted):
    if directed:
        a = snap.page_rank(max_iterations=10, tolerance=0.0, mode="exact")
        b = twin.page_rank(max_iterations=10, tolerance=0.0, mode="exact")
        assert a.scores().tobytes() == b.scores().tobytes() and a.ran_iterations == b.ran_iterations
        assert (snap.wcc().components() == twin.wcc().components()).all()
        if weighted:
            x = snap.delta_stepping(start_node=0, delta=0.5).distances()
            y = twin.delta_stepping(start_node=0, delta=0.5).distances()
            assert x.tobytes() == y.tobytes()
    else:
        assert snap.global_triangle_count().triangles == twin.global_triangle_count().triangles


@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
@pytest.mark.parametrize("directed", [True, False], ids=["directed", "undirected"])
def test_snapshot_algorithms(layout, directed):
    lay, rl = layout
    src, dst = _rmat12()
    n = 1 << 12
    w = (np.random.default_rng(2).random(len(src)) + 0.01).astype(np.float32) if directed else None
    g = _cls(directed).from_numpy(np.stack([src, dst], 1), layout=lay, weights=w, node_count=n)
    ref = ar.FastAL(src, dst, w, n, rl, directed)
    s, d, bw = _batches(n, 3)[2]
    g.add_edges(s, d, np.abs(bw) + 0.01 if directed else None)
    ref.add_edges(s, d, np.abs(bw) + 0.01 if directed else None)
    snap = g.to_graph()
    if directed:
        oo, ot, ov = ref.csr("out")
        io, it, _ = ref.csr("in")
        twin = gb.DiGraph.from_csr(oo, ot, io, it, out_weights=ov)
        assert [a.tobytes() for a in snap.csr("out")] == [oo.tobytes(), ot.tobytes()]
        assert [a.tobytes() for a in snap.csr("in")] == [io.tobytes(), it.tobytes()]
        assert snap.out_weights().tobytes() == ov.tobytes()
    else:
        off, tgt, _ = ref.csr("out")
        twin = gb.Graph.from_csr(off, tgt)
        assert [a.tobytes() for a in snap.csr()] == [off.tobytes(), tgt.tobytes()]
    _same_results(snap, twin, directed, True)
    # the cached snapshot of the algorithm methods follows add_edges
    if directed:
        assert g.wcc().components().tobytes() == twin.wcc().components().tobytes()
        g.add_edge(0, 1, 1.0)
        assert g.edge_count() == snap.edge_count() + 1
        assert g.page_rank(max_iterations=3, tolerance=0.0).ran_iterations == 3
    else:
        assert g.global_triangle_count().triangles == twin.global_triangle_count().triangles


def test_triangle_count_with_self_loops_matches_the_oracle():
    src, dst = _rmat12()
    src = np.concatenate([src, np.arange(0, 4096, 7, dtype=np.uint32)])
    dst = np.concatenate([dst, np.arange(0, 4096, 7, dtype=np.uint32)])
    g = gb.UndirectedALGraph.from_numpy(np.stack([src, dst], 1), layout=gb.Layout.Deduplicated, node_count=4096)
    off, tgt, _ = ar.FastAL(src, dst, None, 4096, ar.DEDUPLICATED, False).csr()
    assert ((tgt == np.repeat(np.arange(4096), np.diff(off.astype(np.int64)))).sum()) > 0  # self-loops kept
    assert g.global_triangle_count().triangles == oracle.triangle_count(off, tgt, threads=0)


def test_threads_on_one_handle():
    # directed_al_graph_add_edge_parallel (adj_list.rs:894-908)
    g = gb.DirectedALGraph.from_numpy(np.array([[0, 1], [0, 2], [0, 3]]), layout=gb.Layout.Unsorted)
    ts = [threading.Thread(target=g.add_edge, args=(0, 1)) for _ in range(4)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert g.edge_count() == 7 and sorted(g.out_neighbors(0).tolist()) == [1, 1, 1, 1, 1, 2, 3]
    # disjoint batches on a Sorted graph end at the restatement of all edges, whatever the order they ran in
    src, dst = _rmat12()
    n = 1 << 12
    g = gb.UndirectedALGraph.from_numpy(np.stack([src, dst], 1), layout=gb.Layout.Sorted, node_count=n)
    rng = np.random.default_rng(4)
    parts = [(rng.integers(0, n, 5000, dtype=np.uint32), rng.integers(0, n, 5000, dtype=np.uint32)) for _ in range(4)]
    ts = [threading.Thread(target=g.add_edges, args=p) for p in parts]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    ref = ar.FastAL(np.concatenate([src] + [p[0] for p in parts]), np.concatenate([dst] + [p[1] for p in parts]),
                    None, n, ar.SORTED, False)
    _same(g, ref, False)


def test_algorithms_in_a_row_reuse_the_snapshot():
    src, dst = _rmat12()
    n = 1 << 12
    d = gb.DirectedALGraph.from_numpy(np.stack([src, dst], 1), layout=gb.Layout.Sorted, node_count=n)
    first = d.wcc().components()
    assert d.page_rank(max_iterations=3, tolerance=0.0).ran_iterations == 3
    assert d.wcc().components().tobytes() == first.tobytes()
    u = gb.UndirectedALGraph.from_numpy(np.stack([src, dst], 1), layout=gb.Layout.Sorted, node_count=n)
    t = u.global_triangle_count().triangles
    assert u.global_triangle_count().triangles == t


@pytest.mark.parametrize("directed", [True, False], ids=["directed", "undirected"])
def test_concurrent_readers_and_writers(directed):
    """Readers copy whole lists and rows while writers add batches: every copy is one state of the graph, between
    the first and the last, and the arrays it lands in are never overrun."""
    src, dst = _rmat12()
    n = 1 << 12
    g = _cls(directed).from_numpy(np.stack([src, dst], 1), layout=gb.Layout.Sorted, node_count=n)
    m0 = len(src) * (1 if directed else 2)
    rng = np.random.default_rng(12)
    parts = [(rng.integers(0, n, 3000, dtype=np.uint32), rng.integers(0, n, 3000, dtype=np.uint32)) for _ in range(8)]
    seen, errors = [], []

    def write(p):
        try:
            g.add_edges(*p)
        except Exception as e:  # pragma: no cover - reported below
            errors.append(e)

    def read():
        try:
            for _ in range(6):
                off, tgt = g.csr("out") if directed else g.csr()
                assert len(tgt) == int(off[-1]) and (np.diff(off.astype(np.int64)) >= 0).all()
                seen.append(len(tgt))
                row = g.out_neighbors(7) if directed else g.neighbors(7)
                assert (np.diff(row.astype(np.int64)) >= 0).all()
        except Exception as e:  # pragma: no cover - reported below
            errors.append(e)

    ts = [threading.Thread(target=write, args=(p,)) for p in parts] + [threading.Thread(target=read) for _ in range(3)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors
    per_batch = 3000 * (1 if directed else 2)
    assert all(m0 <= k <= m0 + 8 * per_batch and (k - m0) % per_batch == 0 for k in seen)
    ref = ar.FastAL(np.concatenate([src] + [p[0] for p in parts]), np.concatenate([dst] + [p[1] for p in parts]),
                    None, n, ar.SORTED, directed)
    _same(g, ref, directed)
