"""Binary graph files on the device: DiGraph.load / Graph.load with FileFormat.Binary (host decoder below 64 MiB,
the streamed path of graph_b200/csrc/load.cu when GB_LOAD_CHUNK_BYTES is set) and serialize().  Files come from
the Python restatement of the reference's format (tests/binary_restatement.py); graphs are checked against the
oracle's CSRs and algorithm results must survive a round trip bit for bit."""
import numpy as np
import pytest

import binary_restatement as br
import graph_b200 as gb
import oracle

pytestmark = pytest.mark.gpu

LAYOUTS = {"Unsorted": gb.Layout.Unsorted, "Sorted": gb.Layout.Sorted, "Deduplicated": gb.Layout.Deduplicated}
KINDS = ["digraph", "weighted", "graph"]
CHUNKS = [None, 64, 4096, 1009]  # None: the host decoder; 1009 is prime, so records straddle chunks


def set_chunk(monkeypatch, chunk):
    if chunk is None:
        monkeypatch.delenv("GB_LOAD_CHUNK_BYTES", raising=False)
    else:
        monkeypatch.setenv("GB_LOAD_CHUNK_BYTES", str(chunk))


def oracle_csrs(src, dst, n, kind, layout, w=None):
    """[(off, tgt, values or None)] as the file holds them (values of a weighted digraph in both CSRs)."""
    lay = layout.value
    if kind == "graph":
        off, tgt = oracle.csr_build(src, dst, n, oracle.UNDIRECTED, lay)
        return [(off, tgt, None)]
    if kind == "weighted":
        oo, ot, ow = oracle.csr_build(src, dst, n, oracle.OUTGOING, lay, w)
        io, it = oracle.csr_build(src, dst, n, oracle.INCOMING, lay)
        return [(oo, ot, ow), (io, it, br.in_values(oo, ot, ow, io, it))]
    oo, ot = oracle.csr_build(src, dst, n, oracle.OUTGOING, lay)
    io, it = oracle.csr_build(src, dst, n, oracle.INCOMING, lay)
    return [(oo, ot, None), (io, it, None)]


def load(path, kind):
    if kind == "graph":
        return gb.Graph.load(path, file_format=gb.FileFormat.Binary)
    if kind == "weighted":
        return gb.DiGraph.load_weighted(path, file_format=gb.FileFormat.Binary)
    return gb.DiGraph.load(path, file_format=gb.FileFormat.Binary)


def graph_arrays(g):
    if isinstance(g, gb.Graph):
        return list(g.csr())
    out = list(g.csr("out")) + list(g.csr("in"))
    if g._info.has_weights:
        out.append(g.out_weights())
    return out


def assert_same(a, b):
    assert (a.node_count(), a.edge_count(), a._info.has_weights) == (b.node_count(), b.edge_count(), b._info.has_weights)
    for x, y in zip(graph_arrays(a), graph_arrays(b), strict=True):
        assert x.dtype == y.dtype and x.tobytes() == y.tobytes()


def assert_matches_csrs(g, csrs):
    arrays = graph_arrays(g)
    want = [a for off, tgt, _ in csrs for a in (off, tgt)]
    if isinstance(g, gb.DiGraph) and csrs[0][2] is not None:
        want.append(csrs[0][2])
    assert len(arrays) == len(want)
    for x, y in zip(arrays, want):
        assert x.tobytes() == np.asarray(y, x.dtype).tobytes()


@pytest.fixture(scope="module")
def edges(scale8_edges):
    src, dst, n = scale8_edges
    w = oracle.rmat_weights(7, 0, len(src))
    return src, dst, n, w


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_load_serialize_round_trip(tmp_path, monkeypatch, edges, layout, kind, chunk):
    src, dst, n, w = edges
    csrs = oracle_csrs(src, dst, n, kind, LAYOUTS[layout], w)
    data = br.write(csrs)
    path = tmp_path / "g.bin"
    path.write_bytes(data)
    set_chunk(monkeypatch, chunk)
    g = load(path, kind)
    assert_matches_csrs(g, csrs)
    info = g.load_info()
    assert info["file_bytes"] == len(data)
    assert info["edges"] == (len(csrs[0][1]) // 2 if kind == "graph" else len(csrs[0][1]))
    assert info["chunks"] == (0 if chunk is None else -(-len(data) // chunk))
    out = tmp_path / "out.bin"
    g.serialize(out)
    assert out.read_bytes() == data
    assert_same(load(out, kind), g)
    assert sorted(p.name for p in tmp_path.iterdir()) == ["g.bin", "out.bin"]  # no temporary file left


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("kind", KINDS)
def test_usize_files_narrow_to_the_u32_graph(tmp_path, monkeypatch, edges, kind, chunk):
    src, dst, n, w = edges
    csrs = oracle_csrs(src, dst, n, kind, gb.Layout.Sorted, w)
    (tmp_path / "a.bin").write_bytes(br.write(csrs, "u32"))
    (tmp_path / "b.bin").write_bytes(br.write(csrs, "usize"))
    (tmp_path / "c.bin").write_bytes(br.write(csrs, "u64"))
    set_chunk(monkeypatch, chunk)
    a = load(tmp_path / "a.bin", kind)
    assert_same(load(tmp_path / "b.bin", kind), a)
    assert_same(load(tmp_path / "c.bin", kind), a)


@pytest.mark.parametrize("chunk", [None, 1009])
def test_values_are_dropped_on_request(tmp_path, monkeypatch, edges, chunk):
    src, dst, n, w = edges
    csrs = oracle_csrs(src, dst, n, "weighted", gb.Layout.Sorted, w)
    (tmp_path / "w.bin").write_bytes(br.write(csrs))
    set_chunk(monkeypatch, chunk)
    g = gb.DiGraph.load(tmp_path / "w.bin", file_format=gb.FileFormat.Binary)
    assert not g._info.has_weights
    assert_matches_csrs(g, [(o, t, None) for o, t, _ in csrs])
    und = oracle_csrs(src, dst, n, "graph", gb.Layout.Sorted)
    (tmp_path / "u.bin").write_bytes(br.write([(und[0][0], und[0][1], np.ones(len(und[0][1]), np.float32))]))
    assert_matches_csrs(gb.Graph.load(tmp_path / "u.bin", file_format=gb.FileFormat.Binary), und)
    (tmp_path / "plain.bin").write_bytes(br.write([(o, t, None) for o, t, _ in csrs]))
    with pytest.raises(ValueError, match="no edge values"):
        gb.DiGraph.load_weighted(tmp_path / "plain.bin", file_format=gb.FileFormat.Binary)


def test_in_csr_values_follow_the_occurrence_rule(tmp_path):
    """Parallel edges with distinct values, in every layout; the values written for the in-CSR are the CPU
    restatement's, and a graph whose in-CSR is not the transpose of its out-CSR cannot be written."""
    edges = [(0, 1, 1.0), (0, 1, 2.0), (1, 0, 3.0), (0, 1, 4.0), (2, 1, 5.0), (1, 1, 6.0), (1, 1, 7.0), (2, 1, 8.0)]
    arr = np.array([e[:2] for e in edges], np.uint32)
    w = np.array([e[2] for e in edges], np.float32)
    for layout in LAYOUTS.values():
        g = gb.DiGraph.from_numpy(arr, layout=layout, weights=w)
        g.serialize(tmp_path / "p.bin")
        (oo, ot, ow), (io, it, iw) = br.read((tmp_path / "p.bin").read_bytes(), 2, True)
        assert iw.tobytes() == br.in_values(oo, ot, ow, io, it).tobytes(), layout
        assert ow.tobytes() == g.out_weights().tobytes()
    oo, ot = np.array([0, 1, 1], np.uint32), np.array([1], np.uint32)
    bad = gb.DiGraph.from_csr(oo, ot, np.array([0, 0, 1], np.uint32), np.array([1], np.uint32),
                              out_weights=np.ones(1, np.float32))
    with pytest.raises(ValueError, match="not the transpose"):
        bad.serialize(tmp_path / "bad.bin")
    assert not (tmp_path / "bad.bin").exists()
    assert list(tmp_path.iterdir()) == [tmp_path / "p.bin"]


def test_page_rank_twin_cannot_be_serialized(tmp_path):
    off = np.array([0, 1, 2], np.uint32)
    g = gb.DiGraph.for_page_rank(off, np.array([1, 0], np.uint32), off)
    with pytest.raises(ValueError, match="page-rank-only"):
        g.serialize(tmp_path / "x.bin")


@pytest.mark.parametrize("chunk", [None, 64])
def test_results_survive_a_round_trip(tmp_path, monkeypatch, edges, chunk):
    src, dst, n, w = edges
    set_chunk(monkeypatch, chunk)
    pairs = np.stack([src, dst], axis=1)
    for layout in LAYOUTS.values():
        g = gb.DiGraph.from_numpy(pairs, layout=layout, weights=w)
        g.serialize(tmp_path / "d.bin")
        h = gb.DiGraph.load_weighted(tmp_path / "d.bin", file_format=gb.FileFormat.Binary)
        a = g.page_rank(max_iterations=10, tolerance=0.0, mode="exact").scores()
        b = h.page_rank(max_iterations=10, tolerance=0.0, mode="exact").scores()
        assert a.tobytes() == b.tobytes()
        assert (g.wcc().components() == h.wcc().components()).all()
        assert g.delta_stepping(start_node=0, delta=0.5).distances().tobytes() == \
            h.delta_stepping(start_node=0, delta=0.5).distances().tobytes()
        u = gb.Graph.from_numpy(pairs, layout=layout)
        u.serialize(tmp_path / "u.bin")
        v = gb.Graph.load(tmp_path / "u.bin", file_format=gb.FileFormat.Binary)
        assert u.global_triangle_count().triangles == v.global_triangle_count().triangles
    # an Unsorted graph whose rows descend: the reloaded rows are unknown-order and TC takes the list-order path
    desc = gb.Graph.from_numpy(pairs[np.lexsort((-pairs[:, 1].astype(np.int64), pairs[:, 0]))],
                               layout=gb.Layout.Unsorted)
    desc.serialize(tmp_path / "desc.bin")
    back = gb.Graph.load(tmp_path / "desc.bin", file_format=gb.FileFormat.Binary)
    off, tgt = back.csr()
    assert any((np.diff(tgt[off[v]:off[v + 1]].astype(np.int64)) < 0).any() for v in range(n))
    assert back.global_triangle_count().triangles == desc.global_triangle_count().triangles == \
        oracle.triangle_count(off, tgt, threads=1)


def test_degree_ordered_scale8_reloads_with_227874_triangles(tmp_path, golden_dir, goldens):
    g = gb.Graph.load(golden_dir / "scale_8.graph500", layout=gb.Layout.Sorted)
    g.make_degree_ordered()
    g.serialize(tmp_path / "ordered.bin")
    h = gb.Graph.load(tmp_path / "ordered.bin", file_format=gb.FileFormat.Binary)
    want = goldens["triangle_count_scale8_degree_ordered"]["triangles"]
    assert want == 227874
    assert h.global_triangle_count().triangles == want
    assert_same(h, g)


@pytest.mark.parametrize("chunk", [None, 64])
def test_single_node_without_edges(tmp_path, monkeypatch, chunk):
    set_chunk(monkeypatch, chunk)
    z = (np.array([0, 0]), np.array([], np.uint64), None)
    for kind, csrs in (("digraph", [z, z]), ("graph", [z])):
        (tmp_path / "z.bin").write_bytes(br.write(csrs, "usize"))
        g = load(tmp_path / "z.bin", kind)
        assert (g.node_count(), g.edge_count()) == (1, 0)
        g.serialize(tmp_path / "z2.bin")
        assert (tmp_path / "z2.bin").read_bytes() == br.write(csrs)


@pytest.mark.parametrize("chunk", [None, 64, 1009])
def test_errors_on_the_device_path(tmp_path, monkeypatch, edges, chunk):
    set_chunk(monkeypatch, chunk)
    src, dst, n, w = edges
    csrs = oracle_csrs(src, dst, n, "digraph", gb.Layout.Sorted)
    good = br.write(csrs)
    p = tmp_path / "e.bin"

    def expect(data, match, kind="digraph"):
        p.write_bytes(data)
        with pytest.raises(ValueError, match=match):
            load(p, kind)

    expect(good[:-3], "end of file")
    expect(good + b"\0", "trailing")
    expect(good[:8] + np.array([3], "<u8").tobytes() + b"i64" + good[19:], "invalid id size")
    expect(good, "holds a directed graph", kind="graph")
    expect(br.write(csrs[:1]), "holds an undirected graph")
    expect(np.array([n + 1], "<u8").tobytes() + good[8:], "number of node values")
    (oo, ot, _), (io, it, _) = csrs
    bad = ot.copy(); bad[5] = n
    expect(br.write([(oo, bad, None), (io, it, None)]), "targets >= node_count")
    bad = io.copy(); bad[3], bad[4] = bad[4] + 1, bad[3]
    expect(br.write([(oo, ot, None), (bad, it, None)]), "not monotone")
    bad = oo.copy(); bad[0] = 1
    expect(br.write([(bad, ot, None), (io, it, None)]), "offsets\\[0\\] must be 0")
    bad = ot.astype(np.uint64); bad[7] = 1 << 32
    expect(br.write([(oo, bad, None), (io, it, None)], "u64"), "does not fit 32 bits")
    bad = io.astype(np.uint64); bad[-1] += 1 << 32
    expect(br.write([(oo, ot, None), (bad, it, None)], "u64"), "does not fit 32 bits|offsets end at")


def test_rmat20_round_trip(tmp_path, monkeypatch):
    g = gb.DiGraph.rmat(20, layout=gb.Layout.Sorted, weights=True)
    g.serialize(tmp_path / "r.bin")
    assert (tmp_path / "r.bin").stat().st_size == 16 * g.edge_count() + 8 * g.node_count() + 54
    for chunk in (None, 1 << 20):
        set_chunk(monkeypatch, chunk)
        h = gb.DiGraph.load_weighted(tmp_path / "r.bin", file_format=gb.FileFormat.Binary)
        assert_same(h, g)
    h.serialize(tmp_path / "r2.bin")
    assert (tmp_path / "r2.bin").read_bytes() == (tmp_path / "r.bin").read_bytes()
