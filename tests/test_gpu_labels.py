"""Node-labelled graphs on the device: DotGraph loads (host reader and device parser), labelled twins, and the
LabelStats / NodeLabelIndex / NeighborLabelFrequencies kernels (graph_b200/csrc/labels.cu), all compared with the
restatement of the reference in tests/dotgraph_restatement.py and the CSR oracle."""
import numpy as np
import pytest

import graph_b200 as gb
import oracle
from conftest import GOLDEN
import dotgraph_restatement as dot

pytestmark = pytest.mark.gpu

LAYOUTS = {"Unsorted": (gb.Layout.Unsorted, oracle.UNSORTED), "Sorted": (gb.Layout.Sorted, oracle.SORTED),
           "Deduplicated": (gb.Layout.Deduplicated, oracle.DEDUPLICATED)}
# None: the host reader; a size: the device parser with buffers of that many bytes (64: lines straddle chunks)
PATHS = [None, 64, 4096, 1 << 20]


@pytest.fixture
def path_mode(monkeypatch):
    def set_mode(chunk):
        if chunk is None:
            monkeypatch.delenv("GB_LOAD_CHUNK_BYTES", raising=False)
        else:
            monkeypatch.setenv("GB_LOAD_CHUNK_BYTES", str(chunk))
    return set_mode


def load(path, directed, labeled, layout):
    cls = gb.DiGraph if directed else gb.Graph
    if labeled:
        return cls.load_labeled(path, layout=layout)
    return cls.load(path, layout=layout, file_format=gb.FileFormat.DotGraph)


def expected_csrs(g: dot.DotGraph, n, directed, layout):
    if directed:
        return [*oracle.csr_build(g.src, g.dst, n, oracle.OUTGOING, layout),
                *oracle.csr_build(g.src, g.dst, n, oracle.INCOMING, layout)]
    return list(oracle.csr_build(g.src, g.dst, n, oracle.UNDIRECTED, layout))


def got_csrs(h):
    if isinstance(h, gb.Graph):
        return list(h.csr())
    return [*h.csr("out"), *h.csr("in")]


def check_graph(h, g: dot.DotGraph, directed, labeled, layout):
    n = len(g.labels) if labeled else int(max(g.src.max(), g.dst.max())) + 1
    assert h.node_count() == n
    for a, b in zip(got_csrs(h), expected_csrs(g, n, directed, layout), strict=True):
        assert a.tobytes() == b.astype(np.uint32).tobytes()
    if labeled:
        assert h.node_values().tolist() == g.labels.tolist()
        assert h.load_info()["edges"] == len(g.src)
    else:
        assert not h.has_node_values()


@pytest.mark.parametrize("chunk", PATHS)
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("labeled", [True, False])
@pytest.mark.parametrize("directed", [True, False])
@pytest.mark.parametrize("name", ["test.graph", "example.graph"])
def test_goldens_load(path_mode, name, directed, labeled, layout, chunk):
    path_mode(chunk)
    g = dot.read((GOLDEN / name).read_bytes())
    check_graph(load(GOLDEN / name, directed, labeled, LAYOUTS[layout][0]), g, directed, labeled, LAYOUTS[layout][1])


def test_builder_node_values(path_mode):
    # builder.rs:370-391: GraphBuilder().csr_layout(Sorted).file_format(DotGraphInput).path(test.graph)
    path_mode(None)
    g = gb.DiGraph.load_labeled(GOLDEN / "test.graph", layout=gb.Layout.Sorted)
    assert [g.node_value(v) for v in range(5)] == [0, 1, 2, 1, 2]
    assert g.copy_out_neighbors(1) == [2, 3] and g.copy_in_neighbors(4) == [2, 3]


def rmat_dotgraph(tmp_path, scale=16, label_range=42, seed=7):
    src, dst = oracle.rmat_edges(scale, seed=seed)
    n = 1 << scale
    labels = np.random.default_rng(seed).integers(0, label_range, n)
    path = tmp_path / f"rmat{scale}.graph"
    path.write_bytes(dot.write(labels, list(zip(src.tolist(), dst.tolist())), degrees=np.arange(n) % 7))
    return path, dot.DotGraph(labels, src, dst, 6)


@pytest.mark.parametrize("chunk", [None, 1 << 16, 1 << 20])
@pytest.mark.parametrize("directed", [True, False])
def test_rmat16_load(tmp_path, path_mode, directed, chunk):
    path, g = rmat_dotgraph(tmp_path)
    path_mode(chunk)
    for labeled in (True, False):
        h = load(path, directed, labeled, gb.Layout.Sorted)
        check_graph(h, g, directed, labeled, oracle.SORTED)
        if chunk:
            assert h.load_info()["chunks"] > 1


@pytest.mark.parametrize("chunk", [None, 64])
@pytest.mark.parametrize("nodes", [3, 9])  # max id + 1 = 6: N below and above it
def test_unlabeled_node_count_rule(tmp_path, path_mode, chunk, nodes):
    path_mode(chunk)
    edges = [(0, 5), (2, 3), (5, 1)]
    path = tmp_path / "g.graph"
    path.write_bytes(dot.write(range(nodes), edges))
    assert gb.DiGraph.load(path, file_format=gb.FileFormat.DotGraph).node_count() == 6
    assert gb.Graph.load(path, file_format=gb.FileFormat.DotGraph).node_count() == 6
    if nodes < 6:
        with pytest.raises(ValueError, match="edge endpoints are >= node_count 3"):
            gb.DiGraph.load_labeled(path)
    else:
        assert gb.Graph.load_labeled(path).node_count() == nodes


@pytest.mark.parametrize("chunk", [None, 64, 4096])
@pytest.mark.parametrize("data, message", dot.MALFORMED)
def test_malformed_files(tmp_path, path_mode, chunk, data, message):
    path_mode(chunk)
    path = tmp_path / "bad.graph"
    path.write_bytes(data)
    for call in (lambda: gb.DiGraph.load_labeled(path), lambda: gb.Graph.load_labeled(path),
                 lambda: gb.Graph.load(path, file_format=gb.FileFormat.DotGraph)):
        with pytest.raises(ValueError) as e:
            call()
        assert str(e.value) == message


@pytest.mark.parametrize("chunk", [None, 64])
def test_accepted_variants(tmp_path, path_mode, chunk):
    path_mode(chunk)
    path = tmp_path / "ok.graph"
    for data in (dot.GOOD[:-1], dot.GOOD + b"garbage\n\r\n", b"t 2 1\n?\t0,4294967295;1\nxx1x6x1\n__0:1",
                 b"t " + b"0" * 9000 + b"2 01\n" + dot.GOOD[6:]):
        path.write_bytes(data)
        g = gb.Graph.load_labeled(path)
        assert g.node_values().tolist() == dot.read(data).labels.tolist()
        assert g.copy_neighbors(0) == [1]
    path.write_bytes(b"t 0 1\ne 0 1\n")
    with pytest.raises(ValueError, match="needs at least one node line"):
        gb.Graph.load_labeled(path)


# ---- the three structures ----------------------------------------------------------------------------
def check_structures(h: gb.Graph, index=True):
    """index=False skips NodeLabelIndex, whose max_label + 2 offsets are too many for labels near 2^32."""
    off, tgt = h.csr()
    labels = h.node_values()
    want = dot.label_stats(off, tgt, labels)
    st = h.label_stats()
    assert (st.max_degree, st.label_count, st.max_label, st.max_label_frequency) == \
        (want["max_degree"], want["label_count"], want["max_label"], want["max_label_frequency"])
    assert st.label_frequency == want["label_frequency"]
    if index:
        idx = h.node_label_index()
        w_off, w_nodes = dot.node_label_index(labels)
        assert idx.offsets.tolist() == w_off.tolist() and idx._nodes.tolist() == w_nodes.tolist()
    nlf = h.neighbor_label_frequencies()
    w_off, w_lab, w_cnt = dot.neighbor_label_frequencies(off, tgt, labels)
    assert nlf.offsets.tolist() == w_off.tolist()
    assert nlf.labels.tolist() == w_lab.tolist() and nlf.counts.tolist() == w_cnt.tolist()
    return nlf


def labeled_graph(src, dst, labels, layout=gb.Layout.Sorted):
    return gb.Graph.from_numpy(np.stack([src, dst], axis=1), layout=layout, node_values=labels)


@pytest.mark.parametrize("name", ["test.graph", "example.graph"])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_structures_goldens(name, layout):
    h = gb.Graph.load_labeled(GOLDEN / name, layout=LAYOUTS[layout][0])
    nlf = check_structures(h)
    if name == "test.graph":
        # dotgraph.rs:585-624
        assert nlf.neighbor_frequency(0).get(0) is None
        assert nlf.neighbor_frequency(1).get(0) == 1 and nlf.neighbor_frequency(4).get(2) == 1
        assert [h.node_label_index().nodes(l).tolist() for l in range(3)] == [[0], [1, 3], [2, 4]]


@pytest.mark.parametrize("label_range", [42, 1 << 20])
@pytest.mark.parametrize("layout", ["Unsorted", "Deduplicated"])
def test_structures_rmat16(label_range, layout):
    src, dst = oracle.rmat_edges(16, seed=11)
    labels = np.random.default_rng(label_range).integers(0, label_range, 1 << 16).astype(np.uint32)
    h = labeled_graph(src, dst, labels, LAYOUTS[layout][0])
    check_structures(h)


def test_structures_every_size_class():
    # rows of 0, 1, 32, 33, 512, 513, 2048, 2049 and 70000 entries; labels up to 2^32 - 1 (the largest key a
    # 32-bit sort holds, as the pads of the CTA rows are)
    rng = np.random.default_rng(5)
    degrees = [0, 1, 32, 33, 512, 513, 2048, 2049, 70000]
    n = 100000
    src = np.concatenate([np.full(d, i, np.uint32) for i, d in enumerate(degrees)])
    dst = rng.integers(len(degrees), n, len(src)).astype(np.uint32)
    for labels in (rng.integers(0, 1 << 20, n), rng.integers(0xFFFFFFF0, 0x100000000, n), rng.integers(0, 3, n)):
        check_structures(labeled_graph(src, dst, labels.astype(np.uint32), gb.Layout.Unsorted),
                         index=labels.max() < 1 << 20)


def test_structures_star_hub():
    n = 300001
    leaves = np.arange(1, n, dtype=np.uint32)
    labels = np.random.default_rng(3).integers(0, 1 << 20, n).astype(np.uint32)
    h = labeled_graph(np.zeros(n - 1, np.uint32), leaves, labels)
    nlf = check_structures(h)
    assert len(nlf.neighbor_frequency(0)) == len(np.unique(labels[1:]))


def test_structures_self_loops_duplicates_isolated_one_label():
    src = np.array([0, 0, 0, 1, 1], np.uint32)
    dst = np.array([0, 1, 1, 2, 2], np.uint32)
    h = labeled_graph(src, dst, np.array([5, 7, 5, 9, 9], np.uint32), gb.Layout.Unsorted)  # 3 and 4 isolated
    nlf = check_structures(h)
    assert dict(nlf.neighbor_frequency(0)) == {5: 2, 7: 2}
    assert len(nlf.neighbor_frequency(3)) == 0 and nlf.neighbor_frequency(3).is_empty()
    h = labeled_graph(src, dst, np.full(5, 4, np.uint32))
    nlf = check_structures(h)
    assert list(nlf.neighbor_frequency(1)) == [(4, 4)] and nlf.neighbor_frequency(1).get(3) is None


# ---- labels through the graph ops and the other algorithms ------------------------------------------------
def test_to_undirected_and_degree_order_keep_labels():
    d = gb.DiGraph.load_labeled(GOLDEN / "test.graph", layout=gb.Layout.Sorted)
    u = d.to_undirected(gb.Layout.Sorted)
    assert u.node_values().tolist() == [0, 1, 2, 1, 2]
    check_structures(u)
    before = u.node_values().copy()
    u.make_degree_ordered()
    # graph_ops.rs:511-538 swaps the CSR and leaves node_values where they were: the labels are not permuted
    assert u.node_values().tolist() == before.tolist()


def test_algorithms_ignore_labels():
    src, dst = oracle.rmat_edges(12, seed=9)
    n = 1 << 12
    arr = np.stack([src, dst], axis=1)
    labels = np.random.default_rng(1).integers(0, 42, n).astype(np.uint32)
    plain, labeled = gb.DiGraph.from_numpy(arr, gb.Layout.Sorted, node_count=n), \
        gb.DiGraph.from_numpy(arr, gb.Layout.Sorted, node_values=labels)
    for kw in ({"max_iterations": 10, "tolerance": 0.0}, {"max_iterations": 10, "tolerance": 0.0, "mode": "jacobi"}):
        assert plain.page_rank(**kw).scores().tobytes() == labeled.page_rank(**kw).scores().tobytes()
    assert (plain.wcc().components() == labeled.wcc().components()).all()
    pu, lu = plain.to_undirected(gb.Layout.Sorted), labeled.to_undirected(gb.Layout.Sorted)
    assert pu.global_triangle_count().triangles == lu.global_triangle_count().triangles
    assert labeled.device_bytes() == plain.device_bytes() + 4 * n


def test_max_label_query_and_timing():
    h = gb.Graph.load_labeled(GOLDEN / "test.graph")
    max_label = gb.C.c_uint32(0)
    assert gb.lib.gb_node_label_index(h._g, gb.C.byref(max_label), None, None) == gb._capi.GB_OK
    assert max_label.value == 2
    buf = np.empty(8, np.uint32)
    assert gb.lib.gb_node_label_index(h._g, None, gb._ptr(buf), None) == gb._capi.GB_ERR_INVALID
    for call in (h.label_stats, h.node_label_index, h.neighbor_label_frequencies):
        call()
        t = h.last_timing()
        assert t["total_ms"] > 0 and t["kernel_launches"] > 0


def test_unsupported(tmp_path):
    d = gb.DiGraph.load_labeled(GOLDEN / "test.graph")
    st = gb._capi.LabelStatsInfo()
    buf = np.empty(16, np.uint32)
    for status in (gb.lib.gb_label_stats(d._g, gb.C.byref(st), None, None),
                   gb.lib.gb_node_label_index(d._g, None, gb._ptr(buf), gb._ptr(buf)),
                   gb.lib.gb_neighbor_label_frequencies(d._g, gb._ptr(buf), gb._ptr(buf), gb._ptr(buf)),
                   gb.lib.gb_graph_serialize(d._g, str(tmp_path / "x.bin").encode())):
        assert status == gb._capi.GB_ERR_UNSUPPORTED
    assert not (tmp_path / "x.bin").exists()
    plain = gb.Graph.load(GOLDEN / "test.graph", file_format=gb.FileFormat.DotGraph)
    assert gb.lib.gb_label_stats(plain._g, gb.C.byref(st), None, None) == gb._capi.GB_ERR_UNSUPPORTED
    assert gb.lib.gb_graph_node_values(plain._g, None) == gb._capi.GB_ERR_UNSUPPORTED
    with pytest.raises(ValueError, match="node values"):
        plain.node_values()
    with pytest.raises(ValueError):
        gb.Graph.from_numpy(np.array([[0, 3]]), node_values=[1, 2])  # id 3 >= 2 labels


def test_graph_mate_names():
    import graph_mate
    g = graph_mate.Graph.load_labeled(GOLDEN / "test.graph", layout=graph_mate.Layout.Sorted)
    stats = g.label_stats()
    assert isinstance(stats, graph_mate.LabelStats)
    assert (stats.max_degree, stats.max_label, stats.max_label_frequency) == (3, 2, 2)
    assert stats.label_frequency == {0: 1, 1: 2, 2: 2}
    nlf = g.neighbor_label_frequencies()
    assert isinstance(nlf.neighbor_frequency(2), graph_mate.NeighborLabelFrequency)
    assert sorted(nlf.neighbor_frequency(2)) == [(0, 1), (1, 1), (2, 1)]
