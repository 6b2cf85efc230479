"""The weighted undirected graph (UndirectedCsrGraph<u32, (), f32>) on the device: every constructor, conversion and
file path against the numpy restatement (tests/weighted_undirected_restatement.py), bit for bit, and against the
unweighted build of the same edges."""
import json

import numpy as np
import pytest

import binary_restatement as br
import graph_b200 as gb
import oracle
import weighted_undirected_restatement as wu
from thread_jobs import run_threads

pytestmark = pytest.mark.gpu

LAYOUTS = {"Unsorted": gb.Layout.Unsorted, "Sorted": gb.Layout.Sorted, "Deduplicated": gb.Layout.Deduplicated}


def _hub():
    """Node 0 holds 3000 parallel edges to node 7 with distinct values, and edges to every other node."""
    rng = np.random.default_rng(5)
    k = 3000
    src = np.concatenate([np.zeros(k, np.uint32), np.zeros(199, np.uint32), rng.integers(1, 200, 500, dtype=np.uint32)])
    dst = np.concatenate([np.full(k, 7, np.uint32), np.arange(1, 200, dtype=np.uint32),
                          rng.integers(0, 200, 500, dtype=np.uint32)])
    perm = rng.permutation(len(src))
    w = np.arange(len(src), dtype=np.float32) + np.float32(0.5)
    return src[perm], dst[perm], w, 0


def _random(seed, n, m, node_count):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, n, m, dtype=np.uint32)
    dst = rng.integers(0, n, m, dtype=np.uint32)
    dst[::11] = src[::11]  # self-loops
    src[1::4], dst[1::4] = src[::4][:len(src[1::4])], dst[::4][:len(dst[1::4])]  # duplicates
    return src, dst, rng.standard_normal(m).astype(np.float32), node_count


def _wel(golden_dir):
    rows = [line.split() for line in (golden_dir / "test.wel").read_text().splitlines() if line.strip()]
    return (np.array([int(r[0]) for r in rows], np.uint32), np.array([int(r[1]) for r in rows], np.uint32),
            np.array([float(r[2]) for r in rows], np.float32), 0)


def _rmat(scale):
    src, dst = oracle.rmat_edges(scale, seed=3)
    return src, dst, oracle.rmat_weights(3, 0, len(src)), 1 << scale


FIXTURES = ["test_wel", "dups_loops", "isolated", "empty", "hub", "rmat12"]


@pytest.fixture(scope="module", params=FIXTURES)
def fixture(request, golden_dir):
    name = request.param
    if name == "test_wel":
        return _wel(golden_dir)
    if name == "dups_loops":
        return _random(1, 40, 600, 0)
    if name == "isolated":
        return _random(2, 30, 100, 1000)  # ids below 30, nodes up to 999 without edges
    if name == "empty":
        return np.empty(0, np.uint32), np.empty(0, np.uint32), np.empty(0, np.float32), 5
    if name == "hub":
        return _hub()
    return _rmat(12)


def node_count(src, dst, n):
    return n if n else int(max(src.max(), dst.max())) + 1


def arrays(g):
    off, tgt = g.csr()
    return off, tgt, g.weights()


def assert_arrays(got, want):
    for x, y in zip(got, want, strict=True):
        assert x.dtype == y.dtype and len(x) == len(y) and x.tobytes() == y.tobytes()


@pytest.mark.parametrize("layout", LAYOUTS)
def test_weighted_build_equals_the_restatement(fixture, layout):
    src, dst, w, n = fixture
    lay = LAYOUTS[layout]
    g = gb.Graph.from_numpy(np.stack([src, dst], 1), lay, node_count=n, weights=w)
    assert g._info.has_weights == 1
    nn = node_count(src, dst, n)
    want = wu.build(src, dst, w, nn, lay.value)
    assert g.node_count() == nn and g.edge_count() == len(want[1]) // 2
    assert_arrays(arrays(g), want)
    # offsets and targets are the unweighted build's, byte for byte
    u = gb.Graph.from_numpy(np.stack([src, dst], 1), lay, node_count=n)
    assert u._info.has_weights == 0
    assert_arrays(u.csr(), want[:2])
    # the device-edge constructor agrees with the host one
    import torch
    dev = torch.device("cuda", 0)
    t = gb.Graph.from_torch(torch.from_numpy(src.astype(np.int64)).to(dev), torch.from_numpy(dst.astype(np.int64)).to(dev),
                            node_count=n, layout=lay, weights=torch.from_numpy(w).to(dev))
    assert t._info.has_weights == 1
    assert_arrays(arrays(t), want)


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("source", ["numpy", "rmat"])
def test_to_undirected_weighted_feeds_the_out_csr_in_csr_order(layout, source):
    if source == "rmat":
        d = gb.DiGraph.rmat(11, weights=True, layout=gb.Layout.Unsorted)
    else:
        src, dst, w, _ = _random(7, 60, 900, 0)
        d = gb.DiGraph.from_numpy(np.stack([src, dst], 1), gb.Layout.Unsorted, weights=w)
    lay = LAYOUTS[layout]
    g = d.to_undirected(lay, weights=True)
    off, tgt = d.csr("out")
    s, t, w = wu.csr_edges(off, tgt, d.out_weights())
    want = wu.build(s, t, w, d.node_count(), lay.value)
    assert_arrays(arrays(g), want)
    assert_arrays(d.to_undirected(lay).csr(), want[:2])
    assert d.to_undirected(lay)._info.has_weights == 0  # the default keeps its behaviour


def test_to_undirected_weighted_needs_a_weighted_digraph():
    d = gb.DiGraph.from_numpy(np.array([[0, 1], [1, 2]], np.uint32))
    with pytest.raises(ValueError, match="edge values"):
        d.to_undirected(weights=True)
    io, it = np.array([0, 0, 1, 2], np.uint32), np.array([0, 1], np.uint32)
    pr = gb.DiGraph.for_page_rank(io, it, np.array([0, 1, 2, 2], np.uint32))
    with pytest.raises(ValueError, match="page-rank-only|edge values"):
        pr.to_undirected(weights=True)


def write_wel(path, src, dst, w):
    with open(path, "w") as f:
        for s, t, x in zip(src.tolist(), dst.tolist(), w.tolist()):
            f.write(f"{s} {t} {np.format_float_positional(np.float32(x), unique=True)}\n")


@pytest.mark.parametrize("layout", LAYOUTS)
def test_load_weighted_host_and_streamed_paths_agree(tmp_path, monkeypatch, layout):
    src, dst, w, _ = _random(9, 500, 20000, 0)
    p = tmp_path / "g.wel"
    write_wel(p, src, dst, w)
    s2, d2, w2 = gb._read_edge_list(p, with_values=True)
    assert (s2 == src).all() and (d2 == dst).all() and w2.tobytes() == w.tobytes()
    lay = LAYOUTS[layout]
    monkeypatch.delenv("GB_LOAD_CHUNK_BYTES", raising=False)
    host = gb.Graph.load_weighted(p, lay)
    monkeypatch.setenv("GB_LOAD_CHUNK_BYTES", "65536")
    streamed = gb.Graph.load_weighted(p, lay)
    assert streamed.load_info()["chunks"] > 1
    want = wu.build(src, dst, w, node_count(src, dst, 0), lay.value)
    assert_arrays(arrays(host), want)
    assert_arrays(arrays(streamed), want)
    # the unweighted load of the same file keeps dropping the values
    assert gb.Graph.load(p, lay, gb.FileFormat.EdgeList)._info.has_weights == 0


@pytest.mark.parametrize("chunk", [None, "64", "1009"])
def test_golden_binary_round_trip(golden_dir, tmp_path, monkeypatch, chunk):
    if chunk is None:
        monkeypatch.delenv("GB_LOAD_CHUNK_BYTES", raising=False)
    else:
        monkeypatch.setenv("GB_LOAD_CHUNK_BYTES", chunk)
    f32 = golden_dir / "binary_undirected_u32_values.bin"
    g = gb.Graph.load_weighted(f32, file_format=gb.FileFormat.Binary)
    (off, tgt, val), = br.read(f32.read_bytes(), 1, True)
    assert_arrays(arrays(g), (off.astype(np.uint32), tgt.astype(np.uint32), val))
    out = tmp_path / "again.bin"
    g.serialize(out)
    assert out.read_bytes() == f32.read_bytes()
    usize = gb.Graph.load_weighted(golden_dir / "binary_undirected_usize_values.bin", file_format=gb.FileFormat.Binary)
    assert_arrays(arrays(usize), arrays(g))
    with pytest.raises(ValueError, match="holds no edge values"):
        gb.Graph.load_weighted(golden_dir / "binary_undirected_u32.bin", file_format=gb.FileFormat.Binary)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_save_and_load_of_a_built_twin(tmp_path, layout):
    src, dst, w, _ = _random(11, 300, 5000, 0)
    lay = LAYOUTS[layout]
    g = gb.Graph.from_numpy(np.stack([src, dst], 1), lay, weights=w)
    p = tmp_path / "g.bin"
    g.serialize(p)
    off, tgt, val = arrays(g)
    assert p.read_bytes() == br.write([(off, tgt, val)], "u32")
    again = gb.Graph.load_weighted(p, file_format=gb.FileFormat.Binary)
    assert_arrays(arrays(again), (off, tgt, val))


def test_degree_ordering_refused_and_triangles_counted(golden_dir):
    src, dst, w, n = _rmat(12)
    g = gb.Graph.from_numpy(np.stack([src, dst], 1), gb.Layout.Deduplicated, node_count=n, weights=w)
    before = [a.copy() for a in arrays(g)]
    with pytest.raises(ValueError, match="EV: Ord"):
        g.make_degree_ordered()
    g._host.clear()
    assert_arrays(arrays(g), before)
    u = gb.Graph.from_numpy(np.stack([src, dst], 1), gb.Layout.Deduplicated, node_count=n)
    assert g.global_triangle_count().triangles == u.global_triangle_count().triangles
    off, tgt = u.csr()
    assert g.global_triangle_count().triangles == oracle.triangle_count(off, tgt, threads=0)


def test_flight_engine_keeps_the_values(tmp_path):
    pa = pytest.importorskip("pyarrow")
    pytest.importorskip("pyarrow.flight")
    from graph_b200.flight import B200Engine, GraphFlightServer
    src, dst, w, _ = _random(13, 50, 400, 0)
    p = tmp_path / "g.wel"
    write_wel(p, src, dst, w)
    kind, g = B200Engine().load(str(p), "EdgeListWeighted", "Undirected", "Sorted")
    assert kind == "undirected+weighted" and g._info.has_weights == 1
    assert_arrays(arrays(g), wu.build(src, dst, w, node_count(src, dst, 0), wu.SORTED))
    server = GraphFlightServer("grpc://127.0.0.1:0")
    try:
        doc = {"graph_name": "w", "file_format": "EdgeListWeighted", "path": str(p), "csr_layout": "Sorted",
               "orientation": "Undirected"}
        server._create(json.dumps(doc).encode())
        assert server._get("w")[0] == "undirected+weighted" and server._get("w")[1]._info.has_weights == 1
        with pytest.raises(pa.ArrowInvalid, match="Triangle count requires an undirected graph"):
            server._compute(json.dumps({"graph_name": "w", "property_key": "tc", "algorithm": "TriangleCount"}).encode())
        doc.update(graph_name="d", orientation="Directed")
        server._create(json.dumps(doc).encode())
        server._to_undirected(json.dumps({"graph_name": "d", "csr_layout": "Sorted"}).encode())
        kind, u = server._get("d")
        assert kind == "undirected+weighted" and u._info.has_weights == 1
        assert_arrays(arrays(u), arrays(g))
    finally:
        server.shutdown()


def test_threads_build_convert_and_read():
    """Two threads build and convert on their own handles while a third reads a shared one."""
    shared_src, shared_dst, shared_w, _ = _random(21, 2000, 30000, 0)
    shared = gb.Graph.from_numpy(np.stack([shared_src, shared_dst], 1), gb.Layout.Sorted, weights=shared_w)
    shared_want = wu.build(shared_src, shared_dst, shared_w, node_count(shared_src, shared_dst, 0), wu.SORTED)

    def builder(seed):
        src, dst, w, _ = _random(seed, 3000, 40000, 0)
        n = node_count(src, dst, 0)

        def build():
            g = gb.Graph.from_numpy(np.stack([src, dst], 1), gb.Layout.Deduplicated, weights=w)
            assert_arrays(arrays(g), wu.build(src, dst, w, n, wu.DEDUPLICATED))

        def convert():
            d = gb.DiGraph.from_numpy(np.stack([src, dst], 1), gb.Layout.Sorted, weights=w)
            g = d.to_undirected(gb.Layout.Unsorted, weights=True)
            s, t, x = wu.csr_edges(*d.csr("out"), d.out_weights())
            assert_arrays(arrays(g), wu.build(s, t, x, n, wu.UNSORTED))
        return [("build", build), ("convert", convert)]

    def read():
        assert_arrays((shared.csr()[0], shared.csr()[1], shared.weights()), shared_want)
        assert shared.device_bytes() > 0

    run_threads([builder(31), builder(32), [("read", read), ("read again", read)]], rounds=3)
