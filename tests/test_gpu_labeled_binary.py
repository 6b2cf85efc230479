"""Labelled binary graph files on the device: load_labeled(file_format=FileFormat.Binary) (host decoder below 64 MiB,
the streamed path of graph_b200/csrc/load.cu when GB_LOAD_CHUNK_BYTES is set) and serialize_labeled().  Files are
checked against the Python restatement of the reference's format (tests/labeled_binary_restatement.py), and a
reloaded twin must equal the one that was saved: CSRs, labels and the three label structures."""
import ctypes as C

import numpy as np
import pytest

import binary_restatement as br
import labeled_binary_restatement as lbr
import dotgraph_restatement as dot
import graph_b200 as gb
import oracle
from conftest import GOLDEN
from thread_jobs import run_threads

pytestmark = pytest.mark.gpu

LAYOUTS = {"Unsorted": gb.Layout.Unsorted, "Sorted": gb.Layout.Sorted, "Deduplicated": gb.Layout.Deduplicated}
CHUNKS = [None, 64, 4096, 1009]  # None: the host decoder; 1009 is prime, so 8-byte labels straddle chunks


def set_chunk(monkeypatch, chunk):
    if chunk is None:
        monkeypatch.delenv("GB_LOAD_CHUNK_BYTES", raising=False)
    else:
        monkeypatch.setenv("GB_LOAD_CHUNK_BYTES", str(chunk))


def cls_of(directed):
    return gb.DiGraph if directed else gb.Graph


def load_binary(path, directed, label_bytes=4, layout=None):
    return cls_of(directed).load_labeled(path, layout=layout, file_format=gb.FileFormat.Binary, label_bytes=label_bytes)


def csrs_of(g):
    if isinstance(g, gb.Graph):
        return [tuple(g.csr())]
    return [tuple(g.csr("out")), tuple(g.csr("in"))]


def restated(g, name="u32", label_bytes=4):
    """the bytes of g as a labelled file: its labels, then its CSRs without values"""
    return lbr.write([(o, t, None) for o, t in csrs_of(g)], name, labels=g.node_values(), label_bytes=label_bytes)


def assert_same(a, b):
    assert type(a) is type(b)
    assert (a.node_count(), a.edge_count(), a._info.has_weights) == (b.node_count(), b.edge_count(), b._info.has_weights)
    for (o1, t1), (o2, t2) in zip(csrs_of(a), csrs_of(b), strict=True):
        assert o1.tobytes() == o2.tobytes() and t1.tobytes() == t2.tobytes()
    assert a.node_values().tobytes() == b.node_values().tobytes()


def assert_same_structures(a, b):
    sa, sb = a.label_stats(), b.label_stats()
    assert (sa.max_degree, sa.label_count, sa.max_label, sa.max_label_frequency, sa.label_frequency) == \
        (sb.max_degree, sb.label_count, sb.max_label, sb.max_label_frequency, sb.label_frequency)
    ia, ib = a.node_label_index(), b.node_label_index()
    assert ia.offsets.tobytes() == ib.offsets.tobytes() and ia._nodes.tobytes() == ib._nodes.tobytes()
    fa, fb = a.neighbor_label_frequencies(), b.neighbor_label_frequencies()
    for x, y in ((fa.offsets, fb.offsets), (fa.labels, fb.labels), (fa.counts, fb.counts)):
        assert x.tobytes() == y.tobytes()


def streamed_h2d(g):
    """bytes a u32 file without values sends to the device: the labels, and per CSR its offsets and targets (the
    host path uploads the same arrays)"""
    n = g.node_count()
    return 4 * n + sum(4 * (n + 1) + 4 * len(t) for _, t in csrs_of(g))


def file_edges(g):
    """load_info()["edges"] of g's file: the entries of a directed CSR, half those of an undirected one"""
    entries = len(csrs_of(g)[0][1])
    return entries if isinstance(g, gb.DiGraph) else entries // 2


def round_trip(g, tmp_path, chunk, layout=None):
    """saves g, checks the file against the restatement, reloads it and checks the reload and its file"""
    directed = isinstance(g, gb.DiGraph)
    p, q = tmp_path / "g.bin", tmp_path / "h.bin"
    g.serialize_labeled(p)
    data = p.read_bytes()
    assert data == restated(g)
    h = load_binary(p, directed, layout=layout)
    assert_same(h, g)
    info = h.load_info()
    assert info["file_bytes"] == len(data)
    assert info["chunks"] == (0 if chunk is None else -(-len(data) // chunk))
    assert info["h2d_bytes"] == streamed_h2d(h)
    assert info["edges"] == file_edges(g)
    h.serialize_labeled(q)
    assert q.read_bytes() == data
    p.unlink()
    q.unlink()
    return h


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("directed", [True, False])
@pytest.mark.parametrize("name", ["test.graph", "example.graph"])
def test_dotgraph_files_round_trip(tmp_path, monkeypatch, name, directed, layout, chunk):
    set_chunk(monkeypatch, chunk)
    g = cls_of(directed).load_labeled(GOLDEN / name, layout=LAYOUTS[layout])
    assert g.node_values().tolist() == dot.read((GOLDEN / name).read_bytes()).labels.tolist()
    h = round_trip(g, tmp_path, chunk, LAYOUTS[layout])
    if not directed:
        assert_same_structures(h, g)


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("values", ["", "_values"])
@pytest.mark.parametrize("kind", ["directed", "undirected"])
def test_goldens_load_alike_at_both_widths(golden_dir, monkeypatch, kind, values, chunk):
    set_chunk(monkeypatch, chunk)
    directed = kind == "directed"
    a = load_binary(golden_dir / f"binary_labeled_{kind}_u32{values}.bin", directed, 4)
    b = load_binary(golden_dir / f"binary_labeled_{kind}_usize{values}.bin", directed, 8)
    assert_same(a, b)
    assert a.node_values().tolist() == lbr.LABELS
    assert a._info.has_weights == 0  # values in the records are dropped
    labels, csrs = lbr.read((golden_dir / f"binary_labeled_{kind}_u32{values}.bin").read_bytes(), 2 if directed else 1,
                           bool(values), label_bytes=4)
    for (o, t), (wo, wt, _) in zip(csrs_of(a), csrs, strict=True):
        assert o.tolist() == wo.tolist() and t.tolist() == wt.tolist()
    # whatever the file held, the twin's file is the u32 one without values
    assert restated(b) == lbr.write([(o, t, None) for o, t, _ in csrs], labels=labels, label_bytes=4)


def malformed_files():
    """(name, bytes, directed, label_bytes) of the malformed files of the CPU tests"""
    o, t = br.sorted_csr(br.EDGES, 4)
    i, it = br.sorted_csr([(d, s) for s, d in br.EDGES], 4)
    csrs = [(o, t, None), (i, it, None)]
    out = []
    for lb in (4, 8):
        name = "u32" if lb == 4 else "usize"
        for labels in ([1, 2, 3], [1, 2, 3, 4, 5]):
            out.append((f"count {len(labels)} {name}", lbr.write(csrs, labels=labels, label_bytes=lb), True, lb))
        good = lbr.write(csrs, name, labels=lbr.LABELS, label_bytes=lb)
        out.append((f"count 2^63 {name}", np.array([1 << 63], "<u8").tobytes() + good[8:], True, lb))
        bad = t.copy()
        bad[0] = 4
        out.append((f"targets {name}", lbr.write([(o, bad, None), (i, it, None)], labels=lbr.LABELS, label_bytes=lb),
                    True, lb))
        out.append((f"trailing {name}", good + b"\0", True, lb))
        out.append((f"kind {name}", good, False, lb))
        out.append((f"other width {name}", good, True, 12 - lb))
    wide = np.array([1, 2, 1 << 32, (1 << 64) - 1], np.uint64)
    out.append(("wide labels", lbr.write(csrs, "usize", labels=wide, label_bytes=8), True, 8))
    out.append(("wide label and targets", lbr.write([(o, bad, None), (i, it, None)], "usize", labels=wide, label_bytes=8),
                True, 8))
    for lb in (0, 2, 16):
        out.append((f"label_bytes {lb}", lbr.labeled_golden_files()["binary_labeled_directed_u32.bin"], True, lb))
    for name, data in lbr.labeled_golden_files().items():
        lb = 8 if "_usize" in name else 4
        out.append((f"{name} under width {lb}", data, "undirected" not in name, 12 - lb))
    for name in ("binary_labeled_directed_usize_values.bin", "binary_labeled_undirected_u32.bin"):
        data = lbr.labeled_golden_files()[name]
        for cut in range(len(data)):
            out.append((f"{name}[:{cut}]", data[:cut], "undirected" not in name, 8 if "_usize" in name else 4))
    for name, data in br.golden_files().items():  # unlabelled files
        for lb in (4, 8):
            out.append((f"{name} as labelled {lb}", data, "undirected" not in name, lb))
    return out


def attempt(path, directed, label_bytes):
    """(status, message) of the C load; a graph that loads is freed"""
    fn = gb.lib.gb_digraph_load_labeled_binary_u32 if directed else gb.lib.gb_graph_load_labeled_binary_u32
    out = C.c_void_p()
    status = fn(gb._device, str(path).encode(), gb._capi.LAYOUT_UNSORTED, label_bytes, C.byref(out))
    if status == gb._capi.GB_OK:
        gb.lib.gb_graph_free(out)
        return status, ""
    return status, gb.lib.gb_last_error().decode()


def test_malformed_files_fail_alike_on_every_path(tmp_path, monkeypatch):
    p = tmp_path / "bad.bin"
    cases = malformed_files()
    for what, data, directed, lb in cases:
        p.write_bytes(data)
        want = gb._capi.GB_ERR_INVALID, None
        for chunk in CHUNKS:
            set_chunk(monkeypatch, chunk)
            got = attempt(p, directed, lb)
            assert got[0] == gb._capi.GB_ERR_INVALID, (what, chunk, got)
            if want[1] is None:
                want = got
            assert got == want, (what, chunk)
        if lb in (4, 8):  # the host decoder gives the same message
            with pytest.raises(ValueError) as e:
                gb._decode_binary_labeled(data, directed, lb)
            assert str(e.value) == want[1], what
    assert sorted(p.parent.iterdir()) == [p]


def test_wide_label_messages(tmp_path, monkeypatch):
    p = tmp_path / "w.bin"
    o, t = br.sorted_csr(br.EDGES, 4)
    p.write_bytes(lbr.write([(o, t, None)], "usize", labels=np.array([1, 2, 1 << 32, 1 << 33], np.uint64),
                           label_bytes=8))
    for chunk in CHUNKS:
        set_chunk(monkeypatch, chunk)
        with pytest.raises(ValueError, match="^binary graph file: the node value of node 2 does not fit 32 bits$"):
            load_binary(p, False, 8)
    p.write_bytes(np.array([1 << 63], "<u8").tobytes() + p.read_bytes()[8:])
    for chunk in CHUNKS:
        set_chunk(monkeypatch, chunk)
        with pytest.raises(ValueError, match="^binary graph file: unexpected end of file$"):
            load_binary(p, False, 8)


def rmat_labeled(directed, scale, seed, label_max=1 << 20):
    src, dst = oracle.rmat_edges(scale, seed=seed)
    labels = np.random.default_rng(seed).integers(0, label_max, 1 << scale, dtype=np.uint64).astype(np.uint32)
    return cls_of(directed).from_numpy(np.stack([src, dst], axis=1), layout=gb.Layout.Sorted, node_values=labels)


@pytest.mark.parametrize("chunk", [None, 1 << 16, 1009])
@pytest.mark.parametrize("directed", [True, False])
def test_rmat16_round_trip(tmp_path, monkeypatch, directed, chunk):
    g = rmat_labeled(directed, 16, 3)
    set_chunk(monkeypatch, chunk)
    h = round_trip(g, tmp_path, chunk)
    if chunk:
        assert h.load_info()["chunks"] > 1
    if not directed:
        assert_same_structures(h, g)


@pytest.mark.parametrize("chunk", CHUNKS)
@pytest.mark.parametrize("id_name", ["u32", "usize"])
@pytest.mark.parametrize("directed", [True, False])
def test_eight_byte_labels_cross_chunks(tmp_path, monkeypatch, directed, id_name, chunk):
    """u32 and usize ids with usize labels (NV's width is independent of NI's), labels up to 2^32 - 1; at chunk
    1009 the labels and ids straddle chunk boundaries.  A wide label far into the file is found on every path."""
    g = rmat_labeled(directed, 12, 5, label_max=1 << 32)
    labels = g.node_values().astype(np.uint64)
    labels[[0, -1]] = 0xFFFFFFFF
    csrs = [(o, t, None) for o, t in csrs_of(g)]
    p = tmp_path / "l.bin"
    p.write_bytes(lbr.write(csrs, id_name, labels=labels, label_bytes=8))
    set_chunk(monkeypatch, chunk)
    h = load_binary(p, directed, 8)
    assert h.node_values().tobytes() == labels.astype(np.uint32).tobytes()
    for (o1, t1), (o2, t2, _) in zip(csrs_of(h), csrs, strict=True):
        assert o1.tobytes() == o2.tobytes() and t1.tobytes() == t2.tobytes()
    h.serialize_labeled(tmp_path / "back.bin")
    assert (tmp_path / "back.bin").read_bytes() == lbr.write(csrs, labels=labels, label_bytes=4)
    wide = labels.copy()
    wide[[2999, 3001, 4000]] += 1 << 32
    p.write_bytes(lbr.write(csrs, id_name, labels=wide, label_bytes=8))
    with pytest.raises(ValueError, match="^binary graph file: the node value of node 2999 does not fit 32 bits$"):
        load_binary(p, directed, 8)


def test_to_undirected_and_degree_order_save_labels_as_stored(tmp_path, monkeypatch):
    d = rmat_labeled(True, 10, 8, label_max=50)
    u = d.to_undirected(gb.Layout.Sorted)
    assert u.node_values().tobytes() == d.node_values().tobytes()
    for chunk in (None, 1009):
        set_chunk(monkeypatch, chunk)
        assert_same_structures(round_trip(u, tmp_path, chunk), u)
    w = rmat_labeled(False, 10, 9, label_max=50)
    before = w.node_values().copy()
    w.make_degree_ordered()
    assert w.node_values().tobytes() == before.tobytes()  # the labels are not permuted
    for chunk in (None, 1009):
        set_chunk(monkeypatch, chunk)
        h = round_trip(w, tmp_path, chunk)
        assert h.node_values().tobytes() == before.tobytes()
        assert_same_structures(h, w)


def test_serialize_labeled_refusals(tmp_path):
    p = tmp_path / "x.bin"
    plain = gb.Graph.from_numpy(np.array([[0, 1], [1, 2]]))
    assert gb.lib.gb_graph_serialize_labeled(plain._g, str(p).encode()) == gb._capi.GB_ERR_UNSUPPORTED
    with pytest.raises(ValueError, match="no node values"):
        plain.serialize_labeled(p)
    off = np.array([0, 1, 2], np.uint32)
    pr = gb.DiGraph.for_page_rank(off, np.array([1, 0], np.uint32), off)
    assert gb.lib.gb_graph_serialize_labeled(pr._g, str(p).encode()) == gb._capi.GB_ERR_INVALID
    # a labelled twin keeps being refused by the unlabelled writer
    lab = gb.Graph.from_numpy(np.array([[0, 1], [1, 2]]), node_values=[4, 5, 6])
    assert gb.lib.gb_graph_serialize(lab._g, str(p).encode()) == gb._capi.GB_ERR_UNSUPPORTED
    assert list(tmp_path.iterdir()) == []
    lab.serialize_labeled(p)
    assert list(tmp_path.iterdir()) == [p]


def test_load_info_on_the_streamed_path(tmp_path, monkeypatch):
    g = rmat_labeled(False, 14, 4)
    g.serialize_labeled(tmp_path / "g.bin")
    size = (tmp_path / "g.bin").stat().st_size
    assert size == 8 + 4 * g.node_count() + 8 + 3 + 8 + 4 * (g.node_count() + 1) + 4 * len(g.csr()[1])
    set_chunk(monkeypatch, 1 << 16)
    info = load_binary(tmp_path / "g.bin", False).load_info()
    assert info == {"file_bytes": size, "chunks": -(-size // (1 << 16)), "edges": file_edges(g), "fallback_lines": 0,
                    "h2d_bytes": streamed_h2d(g)}
    # 8-byte labels are staged: h2d counts whole chunks wherever a staged section lies
    o, t = g.csr()
    (tmp_path / "w.bin").write_bytes(lbr.write([(o, t, None)], labels=g.node_values(), label_bytes=8))
    info = load_binary(tmp_path / "w.bin", False, 8).load_info()
    assert info["h2d_bytes"] >= 8 * g.node_count() + 4 * (g.node_count() + 1) + 4 * len(t)


def test_two_threads_save_and_load(tmp_path, monkeypatch):
    monkeypatch.setenv("GB_LOAD_CHUNK_BYTES", str(4096))
    graphs = [rmat_labeled(False, 12, 21), rmat_labeled(True, 12, 22)]
    files = [restated(g) for g in graphs]

    def job(t):
        def fn():
            p = tmp_path / f"t{t}.bin"
            graphs[t].serialize_labeled(p)
            assert p.read_bytes() == files[t]
            assert_same(load_binary(p, t == 1), graphs[t])
        return fn

    run_threads([[("save and load", job(t))] for t in range(2)], rounds=4)
