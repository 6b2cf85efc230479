"""DiGraph.load / load_weighted / Graph.load parse files of 64 MiB or more on the device (graph_b200/csrc/load.cu).
The graph must be the one the host readers (_read_graph500 / _read_edge_list + _from_edges) give, byte for byte,
with the same errors.  Setting GB_LOAD_CHUNK_BYTES selects the device path for the small test files, and tiny
chunks make lines straddle chunks and tiles."""
import numpy as np
import pytest

import graph_b200 as gb

pytestmark = pytest.mark.gpu

LAYOUTS = [gb.Layout.Unsorted, gb.Layout.Sorted, gb.Layout.Deduplicated]
KINDS = ["digraph", "weighted", "graph"]
DEFAULT = 64 << 20  # the default buffer size; setting the knob selects the device path for small files too
CHUNKS = [64, 4096, DEFAULT]


def host_edges(path, fmt, kind):
    if fmt is gb.FileFormat.Graph500:
        src, dst, n = gb._read_graph500(path)
        return src, dst, None, n
    if kind == "weighted":
        return (*gb._read_edge_list(path, with_values=True), 0)
    return (*gb._read_edge_list(path), None, 0)


def host_graph(path, fmt, kind, layout):
    src, dst, w, n = host_edges(path, fmt, kind)
    if kind == "graph":
        return gb.Graph._from_edges(src, dst, n, layout)
    return gb.DiGraph._from_edges(src, dst, w, n, layout)


def device_graph(path, fmt, kind, layout):
    if kind == "graph":
        return gb.Graph.load(path, layout=layout, file_format=fmt)
    if kind == "weighted":
        return gb.DiGraph.load_weighted(path, layout=layout)
    return gb.DiGraph.load(path, layout=layout, file_format=fmt)


def arrays(g):
    if isinstance(g, gb.Graph):
        return list(g.csr())
    out = list(g.csr("out")) + list(g.csr("in"))
    if g._info.has_weights:
        out.append(g.out_weights())
    return out


def assert_same_graph(got, want):
    assert (got.node_count(), got.edge_count()) == (want.node_count(), want.edge_count())
    assert got._info.has_weights == want._info.has_weights
    for a, b in zip(arrays(got), arrays(want), strict=True):
        assert a.dtype == b.dtype and a.tobytes() == b.tobytes()


def check_file(path, fmt, kind, layout):
    want = host_graph(path, fmt, kind, layout)
    got = device_graph(path, fmt, kind, layout)
    assert_same_graph(got, want)
    info = got.load_info()
    src = host_edges(path, fmt, kind)[0]
    assert info["edges"] == len(src)
    with open(path, "rb") as f:
        assert info["file_bytes"] == len(f.read())
    return got, info


def set_chunk(monkeypatch, chunk):
    if chunk is None:
        monkeypatch.delenv("GB_LOAD_CHUNK_BYTES", raising=False)
    else:
        monkeypatch.setenv("GB_LOAD_CHUNK_BYTES", str(chunk))


# ---- the golden fixtures ---------------------------------------------------------------------------
GOLDEN = [("scale_8.graph500", gb.FileFormat.Graph500), ("example.el", gb.FileFormat.EdgeList),
          ("test.el", gb.FileFormat.EdgeList), ("windows.el", gb.FileFormat.EdgeList),
          ("example.wel", gb.FileFormat.EdgeList), ("test.wel", gb.FileFormat.EdgeList)]


@pytest.mark.parametrize("name,fmt", GOLDEN, ids=[g[0] for g in GOLDEN])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: l.name)
@pytest.mark.parametrize("chunk", [None, DEFAULT], ids=["by_size", "device"])
def test_golden_fixtures_match_host_readers(golden_dir, monkeypatch, name, fmt, kind, layout, chunk):
    if kind == "weighted" and fmt is gb.FileFormat.Graph500:
        pytest.skip("Graph500 files carry no values")
    set_chunk(monkeypatch, chunk)
    _, info = check_file(str(golden_dir / name), fmt, kind, layout)
    # small files are read by the host readers unless the knob is set
    assert (info["chunks"] == 0) == (chunk is None)


# ---- synthetic text files --------------------------------------------------------------------------
ADVERSARIAL_VALUES = [
    "", "+3", "++3", "+-3", "-3", "-", "-.5", ".5", "5.", "5.e3", "1e", "1e+", "1e-", "1E5", "1e5x", "1.5abc",
    "1.5 7", "1.2.3", "1e50", "-1e50", "1e39", "3.4028235e38", "3.40282357e38", "1e-30", "1e-38", "1e-40",
    "1e-45", "1e-46", "1.17549435e-38", "inf", "-inf", "infinity", "nan", "NaN", "nan(123)", "0x1p3", "0X10",
    "0", "-0", "0.0", "-0.0e5", "000001.5000", "0.1", "16777217", "16777219", "16777218.5", "33554435",
    "1.00000005960464477539", "1.0000000596046447", "1.0000000596046448", "1.000000059604644775390625",
    "12345678901234567890", "9007199254740993", "1e22", "1e23", "1e-22", "1e-23", "123456789e-30", "\x01",
    "1" * 300, "0." + "0" * 5000 + "1",
]


def write_text(path, data: str):
    with open(path, "wb") as f:
        f.write(data.encode("latin-1"))
    return str(path)


def synthetic_files(tmp_path):
    rng = np.random.default_rng(5)
    s = rng.integers(0, 300, 2000)
    d = rng.integers(0, 300, 2000)
    v = rng.random(2000).astype(np.float32)
    files = {}
    files["crlf"] = "".join(f"{a} {b} {x:g}\r\n" for a, b, x in zip(s, d, v))
    files["empty_lines"] = "".join(("\n" if k % 7 == 0 else "") + f"{a} {b} {x:.6f}\n"
                                   for k, (a, b, x) in enumerate(zip(s, d, v))) + "\n\n"
    files["no_trailing_newline"] = "".join(f"{a} {b} {x:.9g}\n" for a, b, x in zip(s, d, v)) + "7 8 0.5"
    files["adversarial"] = "".join(f"{k % 50} {(7 * k) % 61} {val}\n" for k, val in enumerate(ADVERSARIAL_VALUES * 3)) \
        + "3 4\n5\n\n9 9 1e5\r\n2 2 +1.25\r\n1 2 "
    return {k: write_text(tmp_path / f"{k}.el", t) for k, t in files.items()}


@pytest.mark.parametrize("chunk", CHUNKS, ids=lambda c: f"chunk{c}")
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: l.name)
def test_synthetic_text_files_match_host_readers(tmp_path, monkeypatch, chunk, kind, layout):
    set_chunk(monkeypatch, chunk)
    for name, path in synthetic_files(tmp_path).items():
        _, info = check_file(path, gb.FileFormat.EdgeList, kind, layout)
        if chunk == 64:
            assert info["chunks"] > 1, name
        if kind == "weighted":
            if name == "adversarial":
                assert info["fallback_lines"] > 0
            elif name in ("crlf", "empty_lines", "no_trailing_newline"):  # %g, %.6f, %.9g values
                assert info["fallback_lines"] == 0, name
        else:
            assert info["fallback_lines"] == 0


@pytest.fixture(scope="module")
def rmat16(tmp_path_factory):
    d = tmp_path_factory.mktemp("rmat16")
    m = 16 << 16
    src = np.empty(m, np.uint32)
    dst = np.empty(m, np.uint32)
    gb.check(gb.lib.gb_rmat_edges(0, 16, 42, 0, m, gb._ptr(src), gb._ptr(dst)))
    w = np.random.default_rng(1).random(m).astype(np.float32)
    g500 = str(d / "rmat16.graph500")
    gb.write_graph500(g500, src, dst)
    el = str(d / "rmat16.el")
    np.savetxt(el, np.stack([src, dst], 1), fmt="%d")
    wel = str(d / "rmat16.wel")
    with open(wel, "w") as f:
        f.write("".join(f"{a} {b} {x:.6g}\n" for a, b, x in zip(src.tolist(), dst.tolist(), w.tolist())))
    return {"g500": g500, "el": el, "wel": wel}


@pytest.mark.parametrize("chunk", [4096, DEFAULT], ids=lambda c: f"chunk{c}")
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: l.name)
def test_rmat16_files_match_host_readers(rmat16, monkeypatch, chunk, kind, layout):
    set_chunk(monkeypatch, chunk)
    if kind != "weighted":
        _, info = check_file(rmat16["g500"], gb.FileFormat.Graph500, kind, layout)
        assert info["fallback_lines"] == 0 and info["h2d_bytes"] == 12 * (16 << 16)
        _, info = check_file(rmat16["el"], gb.FileFormat.EdgeList, kind, layout)
    else:
        _, info = check_file(rmat16["wel"], gb.FileFormat.EdgeList, kind, layout)
    assert info["fallback_lines"] == 0
    if chunk == 4096:
        assert info["chunks"] > 1


@pytest.mark.parametrize("which", ["g500", "el", "wel"])
def test_rmat16_at_64_byte_chunks(rmat16, monkeypatch, which):
    set_chunk(monkeypatch, 64)
    fmt = gb.FileFormat.Graph500 if which == "g500" else gb.FileFormat.EdgeList
    _, info = check_file(rmat16[which], fmt, "weighted" if which == "wel" else "digraph", gb.Layout.Unsorted)
    assert info["chunks"] > 1000


def test_lines_longer_than_a_chunk(tmp_path, monkeypatch):
    set_chunk(monkeypatch, 64)
    text = "1 2 " + "1" * 9000 + "\n3 4 0.5\n" + "5 6 2." + "5" * 70 + "\n" + "7 8 9" + " " * 200
    path = write_text(tmp_path / "long.el", text)
    for kind in KINDS:
        check_file(path, gb.FileFormat.EdgeList, kind, gb.Layout.Unsorted)


# ---- errors ----------------------------------------------------------------------------------------
def host_and_device_error(path, fmt, kind="digraph"):
    errs = []
    for make in (host_graph, device_graph):
        with pytest.raises(Exception) as ei:
            make(path, fmt, kind, gb.Layout.Sorted)
        errs.append((type(ei.value), str(ei.value)))
    assert errs[0] == errs[1]
    return errs[1]


def graph500_bytes(src, dst, high=None):
    rec = np.zeros((len(src), 3), np.uint32)
    rec[:, 0], rec[:, 1] = src, dst
    if high is not None:
        rec[:, 2] = high
    return rec.tobytes()


def test_graph500_high_word_is_an_error(tmp_path, monkeypatch):
    src = np.arange(64, dtype=np.uint32) % 4
    high = np.zeros(64, np.uint32)
    high[37] = 1
    p = tmp_path / "high.graph500"
    p.write_bytes(graph500_bytes(src, src[::-1].copy(), high))
    for chunk in (48, None):
        set_chunk(monkeypatch, chunk)
        for kind in ("digraph", "graph"):
            t, msg = host_and_device_error(str(p), gb.FileFormat.Graph500, kind)
            assert t is ValueError and "32 bits" in msg


@pytest.mark.parametrize("chunk", [48, None])
def test_graph500_ids_beyond_node_count(tmp_path, monkeypatch, chunk):
    set_chunk(monkeypatch, chunk)
    src = np.arange(64, dtype=np.uint32) % 4
    dst = src.copy()
    dst[5] = 4  # node_count = 64 / 16 = 4
    p = tmp_path / "big.graph500"
    p.write_bytes(graph500_bytes(src, dst))
    t, msg = host_and_device_error(str(p), gb.FileFormat.Graph500)
    assert t is ValueError and "edge endpoints are >= node_count 4" in msg


@pytest.mark.parametrize("tail", [1, 5, 11])
def test_graph500_partial_record_tail_is_ignored(tmp_path, monkeypatch, tail):
    src = np.arange(40, dtype=np.uint32) % 2
    p = tmp_path / "tail.graph500"
    p.write_bytes(graph500_bytes(src, src[::-1].copy()) + b"\x07" * tail)
    for chunk in (48, None):
        set_chunk(monkeypatch, chunk)
        for kind in ("digraph", "graph"):
            check_file(str(p), gb.FileFormat.Graph500, kind, gb.Layout.Sorted)


@pytest.mark.parametrize("fmt", [gb.FileFormat.Graph500, gb.FileFormat.EdgeList], ids=lambda f: f.name)
@pytest.mark.parametrize("chunk", [64, None])
def test_empty_file(tmp_path, monkeypatch, fmt, chunk):
    set_chunk(monkeypatch, chunk)
    p = tmp_path / "empty"
    p.write_bytes(b"")
    t, msg = host_and_device_error(str(p), fmt)
    assert t is ValueError and msg == "cannot infer node_count from an empty edge list"


@pytest.mark.parametrize("chunk", [64, None])
def test_text_id_errors(tmp_path, monkeypatch, chunk):
    set_chunk(monkeypatch, chunk)
    p = write_text(tmp_path / "max.el", "0 1\n4294967295 2\n")
    t, msg = host_and_device_error(p, gb.FileFormat.EdgeList)
    assert t is ValueError and msg == "node id 2^32-1 leaves no room for node_count"
    p = write_text(tmp_path / "wide.el", "0 1\n4294967296 2\n")
    t, msg = host_and_device_error(p, gb.FileFormat.EdgeList)
    assert t is ValueError and "32 bits" in msg


def test_missing_file_raises_file_not_found(tmp_path):
    with pytest.raises(FileNotFoundError):
        gb.DiGraph.load(str(tmp_path / "nope.el"), file_format=gb.FileFormat.EdgeList)
    with pytest.raises(FileNotFoundError):
        gb.Graph.load(str(tmp_path / "nope.graph500"))


# ---- from_torch ------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["int32", "int64"])
@pytest.mark.parametrize("layout", LAYOUTS, ids=lambda l: l.name)
def test_from_torch_equals_from_numpy(dtype, layout):
    import torch
    rng = np.random.default_rng(3)
    src = rng.integers(0, 5000, 100000).astype(np.uint32)
    dst = rng.integers(0, 5000, 100000).astype(np.uint32)
    w = rng.random(100000).astype(np.float32)
    dt = getattr(torch, dtype)
    ts = torch.from_numpy(src.astype(np.int64)).to(dt).cuda()
    td = torch.from_numpy(dst.astype(np.int64)).to(dt).cuda()
    tw = torch.from_numpy(w).cuda()
    e = np.stack([src, dst], 1)
    assert_same_graph(gb.DiGraph.from_torch(ts, td, layout=layout), gb.DiGraph.from_numpy(e, layout=layout))
    assert_same_graph(gb.DiGraph.from_torch(ts, td, tw, layout=layout),
                      gb.DiGraph.from_numpy(e, layout=layout, weights=w))
    assert_same_graph(gb.DiGraph.from_torch(ts, td, node_count=6000, layout=layout),
                      gb.DiGraph.from_numpy(e, layout=layout, node_count=6000))
    assert_same_graph(gb.Graph.from_torch(ts, td, layout=layout), gb.Graph.from_numpy(e, layout=layout))


def test_from_torch_rejects_bad_ids():
    import torch
    ok = torch.arange(10, device="cuda")
    with pytest.raises(TypeError, match="32-bit"):
        gb.DiGraph.from_torch(ok - 1, ok)
    with pytest.raises(TypeError, match="32-bit"):
        gb.Graph.from_torch(ok, ok + (1 << 32))
    with pytest.raises(ValueError, match="node_count"):
        gb.DiGraph.from_torch(ok, ok, node_count=5)
    with pytest.raises(ValueError):
        gb.DiGraph.from_torch(ok.cpu(), ok.cpu())
    with pytest.raises(TypeError):
        gb.DiGraph.from_torch(ok.float(), ok)
