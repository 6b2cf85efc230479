"""graph_b200.wcc_file (gb_wcc_file_u32): the WCC of a graph file in one pass, each chunk's edges linked on the device as
they are decoded.  For every file DiGraph.load accepts, the node count and labels must be those of
DiGraph.load(...).wcc() and of the oracle's minimum-id labels over the twin's edges; every other file must fail with
the load's exception and message.  GB_LOAD_CHUNK_BYTES makes lines, records and binary elements straddle chunks."""
import os
import threading

import numpy as np
import pytest

import graph_b200 as gb
import oracle

pytestmark = pytest.mark.gpu

F = gb.FileFormat
CHUNKS = [None, 64, 4096]


def set_chunk(monkeypatch, chunk):
    if chunk is None:
        monkeypatch.delenv("GB_LOAD_CHUNK_BYTES", raising=False)
    else:
        monkeypatch.setenv("GB_LOAD_CHUNK_BYTES", str(chunk))


def min_labels(n, src, dst):
    """The oracle's labels (the minimum node id of each component) of the graph with these edges."""
    off, tgt = oracle.csr_build(np.asarray(src, np.uint32), np.asarray(dst, np.uint32), n, oracle.OUTGOING,
                                oracle.SORTED)
    return oracle.wcc_min_label(off, tgt)


def twin_edges(g):
    """Every edge of the twin's out- and in-CSR, as (src, dst)."""
    src, dst = [], []
    for which in ("out", "in"):
        off, tgt = g.csr(which)
        src.append(np.repeat(np.arange(len(off) - 1, dtype=np.uint32), np.diff(off.astype(np.int64))))
        dst.append(tgt)
    return np.concatenate(src), np.concatenate(dst)


def outcome(fn):
    try:
        return ("ok", fn())
    except Exception as e:  # noqa: BLE001 - the exception itself is what is compared
        return ("error", type(e), str(e))


def check_file(path, fmt):
    """wcc_file against DiGraph.load + wcc and the oracle; returns (labels, wcc_file_info()) or None for a file the
    load refuses (after checking that wcc_file refuses it the same way)."""
    path = str(path)
    load = outcome(lambda: gb.DiGraph.load(path, file_format=fmt))
    got = outcome(lambda: gb.wcc_file(path, fmt))
    if load[0] == "error":
        assert got == load
        assert gb.wcc_file_info()["node_count"] == 0
        return None
    g = load[1]
    assert got[0] == "ok", got
    labels = got[1].components()
    info = gb.wcc_file_info()
    want = g.wcc().components()
    assert labels.dtype == np.uint32 and labels.shape == (g.node_count(),)
    assert labels.tobytes() == want.tobytes()
    assert (labels == min_labels(g.node_count(), *twin_edges(g))).all()
    assert info["node_count"] == g.node_count()
    assert info["file_bytes"] == os.path.getsize(path)
    assert info["edges"] == g.load_info()["edges"]
    assert info["chunks"] >= 1 and info["device_bytes"] > 0 and info["total_ms"] > 0
    return labels, info


def write_text(path, text):
    with open(path, "wb") as f:
        f.write(text.encode("latin-1"))
    return str(path)


def el_bytes(src, dst):
    """Fixed-width decimal lines "sssssssssss ddddddddddd\\n" (leading zeros read as the same ids), written fast."""
    m = len(src)
    out = np.empty((m, 22), np.uint8)
    for col, a in ((0, src), (11, dst)):
        a = np.asarray(a, np.uint64).copy()
        for k in range(10):
            out[:, col + 9 - k] = ord("0") + (a % 10).astype(np.uint8)
            a //= 10
    out[:, 10] = ord(" ")
    out[:, 21] = ord("\n")
    return out.tobytes()


def rmat(scale):
    m = 16 << scale
    src = np.empty(m, np.uint32)
    dst = np.empty(m, np.uint32)
    gb.check(gb.lib.gb_rmat_edges(0, scale, 42, 0, m, gb._ptr(src), gb._ptr(dst)))
    return src, dst


# ---- every golden fixture ------------------------------------------------------------------------------
def golden_files():
    from pathlib import Path
    d = Path(__file__).resolve().parent / "golden"
    files = [("scale_8.graph500", F.Graph500)]
    files += [(n, F.EdgeList) for n in ("example.el", "test.el", "windows.el", "example.wel", "test.wel")]
    files += [(n, F.DotGraph) for n in ("example.graph", "test.graph")]
    files += [(p.name, F.Binary) for p in sorted(d.glob("binary_*.bin"))]
    return d, files


GOLDEN_DIR, GOLDEN = golden_files()


@pytest.mark.parametrize("chunk", CHUNKS, ids=lambda c: f"chunk{c}")
@pytest.mark.parametrize("name,fmt", GOLDEN, ids=[g[0] for g in GOLDEN])
def test_golden_fixtures_match_the_load(monkeypatch, chunk, name, fmt):
    set_chunk(monkeypatch, chunk)
    r = check_file(GOLDEN_DIR / name, fmt)
    if name.startswith("binary_directed"):
        assert r is not None, "every directed binary golden loads"
    if name.startswith("binary_undirected"):
        assert r is None
    if chunk == 64 and r is not None and os.path.getsize(GOLDEN_DIR / name) > 200:
        assert r[1]["chunks"] > 1


def test_undirected_binary_golden_message():
    with pytest.raises(ValueError) as ei:
        gb.wcc_file(GOLDEN_DIR / "binary_undirected_u32.bin", F.Binary)
    assert str(ei.value) == "binary graph file holds an undirected graph, not a directed one"


# ---- generated inputs with many chunks ----------------------------------------------------------------------
@pytest.fixture(scope="module")
def rmat_files(tmp_path_factory):
    d = tmp_path_factory.mktemp("rmat_files")
    files = {}
    for scale in (16, 20):
        src, dst = rmat(scale)
        g500 = str(d / f"rmat{scale}.graph500")
        gb.write_graph500(g500, src, dst)
        el = str(d / f"rmat{scale}.el")
        with open(el, "wb") as f:
            f.write(el_bytes(src, dst))
        binary = str(d / f"rmat{scale}.bin")
        gb.DiGraph.load(g500).serialize(binary)
        files[scale] = {F.Graph500: g500, F.EdgeList: el, F.Binary: binary}
    return files


@pytest.mark.parametrize("fmt", [F.Graph500, F.EdgeList, F.Binary], ids=lambda f: f.name)
@pytest.mark.parametrize("scale,chunk", [(16, 4096), (16, None), (20, 1 << 20), (20, None)])
def test_rmat_files(rmat_files, monkeypatch, fmt, scale, chunk):
    set_chunk(monkeypatch, chunk)
    labels, info = check_file(rmat_files[scale][fmt], fmt)
    assert labels.shape == (1 << scale,)
    if chunk is not None:
        assert info["chunks"] > 10


@pytest.mark.parametrize("chunk", [64, 4096], ids=lambda c: f"chunk{c}")
def test_deep_chains_stars_and_isolated_nodes(tmp_path, monkeypatch, chunk):
    set_chunk(monkeypatch, chunk)
    n = 30000
    ids = np.arange(n - 1, dtype=np.uint32)
    # a path in increasing id order: the largest id rises chunk after chunk, so parent[] grows many times
    check_file(write_text(tmp_path / "up.el", "".join(f"{i} {i + 1}\n" for i in ids)), F.EdgeList)
    # the same path listed from its far end, each edge written high -> low
    check_file(write_text(tmp_path / "down.el", "".join(f"{i + 1} {i}\n" for i in ids[::-1])), F.EdgeList)
    # a star whose hub is the last id, and a Graph500 chain padded with (0, 0) records
    check_file(write_text(tmp_path / "star.el", "".join(f"{i} {n}\n" for i in range(n))), F.EdgeList)
    src = np.zeros(16 * 2000, np.uint32)
    dst = np.zeros(16 * 2000, np.uint32)
    src[:1999], dst[:1999] = np.arange(1999, 0, -1), np.arange(1998, -1, -1)
    p = str(tmp_path / "chain.graph500")
    gb.write_graph500(p, src, dst)
    labels, _ = check_file(p, F.Graph500)
    assert (labels == 0).all()
    # isolated nodes around a few edges
    labels, _ = check_file(write_text(tmp_path / "iso.el", "7 3\n100000 99999\n5 5\n3 1\n"), F.EdgeList)
    assert labels.shape == (100001,) and labels[7] == 1 and labels[100000] == 99999 and labels[50000] == 50000


@pytest.mark.parametrize("chunk", [64, 4096, None], ids=lambda c: f"chunk{c}")
def test_text_shapes(tmp_path, monkeypatch, chunk):
    set_chunk(monkeypatch, chunk)
    rng = np.random.default_rng(3)
    s = rng.integers(0, 500, 3000)
    d = rng.integers(0, 500, 3000)
    v = rng.random(3000)
    check_file(write_text(tmp_path / "crlf.el", "".join(f"{a} {b}\r\n" for a, b in zip(s, d))), F.EdgeList)
    check_file(write_text(tmp_path / "open_end.el", "".join(f"{a} {b}\n" for a, b in zip(s, d)) + "600 2"),
               F.EdgeList)
    check_file(write_text(tmp_path / "values.wel", "".join(f"{a} {b} {x:.7g}\n" for a, b, x in zip(s, d, v))),
               F.EdgeList)
    check_file(write_text(tmp_path / "long_lines.el", "1 2 " + "9" * 9000 + "\n3 4\n5 6 " + " " * 300 + "\n"),
               F.EdgeList)
    nodes = "".join(f"v {i} {i % 3} 1\n" for i in range(400))
    edges = "".join(f"e {a % 400} {b % 400}\n" for a, b in zip(s[:800], d[:800]))
    check_file(write_text(tmp_path / "gen.graph", f"t 400 800\n{nodes}{edges}"), F.DotGraph)


# ---- errors: the load's exception and message ------------------------------------------------------------
def graph500_bytes(src, dst, high=None):
    rec = np.zeros((len(src), 3), np.uint32)
    rec[:, 0], rec[:, 1] = src, dst
    if high is not None:
        rec[:, 2] = high
    return rec.tobytes()


def error_files(tmp_path):
    src = np.arange(64, dtype=np.uint32) % 4
    high = np.zeros(64, np.uint32)
    high[37] = 1
    files = []

    def put(name, data, fmt):
        p = tmp_path / name
        p.write_bytes(data)
        files.append((str(p), fmt))
    put("high.graph500", graph500_bytes(src, src[::-1].copy(), high), F.Graph500)
    dst = src.copy()
    dst[5] = 4  # node_count = 64 / 16 = 4
    put("beyond.graph500", graph500_bytes(src, dst), F.Graph500)
    put("empty.graph500", b"", F.Graph500)
    put("short.graph500", b"\x01" * 11, F.Graph500)
    put("empty.el", b"", F.EdgeList)
    put("max.el", b"0 1\n4294967295 2\n", F.EdgeList)
    put("wide.el", b"0 1\n4294967296 2\n", F.EdgeList)
    put("wide_late.el", b"0 1\n" * 3000 + b"4294967296 2\n" + b"1 2\n" * 3000, F.EdgeList)
    put("max_late.el", b"0 1\n" * 3000 + b"4294967295 2\n" + b"1 2\n" * 3000, F.EdgeList)
    good = (GOLDEN_DIR / "binary_directed_u32.bin").read_bytes()
    put("bad_name.bin", good[:8] + b"\x03\x00\x00\x00\x00\x00\x00\x00" + b"u16" + good[19:], F.Binary)
    put("truncated.bin", good[:-3], F.Binary)
    put("trailing.bin", good + b"\x00" * 4, F.Binary)
    put("empty.bin", b"", F.Binary)
    put("bad_line.graph", b"t 2 2\nv 0 1 1\nv 1 1 1\ne 0 1\ne 0 x\n", F.DotGraph)
    put("missing.graph", b"t 2 3\nv 0 1 1\nv 1 1 1\ne 0 1\n", F.DotGraph)
    put("no_edges.graph", b"t 2 0\nv 0 1 1\nv 1 1 1\n", F.DotGraph)
    put("empty.graph", b"", F.DotGraph)
    return files


@pytest.mark.parametrize("chunk", [48, 64, None], ids=lambda c: f"chunk{c}")
def test_errors_match_the_load(tmp_path, monkeypatch, chunk):
    set_chunk(monkeypatch, chunk)
    for path, fmt in error_files(tmp_path):
        load = outcome(lambda: gb.DiGraph.load(path, file_format=fmt))
        got = outcome(lambda: gb.wcc_file(path, fmt))
        assert load[0] == "error", path
        assert got == load, path
        assert gb.wcc_file_info()["node_count"] == 0


def test_corrupt_binary_offsets_match_the_load(tmp_path, monkeypatch):
    good = bytearray((GOLDEN_DIR / "binary_directed_u32.bin").read_bytes())
    # the out-CSR's offsets start at byte 27 (8 + 8 + 3 + 4 + 4): a decreasing row, a wrong first and last entry,
    # and a target past node_count
    n = int.from_bytes(good[19:23], "little")
    cases = {"first": (27, 1), "middle": (27 + 4 * (n // 2), 0xFFFF), "last": (27 + 4 * n, 1)}
    cases["target"] = (27 + 4 * (n + 1), n + 5)
    for chunk in (64, None):
        set_chunk(monkeypatch, chunk)
        for name, (pos, value) in cases.items():
            bad = bytearray(good)
            bad[pos:pos + 4] = int(value).to_bytes(4, "little")
            p = tmp_path / f"{name}.bin"
            p.write_bytes(bytes(bad))
            load = outcome(lambda: gb.DiGraph.load(str(p), file_format=F.Binary))
            got = outcome(lambda: gb.wcc_file(p, F.Binary))
            assert got == load, name


@pytest.mark.parametrize("tail", [1, 5, 11])
def test_graph500_partial_record_tail_is_ignored(tmp_path, monkeypatch, tail):
    src = np.arange(40, dtype=np.uint32) % 2
    p = tmp_path / "tail.graph500"
    p.write_bytes(graph500_bytes(src, src[::-1].copy()) + b"\x07" * tail)
    for chunk in (48, None):
        set_chunk(monkeypatch, chunk)
        assert check_file(p, F.Graph500) is not None


def test_missing_file(tmp_path):
    with pytest.raises(FileNotFoundError):
        gb.wcc_file(tmp_path / "nope.graph500")
    with pytest.raises(FileNotFoundError):
        gb.wcc_file(str(tmp_path / "nope.el"), F.EdgeList)


# ---- no edge arrays ----------------------------------------------------------------------------------------
def test_device_bytes_do_not_grow_with_the_edges(tmp_path, monkeypatch):
    set_chunk(monkeypatch, 1 << 16)
    rng = np.random.default_rng(11)
    m = 100000
    src = rng.integers(0, 1000, m).astype(np.uint32)
    dst = rng.integers(0, 1000, m).astype(np.uint32)
    src[0], dst[0] = 999, 998  # the largest id comes first: parent[] is sized once
    once = el_bytes(src, dst)
    peaks = []
    for copies in (1, 4):
        p = tmp_path / f"x{copies}.el"
        p.write_bytes(once * copies)
        labels, info = check_file(p, F.EdgeList)
        assert info["edges"] == copies * m
        assert info["device_bytes"] < 8 * m
        peaks.append(info["device_bytes"])
    assert peaks[0] == peaks[1]


# ---- past 2^32 bytes and 2^32 records -------------------------------------------------------------------------
def sparse_dir(tmp_path):
    """A directory whose file system keeps files sparse: the test's temporary directory, else /dev/shm (tmpfs).  A
    1 GiB probe is extended there first; a file system whose free space drops by it is not used.  (Free space, not
    st_blocks: some file systems report a file's apparent size as its blocks.)"""
    for d in (str(tmp_path), "/dev/shm"):
        probe = os.path.join(d, f"sparse_probe_{os.getpid()}")
        try:
            before = os.statvfs(d)
            with open(probe, "wb") as f:
                f.truncate(1 << 30)
            after = os.statvfs(d)
            sparse = (before.f_bfree - after.f_bfree) * before.f_frsize < (256 << 20)
        except OSError:
            sparse = False
        finally:
            if os.path.exists(probe):
                os.unlink(probe)
        if sparse:
            return d
    pytest.skip("neither the temporary directory nor /dev/shm keeps files sparse")


def sparse_graph500(path, m, records):
    """A Graph500 file of m records, all (0, 0) except `records` {index: (src, dst)}, written as a sparse file."""
    try:
        with open(path, "wb") as f:
            f.truncate(12 * m)
            for r, (s, d) in records.items():
                f.seek(12 * r)
                f.write(np.array([s, d, 0], np.uint32).tobytes())
    except OSError as e:
        if os.path.exists(path):
            os.unlink(path)
        pytest.skip(f"the temporary directory cannot hold a sparse file of {12 * m} bytes: {e}")


def check_sparse(path, m, records):
    n = m // 16
    labels = gb.wcc_file(path).components()
    info = gb.wcc_file_info()
    assert labels.shape == (n,) and info["edges"] == m and info["node_count"] == n
    assert info["file_bytes"] == 12 * m and info["device_bytes"] < 4 * n + (1 << 30)
    ids = sorted({v for e in records.values() for v in e} | {0})
    idx = {v: i for i, v in enumerate(ids)}
    src = np.array([idx[s] for s, _ in records.values()], np.uint32)
    dst = np.array([idx[d] for _, d in records.values()], np.uint32)
    small = min_labels(len(ids), src, dst)
    want = np.arange(n, dtype=np.uint32)
    want[ids] = np.array(ids, np.uint32)[small]
    assert labels.tobytes() == want.tobytes()


def test_past_2_32_bytes(tmp_path):
    m = (1 << 32) // 12 + 1000  # about 4.3 GB
    n = m // 16
    b = (1 << 32) // 12  # the record that holds byte 2^32
    records = {b - 1: (5, n - 1), b: (n - 1, 7), b + 1: (7, 123456), 3: (9, 5), m - 1: (n - 2, 9)}
    p = os.path.join(sparse_dir(tmp_path), f"big_{os.getpid()}.graph500")
    sparse_graph500(p, m, records)
    try:
        check_sparse(p, m, records)
    finally:
        os.unlink(p)


def test_past_2_32_records(tmp_path):
    m = (1 << 32) + 8  # about 51.5 GB; n = 2^28.  The load refuses this file: its edge count does not fit u32 offsets
    n = m // 16
    assert n == 1 << 28
    records = {(1 << 32) - 2: (n - 1, 3), (1 << 32) - 1: (3, 77), 1 << 32: (77, 1 << 20), (1 << 32) + 1: (12, 13),
               m - 1: (n - 5, 1 << 20), 0: (13, n - 5)}
    p = os.path.join(sparse_dir(tmp_path), f"huge_{os.getpid()}.graph500")
    sparse_graph500(p, m, records)
    try:
        check_sparse(p, m, records)
    finally:
        os.unlink(p)


# ---- concurrency ---------------------------------------------------------------------------------------------
def test_two_threads_get_their_own_labels(rmat_files):
    jobs = {"g500": (rmat_files[16][F.Graph500], F.Graph500), "path": (None, F.EdgeList)}
    want = {"g500": gb.DiGraph.load(jobs["g500"][0]).wcc().components()}
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        path = write_text(os.path.join(d, "path.el"), "".join(f"{i} {i + 1}\n" for i in range(0, 200000, 2)))
        jobs["path"] = (path, F.EdgeList)
        want["path"] = gb.DiGraph.load(path, file_format=F.EdgeList).wcc().components()
        results, infos, errors = {}, {}, []

        def run(key):
            try:
                for _ in range(3):
                    results[key] = gb.wcc_file(*jobs[key]).components()
                    infos[key] = gb.wcc_file_info()
            except Exception as e:  # noqa: BLE001
                errors.append(e)
        threads = [threading.Thread(target=run, args=(k,)) for k in jobs]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    assert not errors, errors
    for key in jobs:
        assert results[key].tobytes() == want[key].tobytes(), key
        assert infos[key]["node_count"] == len(want[key])
