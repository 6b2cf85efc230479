"""The weighted undirected graph (UndirectedCsrGraph<u32, (), f32>) without a device: the numpy restatement of its
build (tests/weighted_undirected_restatement.py) pinned to the reference's fixtures, the new C ABI symbols, and the
argument checks of the Python API that run before any device call."""
import ctypes as C

import numpy as np
import pytest

import binary_restatement as br
import weighted_undirected_restatement as wu
from graph_b200 import _capi

LAYOUTS = [wu.UNSORTED, wu.SORTED, wu.DEDUPLICATED]
NEW_SYMBOLS = ["gb_graph_from_weighted_edges_u32", "gb_graph_from_device_weighted_edges_u32",
               "gb_graph_load_weighted_u32", "gb_to_undirected_weighted"]


def random_edges(seed, n, m):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, n, m, dtype=np.uint32)
    dst = rng.integers(0, n, m, dtype=np.uint32)
    dst[::7] = src[::7]  # self-loops
    src[1::5], dst[1::5] = src[::5][:len(src[1::5])], dst[::5][:len(dst[1::5])]  # parallel edges
    return src, dst, rng.standard_normal(m).astype(np.float32)


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("seed,n,m", [(0, 1, 5), (1, 6, 40), (2, 50, 300), (3, 9, 0)])
def test_vectorised_restatement_equals_the_row_by_row_one(seed, n, m, layout):
    src, dst, w = random_edges(seed, n, m)
    a = wu.build(src, dst, w, n, layout)
    b = wu.build_rows(src, dst, w, n, layout)
    for x, y in zip(a, b, strict=True):
        assert x.dtype == y.dtype and x.tobytes() == y.tobytes()


@pytest.mark.parametrize("layout", LAYOUTS)
def test_offsets_and_targets_do_not_depend_on_the_values(layout):
    src, dst, w = random_edges(4, 30, 200)
    a = wu.build(src, dst, w, 30, layout)
    b = wu.build(src, dst, np.zeros_like(w), 30, layout)
    assert a[0].tobytes() == b[0].tobytes() and a[1].tobytes() == b[1].tobytes()


def test_restatement_gives_the_test_wel_rows(golden_dir):
    rows = [line.split() for line in (golden_dir / "test.wel").read_text().splitlines() if line.strip()]
    src = np.array([int(r[0]) for r in rows], np.uint32)
    dst = np.array([int(r[1]) for r in rows], np.uint32)
    w = np.array([float(r[2]) for r in rows], np.float32)
    f = np.float32
    off, tgt, val = wu.build(src, dst, w, 5, wu.UNSORTED)
    assert wu.rows_of(off, tgt, val, 1) == [(2, f(0.3)), (3, f(0.4)), (0, f(0.1))]
    assert wu.rows_of(off, tgt, val, 2) == [(4, f(0.5)), (0, f(0.2)), (1, f(0.3))]
    off, tgt, val = wu.build(src, dst, w, 5, wu.SORTED)
    assert wu.rows_of(off, tgt, val, 1) == [(0, f(0.1)), (2, f(0.3)), (3, f(0.4))]
    assert wu.rows_of(off, tgt, val, 2) == [(0, f(0.2)), (1, f(0.3)), (4, f(0.5))]


@pytest.mark.parametrize("name", ["u32", "usize"])
def test_restatement_gives_the_golden_binary_rows(golden_dir, name):
    """The golden holds the Sorted CSR of the reference's serialize graph, and per-entry values that the two
    entries of an edge do not share: a loaded file keeps them as stored."""
    data = (golden_dir / f"binary_undirected_{name}_values.bin").read_bytes()
    (off, tgt, val), = br.read(data, 1, True)
    src = np.array([s for s, _ in br.EDGES], np.uint32)
    dst = np.array([t for _, t in br.EDGES], np.uint32)
    w_off, w_tgt, _ = wu.build(src, dst, np.ones(len(src), np.float32), 4, wu.SORTED)
    assert off.astype(np.uint32).tobytes() == w_off.tobytes()
    assert tgt.astype(np.uint32).tobytes() == w_tgt.tobytes()
    assert val.tobytes() == (np.arange(len(tgt), dtype=np.float32) * np.float32(0.25)).tobytes()
    assert br.write([(off, tgt, val)], name) == data


def test_new_abi_symbols_exist():
    lib = C.CDLL(str(_capi.LIB_PATH))
    for name in NEW_SYMBOLS:
        assert name in _capi.SIGNATURES
        assert hasattr(lib, name)


def test_abi_rejects_missing_weights_before_any_device_call():
    lib = _capi.lib
    src = np.array([0, 1], np.uint32)
    g = C.c_void_p()
    p = src.ctypes.data_as(C.c_void_p)
    assert lib.gb_graph_from_weighted_edges_u32(0, p, p, None, 2, 0, 0, C.byref(g)) == _capi.GB_ERR_INVALID
    assert b"weights" in lib.gb_last_error()
    assert lib.gb_graph_from_device_weighted_edges_u32(0, p, p, None, 2, 0, 0, None, C.byref(g)) == _capi.GB_ERR_INVALID
    assert lib.gb_to_undirected_weighted(None, 0, C.byref(g)) == _capi.GB_ERR_INVALID


def test_python_argument_checks(tmp_path):
    import graph_b200 as gb
    edges = np.array([[0, 1], [1, 2]], np.uint32)
    with pytest.raises(ValueError, match="one entry per edge"):
        gb.Graph.from_numpy(edges, weights=[1.0])
    with pytest.raises(ValueError, match="one entry per edge"):
        gb.Graph.from_numpy(edges, weights=[[1.0, 2.0]])
    with pytest.raises(ValueError, match="node values carries no edge weights"):
        gb.Graph.from_numpy(edges, weights=[1.0, 2.0], node_values=[0, 0, 0])
    p = tmp_path / "g.wel"
    p.write_text("0 1 0.5\n")
    with pytest.raises(ValueError, match="Graph500 files carry no edge values"):
        gb.Graph.load_weighted(p, file_format=gb.FileFormat.Graph500)
    with pytest.raises(ValueError, match="DotGraph files carry no edge values"):
        gb.Graph.load_weighted(p, file_format=gb.FileFormat.DotGraph)
