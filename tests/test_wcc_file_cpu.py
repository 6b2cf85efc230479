"""CPU-side checks of graph_b200.wcc_file (one-pass WCC of a graph file): the C symbols and their ctypes
declarations, the Python argument checks, and — with no GPU — a loud failure instead of a CPU path."""
import ctypes

import pytest

GOLDEN_EL = "0 1\n1 2\n4 5\n"


@pytest.fixture
def el_file(tmp_path):
    p = tmp_path / "small.el"
    p.write_text(GOLDEN_EL)
    return p


def test_symbols_are_exported_and_declared():
    import graph_b200 as gb
    import graph_b200._capi as capi
    lib = ctypes.CDLL(str(capi.LIB_PATH))
    arity = {"gb_wcc_file_u32": 5, "gb_components_node_count": 2, "gb_components_copy": 2,
             "gb_components_free": 1, "gb_wcc_file_info": 1}
    for name, n in arity.items():
        assert hasattr(lib, name), name
        res, args = capi.SIGNATURES[name]
        assert res is ctypes.c_int and len(args) == n, name
    assert ctypes.sizeof(capi.WccFileStats) == 6 * 8 + 2 * 4
    assert "wcc_file" in gb.__all__ and "wcc_file_info" in gb.__all__


def test_path_and_format_are_checked(tmp_path, el_file):
    import graph_b200 as gb
    with pytest.raises(FileNotFoundError):
        gb.wcc_file(tmp_path / "missing.el", gb.FileFormat.EdgeList)
    with pytest.raises(TypeError):
        gb.wcc_file(None)
    with pytest.raises(TypeError):
        gb.wcc_file(el_file, "EdgeList")
    with pytest.raises(TypeError):
        gb.wcc_file(el_file, gb.Layout.Sorted)


def test_config_is_keyword_only(el_file):
    import graph_b200 as gb
    with pytest.raises(TypeError):
        gb.wcc_file(el_file, gb.FileFormat.EdgeList, 16384)
    with pytest.raises(TypeError):
        gb.wcc_file(el_file, gb.FileFormat.EdgeList, chunk_sizes=16384)


def test_missing_device_is_reported(el_file):
    import torch
    if torch.cuda.is_available():
        pytest.skip("this box has a GPU")
    import graph_b200 as gb
    for fmt in (gb.FileFormat.EdgeList, gb.FileFormat.Graph500, gb.FileFormat.Binary, gb.FileFormat.DotGraph):
        with pytest.raises(gb.GraphB200Error, match="no CUDA device"):
            gb.wcc_file(el_file, fmt, neighbor_rounds=1)
    assert set(gb.wcc_file_info().values()) == {0}


def test_null_arguments_are_rejected_by_the_library():
    import graph_b200 as gb
    from graph_b200._capi import GB_ERR_INVALID, WccConfig
    lib = gb.lib
    cfg = WccConfig(16384, 2, 1024)
    out = ctypes.c_void_p()
    assert lib.gb_wcc_file_u32(0, b"x", 0, ctypes.byref(cfg), None) == GB_ERR_INVALID
    assert lib.gb_wcc_file_u32(0, b"x", 0, None, ctypes.byref(out)) == GB_ERR_INVALID
    assert lib.gb_wcc_file_u32(0, None, 0, ctypes.byref(cfg), ctypes.byref(out)) == GB_ERR_INVALID
    assert lib.gb_wcc_file_u32(0, b"x", 9, ctypes.byref(cfg), ctypes.byref(out)) == GB_ERR_INVALID
    assert b"unknown file format 9" in lib.gb_last_error()
    assert lib.gb_components_free(None) == 0
    assert lib.gb_wcc_file_info(None) == GB_ERR_INVALID
