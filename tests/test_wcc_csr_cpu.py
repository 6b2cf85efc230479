"""CPU-side checks of graph_b200.wcc_csr (one-shot WCC of a host out-CSR): argument checks in Python, the C
symbol and its ctypes declaration, and — with no GPU — a loud failure instead of a CPU path."""
import ctypes

import numpy as np
import pytest

OFF = np.array([0, 1, 2, 2], np.uint32)
TGT = np.array([1, 0], np.uint32)


def test_missing_device_is_reported():
    import torch
    if torch.cuda.is_available():
        pytest.skip("this box has a GPU")
    import graph_b200 as gb
    with pytest.raises(gb.GraphB200Error, match="no CUDA device"):
        gb.wcc_csr(OFF, TGT)
    with pytest.raises(gb.GraphB200Error, match="no CUDA device"):
        gb.wcc_csr(np.zeros(4, np.uint32), np.zeros(0, np.uint32))


def test_arrays_must_be_contiguous_uint32():
    import graph_b200 as gb
    with pytest.raises(TypeError):
        gb.wcc_csr(OFF.astype(np.int64), TGT)
    with pytest.raises(TypeError):
        gb.wcc_csr(OFF, TGT.astype(np.int32))
    with pytest.raises(TypeError):
        gb.wcc_csr(OFF, np.array([1, 9, 0, 9], np.uint32)[::2])
    with pytest.raises(TypeError):
        gb.wcc_csr(OFF.tolist(), TGT)


def test_short_arrays_are_rejected():
    import graph_b200 as gb
    with pytest.raises(ValueError, match="targets hold 1 entries"):
        gb.wcc_csr(OFF, TGT[:1])
    with pytest.raises(ValueError, match="offsets need"):
        gb.wcc_csr(np.array([0], np.uint32), TGT)


def test_config_is_keyword_only():
    import graph_b200 as gb
    with pytest.raises(TypeError):
        gb.wcc_csr(OFF, TGT, 16384)


def test_symbol_is_exported_and_declared():
    import graph_b200 as gb
    import graph_b200._capi as capi
    lib = ctypes.CDLL(str(capi.LIB_PATH))
    assert hasattr(lib, "gb_wcc_csr_u32")
    res, args = capi.SIGNATURES["gb_wcc_csr_u32"]
    assert res is ctypes.c_int and len(args) == 6
    assert "wcc_csr" in gb.__all__
