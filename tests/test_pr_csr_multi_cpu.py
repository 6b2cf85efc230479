"""CPU-side checks of the multi-GPU one-shot PageRank (gb_page_rank_csr_multi_u32 / gb_pr_shards_csr_u32 /
graph_b200.Comm.page_rank_csr): the part split (pr_split, graph_b200/csrc/csr_split.h) compiled with g++ and
checked on random, tiny, hub-heavy, all-empty and non-monotone offsets for 1..8 parts, the C symbols with their ctypes
declarations and header lines, and the Python argument checks, which raise before any device is touched."""
import ctypes
import subprocess
from pathlib import Path

import numpy as np
import pytest

ROOT = Path(__file__).resolve().parent.parent


def test_split_tiles_rows_and_edges(tmp_path):
    exe = tmp_path / "pr_split_check"
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'graph_b200' / 'csrc'}",
           str(ROOT / "tests" / "cpp" / "pr_split_check.cpp"), "-o", str(exe)]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "pr_split ok" in r.stdout, r.stdout + r.stderr


def test_symbols_are_exported_and_declared():
    import graph_b200 as gb
    import graph_b200._capi as capi
    lib = ctypes.CDLL(str(capi.LIB_PATH))
    header = (ROOT / "include" / "graph_b200.h").read_text()
    for name, nargs, decl in (
            ("gb_page_rank_csr_multi_u32", 9, "gb_status gb_page_rank_csr_multi_u32(gb_comm* comm, uint32_t node_count,"),
            ("gb_pr_shards_csr_u32", 7, "gb_status gb_pr_shards_csr_u32(gb_comm* comm, uint32_t ranks_per_device,")):
        assert hasattr(lib, name)
        res, args = capi.SIGNATURES[name]
        assert res is ctypes.c_int and len(args) == nargs
        assert decl in header
    assert "page_rank_csr_multi(" in (ROOT / "include" / "graph_b200.hpp").read_text()
    assert callable(gb.Comm.page_rank_csr) and callable(gb.Comm.pr_shards_csr)


class _NoComm:
    """Stands in for a Comm: the argument checks must raise before the C library is called."""
    devices = [0]
    _c = None


@pytest.mark.parametrize("method", ["page_rank_csr", "pr_shards_csr"])
def test_python_argument_checks(method):
    import graph_b200 as gb
    call = getattr(gb.Comm, method)
    io = np.array([0, 1, 2, 2], np.uint32)
    it = np.array([1, 0], np.uint32)
    oo = np.array([0, 1, 1, 2], np.uint32)
    c = _NoComm()
    with pytest.raises(TypeError):
        call(c, io.astype(np.int64), it, oo)
    with pytest.raises(TypeError):
        call(c, io, it, oo.astype(np.int32))
    with pytest.raises(TypeError):  # not contiguous
        call(c, io, np.arange(4, dtype=np.uint32)[::2], oo)
    with pytest.raises(ValueError, match="targets hold 1 entries"):
        call(c, io, it[:1], oo)
    with pytest.raises(ValueError, match="same length"):
        call(c, io, it, oo[:-1])
    with pytest.raises(TypeError):
        call(c, io, it, oo, 20)
