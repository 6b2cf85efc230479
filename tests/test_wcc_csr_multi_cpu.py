"""CPU-side checks of the multi-GPU one-shot WCC (gb_wcc_csr_multi_u32 / graph_b200.Comm.wcc_csr): the part
split (wcc_split, graph_b200/csrc/csr_split.h) compiled with g++ and checked on random, tiny, hub, sparse and
non-monotone offsets, and the C symbol with its ctypes declaration."""
import ctypes
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_split_partitions_edges_and_tiles_rows(tmp_path):
    exe = tmp_path / "wcc_split_check"
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'graph_b200' / 'csrc'}",
           str(ROOT / "tests" / "cpp" / "wcc_split_check.cpp"), "-o", str(exe)]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "wcc_split ok" in r.stdout, r.stdout + r.stderr


def test_symbol_is_exported_and_declared():
    import graph_b200 as gb
    import graph_b200._capi as capi
    lib = ctypes.CDLL(str(capi.LIB_PATH))
    assert hasattr(lib, "gb_wcc_csr_multi_u32")
    res, args = capi.SIGNATURES["gb_wcc_csr_multi_u32"]
    assert res is ctypes.c_int and len(args) == 6
    assert callable(gb.Comm.wcc_csr)
    header = (ROOT / "include" / "graph_b200.h").read_text()
    assert "gb_status gb_wcc_csr_multi_u32(gb_comm* comm, uint32_t node_count," in header
