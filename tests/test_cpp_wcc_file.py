"""The C++ mirror of the one-pass file WCC (include/graph_b200.hpp: graph::prelude::wcc_file), driven through
tests/cpp/wcc_file.cpp.  It compiles and links on the CPU; on a GPU it runs its checks."""
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def build(tmp_path):
    exe = tmp_path / "wcc_file"
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'include'}",
           str(ROOT / "tests" / "cpp" / "wcc_file.cpp"), "-o", str(exe), f"-L{ROOT / 'graph_b200'}",
           "-lgraph_b200", f"-Wl,-rpath,{ROOT / 'graph_b200'}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return exe


def test_wcc_file_program_compiles_and_links(tmp_path):
    assert build(tmp_path).exists()


@pytest.mark.gpu
def test_wcc_file_program(tmp_path):
    exe = build(tmp_path)
    r = subprocess.run([str(exe), str(ROOT / "tests" / "golden")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "wcc_file ok" in r.stdout
