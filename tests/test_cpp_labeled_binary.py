"""The C++ mirror of labelled binary files (include/graph_b200.hpp): CsrGraphBase::serialize_labeled and
GraphBuilder::build_directed_labeled / build_undirected_labeled, driven through tests/cpp/labeled_binary.cpp.  It
compiles and links on the CPU; on a GPU it runs its checks."""
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def build(tmp_path):
    exe = tmp_path / "labeled_binary"
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'include'}",
           str(ROOT / "tests" / "cpp" / "labeled_binary.cpp"), "-o", str(exe), f"-L{ROOT / 'graph_b200'}",
           "-lgraph_b200", f"-Wl,-rpath,{ROOT / 'graph_b200'}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return exe


def test_labeled_binary_program_compiles_and_links(tmp_path):
    assert build(tmp_path).exists()


@pytest.mark.gpu
def test_labeled_binary_program(tmp_path):
    exe = build(tmp_path)
    scratch = tmp_path / "files"
    scratch.mkdir()
    r = subprocess.run([str(exe), str(ROOT / "tests" / "golden"), str(scratch)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "labeled_binary ok" in r.stdout
