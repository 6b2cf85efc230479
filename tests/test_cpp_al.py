"""The C++ mirror of the adjacency-list graphs (include/graph_b200.hpp): the reference's adj_list.rs unit tests and
crate doc-test through GraphBuilder::build_directed_al / build_undirected_al, driven by tests/cpp/al_graph.cpp.  It
compiles and links on the CPU; on a GPU it runs its checks."""
import subprocess
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def build(tmp_path):
    exe = tmp_path / "al_graph"
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-pthread", f"-I{ROOT / 'include'}",
           str(ROOT / "tests" / "cpp" / "al_graph.cpp"), "-o", str(exe), f"-L{ROOT / 'graph_b200'}",
           "-lgraph_b200", f"-Wl,-rpath,{ROOT / 'graph_b200'}"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return exe


def test_al_graph_program_compiles_and_links(tmp_path):
    assert build(tmp_path).exists()


@pytest.mark.gpu
def test_al_graph_program(tmp_path):
    exe = build(tmp_path)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "al_graph ok" in r.stdout
