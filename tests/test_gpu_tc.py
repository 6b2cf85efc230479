"""gb_triangle_count on the H100 against the oracle, on the CSR read back from the device: every fixture of
tc_fixtures.py through Graph.from_csr (the exact CSR) and, where it is an edge list, through from_numpy in
its own layout and in the default one; RMAT, Graph.load and DiGraph.to_undirected with the default Unsorted
layout; an Unsorted graph after make_degree_ordered; a total above 2^32; and the launches of each call:
one kernel on rows known to be sorted, the row-order check at most once per CSR."""
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
import tc_fixtures as fx

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import tc_model as tm  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


def run(g):
    return g.global_triangle_count().triangles, g.last_timing()["kernel_launches"]


def path_launches(rows_sorted: bool) -> int:
    return 1 if rows_sorted else 2         # k_tc, or k_tc_cut + k_tc_list


def check(g, known_sorted: bool, label):
    """the count is the oracle's on g's CSR, twice; the row-order check runs on the first call only, and
    not at all when the build wrote sorted rows"""
    off, tgt = (a.copy() for a in g.csr())
    want = oracle.triangle_count(off, tgt, threads=0)
    path = path_launches(tm.rows_sorted(off, tgt))
    assert not known_sorted or tm.rows_sorted(off, tgt), label
    assert run(g) == (want, path + (0 if known_sorted else 1)), label
    assert run(g) == (want, path), label
    return want


@pytest.mark.parametrize("name", sorted(fx.FIXTURES))
def test_fixture_matches_oracle(gb, name):
    f = fx.FIXTURES[name]()
    g = gb.Graph.from_csr(f.off, f.tgt)
    off, tgt = g.csr()
    assert (off == f.off).all() and (tgt == f.tgt).all(), name
    want = oracle.triangle_count(f.off, f.tgt, threads=0)
    assert run(g) == (want, 1 + path_launches(f.sorted_rows)), name
    assert run(g) == (want, path_launches(f.sorted_rows)), name
    if f.edges is None:
        return
    e = gb.Graph.from_numpy(f.edges, layout=getattr(gb.Layout, f.layout), node_count=f.n)
    off, tgt = e.csr()
    assert (off == f.off).all() and (tgt == f.tgt).all(), name
    assert check(e, f.layout == "Sorted", name) == want
    # the default layout keeps every row in edge-list order
    check(gb.Graph.from_numpy(f.edges, node_count=f.n), False, (name, "default layout"))


@pytest.mark.parametrize("scale", [8, 10, 13])
def test_rmat_unsorted(gb, scale):
    g = gb.Graph.rmat(scale, seed=42, layout=gb.Layout.Unsorted)
    off, tgt = g.csr()
    assert not tm.rows_sorted(off, tgt)
    check(g, False, scale)


@pytest.mark.parametrize("layout", ["Sorted", "Deduplicated"])
def test_sorted_builds_launch_one_kernel(gb, layout):
    g = gb.Graph.rmat(10, seed=42, layout=getattr(gb.Layout, layout))
    check(g, True, layout)
    d = gb.DiGraph.rmat(9, seed=3, layout=gb.Layout.Unsorted)
    check(d.to_undirected(getattr(gb.Layout, layout)), True, (layout, "to_undirected"))


def test_load_default_layout(gb, golden_dir):
    g = gb.Graph.load(str(golden_dir / "scale_8.graph500"))
    assert check(g, False, "scale_8") == 26     # the Sorted build of the same file has 256533
    # test.el has no triangle in either layout: this only takes the text path through the row-order check
    g = gb.Graph.load(str(golden_dir / "test.el"), file_format=gb.FileFormat.EdgeList)
    assert check(g, False, "test.el") == 0


def test_to_undirected_default_layout(gb, scale8_edges):
    src, dst, n = scale8_edges
    d = gb.DiGraph.from_numpy(np.stack([src, dst], 1), node_count=n)
    assert check(d.to_undirected(), False, "to_undirected") == 68


def test_degree_ordered_unsorted_graph(gb):
    g = gb.Graph.rmat(10, seed=42, layout=gb.Layout.Unsorted)
    off, tgt = (a.copy() for a in g.csr())
    g.make_degree_ordered()
    noff, ntgt = g.csr()
    woff, wtgt, _ = oracle.make_degree_ordered(off, tgt)
    assert (noff == woff).all() and (ntgt == wtgt).all()
    assert check(g, True, "degree ordered") == oracle.triangle_count(woff, wtgt, threads=0)


def test_total_above_2_32(gb):
    n, reps = 1200, 4
    s, d = fx.multi_clique_edges(n, reps)
    want = fx.multi_clique_count(n, reps)
    assert want == 4_596_486_400
    g = gb.Graph.from_numpy(np.stack([s, d], 1), layout=gb.Layout.Sorted, node_count=n)
    assert run(g) == (want, 1)
    off, tgt = g.csr()
    assert (np.diff(off.astype(np.int64)) == reps * (n - 1)).all()
    h = gb.Graph.from_csr(off, tgt)
    assert run(h) == (want, 2)
    assert run(h) == (want, 1)
