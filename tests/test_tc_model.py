"""The CPU replay of gb_triangle_count (tools/tc_model.py) on the fixtures of test_gpu_tc.py: its count is the
oracle's on every one, every fixture still reaches the k_tc class (direction, short/long, walk length,
repeated run) it is named for, and the fixtures meant for the list-order path hold a descent inside a row
while the others do not.  A change of TC_SHORT or of the direction rule that moves a fixture off its path
fails here, without a GPU."""
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
import tc_fixtures as fx

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import tc_model as tm  # noqa: E402


@pytest.fixture(scope="module", params=sorted(fx.FIXTURES))
def case(request):
    return request.param, fx.FIXTURES[request.param]()


def test_model_count_is_the_oracle_count(case):
    name, f = case
    assert tm.triangle_count(f.off, f.tgt) == oracle.triangle_count(f.off, f.tgt), name


def test_fixture_reaches_its_class(case):
    name, f = case
    r = tm.replay_sorted(f.off, f.tgt)
    assert f.walks <= set(r.walks), (name, sorted(r.walks))
    assert f.classes <= set(r.classes), (name, sorted(r.classes))
    assert f.runs <= set(r.runs), (name, sorted(r.runs))
    assert (r.crossings > 0) == f.crossing or not f.sorted_rows, (name, r.crossings)


def test_row_order_is_what_the_fixture_claims(case):
    name, f = case
    assert tm.rows_sorted(f.off, f.tgt) == f.sorted_rows, name
    if f.edges is not None:     # the CSR is the oracle's build of the edge list
        off, tgt = oracle.csr_build(f.edges[:, 0].copy(), f.edges[:, 1].copy(), f.n, oracle.UNDIRECTED,
                                    fx._LAYOUT[f.layout])
        assert (off == f.off).all() and (tgt == f.tgt).all(), name


def test_walk_matrix_names():
    for d in ("by_u", "by_v"):
        for k in fx.WALKS:
            f = fx.FIXTURES[f"walk_{d}_{k}"]()
            assert f.walks == {(d, k)} and f.classes == {(d, "short" if k <= 16 else "long")}


def test_repeated_runs_cross_the_warp_step_where_named():
    cross = {a: fx.FIXTURES[f"run_by_u_at_{a}"]().crossing for a in (30, 31, 32, 33)}
    assert cross == {30: True, 31: True, 32: False, 33: False}
    assert fx.FIXTURES["run_by_u_40"]().runs == {(10, 40)}      # longer than one step


def test_list_order_fixtures_would_fail_on_k_tc_alone():
    """k_tc's binary searches on these rows give another number than the reference loop"""
    for name in ("inversion_last_row", "inversion_row_of_2", "shuffled_rows", "descending_rows",
                 "rmat8_unsorted", "rmat10_unsorted"):
        f = fx.FIXTURES[name]()
        assert tm.replay_sorted(f.off, f.tgt).count != oracle.triangle_count(f.off, f.tgt), name


def test_boundary_drops_are_not_inversions():
    f = fx.FIXTURES["boundary_drops"]()
    ends = f.off[1:-1].astype(np.int64)
    assert (np.diff(f.off.astype(np.int64)) > 0).all()
    assert (f.tgt[ends - 1] > f.tgt[ends]).all()                # a drop at every row boundary
    assert tm.rows_sorted(f.off, f.tgt)
    assert [len(r) for r in fx.rows_of(f)][6] == 2 and fx.rows_of(f)[12][:2] == [0, 1]


def test_row_search_fixtures():
    f = fx.FIXTURES["empty_rows"]()
    deg = np.diff(f.off.astype(np.int64))
    assert (deg[:24] == 0).all() and (deg[41:] == 0).all()
    f = fx.FIXTURES["all_in_last_row"]()
    assert f.off[-2] == 0 and f.off[-1] == len(f.tgt)
    f = fx.FIXTURES["single_vertex"]()
    assert f.n == 1 and f.tgt.tolist() == [0] * 6
    assert len(fx.FIXTURES["straddle"]().tgt) % 32 != 0


@pytest.mark.parametrize("n,reps", [(30, 3), (41, 4), (12, 1), (9, 2)])
def test_multi_clique_closed_form(n, reps):
    s, d = fx.multi_clique_edges(n, reps)
    off, tgt = oracle.csr_build(s, d, n, oracle.UNDIRECTED, oracle.SORTED)
    want = fx.multi_clique_count(n, reps)
    assert oracle.triangle_count(off, tgt) == want
    assert tm.triangle_count(off, tgt) == want


def test_multi_clique_1200_passes_2_32():
    assert fx.multi_clique_count(1200, 4) == 4_596_486_400 > 2 ** 32


def test_list_pairs_reach_the_lengths_around_tc_short():
    """test_gpu_shapes.py's list_lengths graph: the shared and private neighbours are below both endpoints,
    so the items walk 15, 16, 17 and 33 entries"""
    from test_gpu_shapes import tc_graph
    src, dst, n, layout = tc_graph("list_lengths")
    off, tgt = oracle.csr_build(src, dst, n, oracle.UNDIRECTED, layout)
    r = tm.replay_sorted(off, tgt)
    assert {15, 16, 17, 33} <= {w for _, w in r.walks}, sorted(r.walks)
    assert set(r.classes) == {("by_u", "short"), ("by_u", "long"), ("by_v", "short"), ("by_v", "long")}
    assert r.count == oracle.triangle_count(off, tgt)
