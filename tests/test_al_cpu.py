"""CPU: the adjacency-list restatement (tests/al_restatement.py) pinned to every assertion of the reference's
adj_list.rs tests and its crate doc-test, to the two orders this library pins (undirected Unsorted interleaving,
Deduplicated self-loops), and the vectorised form against one-at-a-time add_edge."""
import numpy as np
import pytest

from al_restatement import DEDUPLICATED, SORTED, UNSORTED, ALGraph, FastAL, MissingNode, adjacency_list


def targets(g, node, which="out"):
    return [t for t, _ in g.rows(which)[node]]


def pairs(g, node, which="out"):
    return [(t, float(v)) for t, v in g.rows(which)[node]]


def test_from_edges_outgoing_incoming_undirected():
    # adj_list.rs:652-736 (rows compared after sorting by target, as the reference does)
    s, t, w = [0, 0, 1, 2], [1, 2, 0, 0], [42, 1337, 43, 1338]
    out = ALGraph(s, t, w, 3, UNSORTED)
    assert sorted(pairs(out, 0)) == [(1, 42), (2, 1337)]
    assert pairs(out, 1) == [(0, 43)]  # the value of edge (1, 0, 43)
    assert pairs(out, 2) == [(0, 1338)]
    assert sorted(pairs(out, 0, "in")) == [(1, 43), (2, 1338)]
    assert pairs(out, 1, "in") == [(0, 42)]
    assert pairs(out, 2, "in") == [(0, 1337)]
    und = ALGraph(s, t, w, 3, UNSORTED, directed=False)
    assert sorted(pairs(und, 0)) == [(1, 42), (1, 43), (2, 1337), (2, 1338)]
    assert sorted(pairs(und, 1)) == [(0, 42), (0, 43)]
    assert sorted(pairs(und, 2)) == [(0, 1337), (0, 1338)]


def test_from_edges_sorted_and_deduplicated():
    # adj_list.rs:738-781
    rows = adjacency_list([0, 0, 0, 1, 1, 1], [1, 3, 2, 3, 2, 0], None, 3, "out", SORTED)
    assert [t for t, _ in rows[0]] == [1, 2, 3] and [t for t, _ in rows[1]] == [0, 2, 3]
    rows = adjacency_list([0, 0, 0, 0, 0, 1, 1, 1, 1, 1, 1], [1, 3, 3, 2, 2, 3, 3, 2, 2, 0, 0], None, 3, "out",
                          DEDUPLICATED)
    assert [t for t, _ in rows[0]] == [1, 2, 3] and [t for t, _ in rows[1]] == [0, 2, 3]


def test_directed_and_undirected_graph():
    # adj_list.rs:783-796, 1023-1051
    g = ALGraph([0, 0, 1], [1, 2, 2], None, 0, SORTED)
    assert (g.node_count(), g.edge_count()) == (3, 3)
    assert len(g.out[0]) == 2 and targets(g, 0) == [1, 2]
    assert len(g.inc[2]) == 2 and targets(g, 2, "in") == [0, 1]
    u = ALGraph([0, 0, 1], [1, 2, 2], None, 0, SORTED, directed=False)
    assert (u.node_count(), u.edge_count()) == (3, 3)
    assert targets(u, 0) == [1, 2] and targets(u, 2) == [0, 1] and len(u.out[2]) == 2
    c = ALGraph([0, 1], [1, 0], None, 0, SORTED, directed=False)
    assert (c.node_count(), c.edge_count()) == (2, 2)
    assert targets(c, 0) == [1, 1] and targets(c, 1) == [0, 0]


@pytest.mark.parametrize("directed", [True, False])
def test_add_edge_unsorted_sorted_deduplicated(directed):
    # adj_list.rs:811-853 and 910-959
    g = ALGraph([0, 1], [2, 2], None, 0, UNSORTED, directed)
    assert targets(g, 0) == [2]
    g.add_edge(0, 1)
    assert targets(g, 0) == [2, 1]
    if not directed:
        assert targets(g, 1) == [2, 0]
    g.add_edge(0, 2)
    assert targets(g, 0) == [2, 1, 2]

    g = ALGraph([0, 1], [2, 2], None, 0, SORTED, directed)
    g.add_edge(0, 1)
    assert targets(g, 0) == [1, 2]
    if not directed:
        assert targets(g, 1) == [0, 2]
    g.add_edge(0, 1)
    assert targets(g, 0) == [1, 1, 2]

    g = ALGraph([0, 1, 1], [2, 2, 3], None, 0, DEDUPLICATED, directed)
    if not directed:
        assert targets(g, 1) == [2, 3]
    g.add_edge(0, 1)
    assert targets(g, 0) == [1, 2]
    if not directed:
        assert targets(g, 1) == [0, 2, 3]
    g.add_edge(0, 1)
    assert targets(g, 0) == [1, 2]
    g.add_edge(0, 3)
    assert targets(g, 0) == [1, 2, 3]


@pytest.mark.parametrize("directed", [True, False])
def test_add_edge_with_value_and_missing_node(directed):
    # adj_list.rs:855-892 and 961-1006
    g = ALGraph([0, 1], [2, 2], [4.2, 13.37], 0, UNSORTED, directed)
    f = np.float32
    assert pairs(g, 0) == [(2, f(4.2))]
    g.add_edge(0, 1, 19.84)
    assert pairs(g, 0) == [(2, f(4.2)), (1, f(19.84))]
    if not directed:
        assert pairs(g, 1) == [(2, f(13.37)), (0, f(19.84))]
    g.add_edge(0, 2, 1.23)
    assert pairs(g, 0) == [(2, f(4.2)), (1, f(19.84)), (2, f(1.23))]
    g = ALGraph([0, 1], [2, 2], None, 0, UNSORTED, directed)
    with pytest.raises(MissingNode) as e:
        g.add_edge(0, 3)
    assert e.value.node == "3" and str(e.value) == 'node "3" does not exist in the graph'


@pytest.mark.parametrize("directed", [True, False])
def test_add_edge_parallel_count(directed):
    # adj_list.rs:894-908, 1008-1022: four add_edge(0, 1) on three edges
    g = ALGraph([0, 0, 0], [1, 2, 3], None, 0, UNSORTED, directed)
    for _ in range(4):
        g.add_edge(0, 1)
    assert g.edge_count() == 7


def test_crate_doc_example():
    # lib.rs:234-255: a Unsorted DirectedALGraph from (0,1),(0,2),(1,2),(1,3),(2,3) takes add_edge(1, 0)
    g = ALGraph([0, 0, 1, 1, 2], [1, 2, 2, 3, 3], None, 0, UNSORTED)
    assert (g.node_count(), g.edge_count()) == (4, 5)
    assert (len(g.out[1]), len(g.inc[1])) == (2, 1)
    assert targets(g, 1) == [2, 3] and targets(g, 1, "in") == [0]
    g.add_edge(1, 0)
    assert g.edge_count() == 6
    assert targets(g, 1) == [2, 3, 0]


def test_undirected_unsorted_interleaves_and_dedup_keeps_self_loops():
    g = ALGraph([0, 1], [1, 2], None, 0, UNSORTED, directed=False)
    assert targets(g, 1) == [0, 2]  # the CSR twin's row 1 is [2, 0]
    g = ALGraph([3, 0], [3, 3], None, 0, UNSORTED, directed=False)
    assert targets(g, 3) == [3, 3, 0]
    g = ALGraph([3, 0], [3, 3], None, 0, DEDUPLICATED, directed=False)
    assert targets(g, 3) == [0, 3]
    g.add_edge(2, 2)
    assert targets(g, 2) == [2]  # an undirected self-loop adds u once
    g = ALGraph([3, 3, 0], [3, 3, 3], None, 0, DEDUPLICATED)
    assert targets(g, 3) == [3] and targets(g, 3, "in") == [0, 3]


@pytest.mark.parametrize("layout", [UNSORTED, SORTED, DEDUPLICATED])
@pytest.mark.parametrize("directed", [True, False])
@pytest.mark.parametrize("with_values", [False, True])
def test_vectorised_form_equals_add_edge(layout, directed, with_values):
    rng = np.random.default_rng(7 + layout + 3 * directed)
    n = 12
    s, t = rng.integers(0, n, 40), rng.integers(0, n, 40)
    w = rng.integers(0, 1000, 40).astype(np.float32) if with_values else None
    slow = ALGraph(s, t, w, n, layout, directed)
    fast = FastAL(s, t, w, n, layout, directed)
    for size in (0, 1, 7, 30):
        bs, bt = rng.integers(0, n, size), rng.integers(0, n, size)
        bw = rng.integers(0, 1000, size).astype(np.float32) if with_values else None
        slow.add_edges(bs, bt, bw)
        fast.add_edges(bs, bt, bw)
        for which in (("out", "in") if directed else ("out",)):
            a, b = slow.csr(which), fast.csr(which)
            assert (a[0] == b[0]).all() and (a[1] == b[1]).all()
            assert (a[2] is None) == (b[2] is None)
            if a[2] is not None:
                assert a[2].tobytes() == b[2].tobytes()
        assert slow.edge_count() == fast.edge_count()


def test_batch_is_all_or_nothing():
    g = FastAL([0, 1], [1, 2], None, 0, SORTED)
    before = g.csr()
    with pytest.raises(MissingNode) as e:
        g.add_edges([0, 5, 1], [1, 9, 7])
    assert e.value.node == "5"
    after = g.csr()
    assert all((x == y).all() for x, y in zip(before[:2], after[:2]))
