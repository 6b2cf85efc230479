"""The DotGraph restatement (tests/dotgraph_restatement.py) pinned to every assertion the reference makes about
node-labelled graphs, and to the malformed-file rules the library enforces on both of its readers."""
import json

import numpy as np
import pytest

import oracle
from conftest import GOLDEN
import dotgraph_restatement as dot

GOLD = json.loads((GOLDEN / "dotgraph_goldens.json").read_text())


def _undirected_sorted(g: dot.DotGraph):
    return oracle.csr_build(g.src, g.dst, len(g.labels), oracle.UNDIRECTED, oracle.SORTED)


def test_dotgraph_from_file():
    # dotgraph.rs:548-557 and :560-566
    g = dot.read((GOLDEN / "test.graph").read_bytes())
    assert len(g.labels) == 5 and len(g.src) == 6
    assert g.max_label == 2 and g.max_degree == 3
    assert g.max_label_frequency() == 2
    want = GOLD["test.graph"]
    assert g.labels.tolist() == want["labels"]  # builder.rs:384-388
    assert list(zip(g.src.tolist(), g.dst.tolist())) == [tuple(e) for e in want["edges"]]


def test_example_graph_with_n_tags():
    g = dot.read((GOLDEN / "example.graph").read_bytes())
    want = GOLD["example.graph"]
    assert g.labels.tolist() == want["labels"]
    assert list(zip(g.src.tolist(), g.dst.tolist())) == [tuple(e) for e in want["edges"]]
    assert g.max_label == want["max_label"] and g.max_degree == want["declared_max_degree"]


def test_label_stats():
    # dotgraph.rs:568-583
    g = dot.read((GOLDEN / "test.graph").read_bytes())
    off, tgt = _undirected_sorted(g)
    st = dot.label_stats(off, tgt, g.labels)
    assert st["max_degree"] == 3 and st["max_label"] == 2 and st["max_label_frequency"] == 2
    assert st["label_frequency"] == {0: 1, 1: 2, 2: 2}
    assert st["label_count"] == 3


def test_neighbor_label_frequency():
    # dotgraph.rs:585-611
    g = dot.read((GOLDEN / "test.graph").read_bytes())
    off, tgt = _undirected_sorted(g)
    maps = dot.frequency_maps(*dot.neighbor_label_frequencies(off, tgt, g.labels))
    want = [{int(k): v for k, v in m.items()} for m in GOLD["test.graph"]["neighbor_label_frequency"]]
    assert maps == want
    assert maps[0].get(0) is None and maps[3].get(0) is None and maps[4].get(0) is None


def test_node_label_index():
    # dotgraph.rs:613-624
    g = dot.read((GOLDEN / "test.graph").read_bytes())
    offsets, nodes = dot.node_label_index(g.labels)
    rows = [nodes[offsets[l]:offsets[l + 1]].tolist() for l in range(len(offsets) - 1)]
    assert rows == GOLD["test.graph"]["node_label_index"]


def test_self_loops_and_duplicates_count_as_listed():
    labels = [5, 7, 5]
    src, dst = np.array([0, 0, 0, 1], np.uint32), np.array([0, 1, 1, 2], np.uint32)
    off, tgt = oracle.csr_build(src, dst, 3, oracle.UNDIRECTED, oracle.SORTED)
    maps = dot.frequency_maps(*dot.neighbor_label_frequencies(off, tgt, labels))
    assert maps[0] == {5: 2, 7: 2}  # the self-loop twice, the duplicate edge twice
    assert maps[1] == {5: 3} and maps[2] == {7: 1}


def test_writer_round_trip():
    labels = [3, 0, 3, 9]
    edges = [(0, 1), (3, 2), (1, 1)]
    g = dot.read(dot.write(labels, edges, degrees=[1, 2, 1, 4], tag=b"n"))
    assert g.labels.tolist() == labels and g.max_degree == 4
    assert list(zip(g.src.tolist(), g.dst.tolist())) == edges


GOOD = dot.GOOD


@pytest.mark.parametrize("data, message", dot.MALFORMED)
def test_malformed_files(data, message):
    with pytest.raises(ValueError) as e:
        dot.read(data)
    assert str(e.value) == message


def test_accepted_variants():
    # the last line may lack its '\n'; lines after 1 + N + M are never read; the tag byte is not looked at;
    # the separator is any one byte; 2^32 - 1 fits
    assert dot.read(GOOD[:-1]).src.tolist() == [0]
    assert dot.read(GOOD + b"garbage\n\r\n").labels.tolist() == [4, 6]
    g = dot.read(b"t 2 1\n?\t0,4294967295;1\nxx1x6x1\n__0:1\n")
    assert g.labels.tolist() == [4294967295, 6] and g.src.tolist() == [0] and g.dst.tolist() == [1]
    assert dot.read(b"t 0 0\n").labels.tolist() == []
