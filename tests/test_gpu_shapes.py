"""SSSP, WCC, triangle count and the CSR build on graphs that are not RMAT: zero and subnormal weights,
parallel edges, tiny bucket widths, empty and self-loop-only graphs, tied component sizes, cliques and
multigraphs, adjacency lists around the warp-walk threshold of k_tc, weighted Unsorted builds and ids past
2^16.  Bit-exact against the oracle."""
import math

import numpy as np
import pytest

import oracle

pytestmark = pytest.mark.gpu

FLT_MAX = np.finfo(np.float32).max


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


# ---- SSSP ----------------------------------------------------------------------------------------
def sssp_graph(kind, rng):
    """(src, dst, w, n, start) of one shape"""
    n = 1003
    src = rng.integers(0, n, 6 * n).astype(np.uint32)
    dst = rng.integers(0, n, 6 * n).astype(np.uint32)
    w = rng.random(len(src), dtype=np.float32)
    start = 0
    if kind == "zero_chains":          # long chains of zero-weight edges among positive ones
        chain = rng.permutation(n)[:n // 3].astype(np.uint32)
        src, dst = np.concatenate([src, chain[:-1]]), np.concatenate([dst, chain[1:]])
        w = np.concatenate([w, np.zeros(len(chain) - 1, np.float32)])
        w[rng.random(len(w)) < 0.05] = 0.0
        start = int(chain[0])
    elif kind == "parallel":           # every edge three times, with different weights
        src, dst = np.tile(src, 3), np.tile(dst, 3)
        w = np.concatenate([w, rng.random(len(w), dtype=np.float32), w * np.float32(0.5)])
    elif kind == "subnormal":          # weights of 1..1000 times the smallest subnormal, and some zeros
        w = (rng.integers(0, 1000, len(src)).astype(np.float32) * np.float32(1e-45)).astype(np.float32)
    elif kind == "sink_start":         # the start node has no out-edges
        start = int(src.max()) + 1 if src.max() + 1 < n else n - 1
        keep = src != start
        src, dst, w = src[keep], dst[keep], w[keep]
    elif kind == "unreachable":        # two halves, no edge from the first into the second
        h = n // 2
        src = rng.integers(0, h, 4 * n).astype(np.uint32)
        dst = rng.integers(0, h, 4 * n).astype(np.uint32)
        src = np.concatenate([src, rng.integers(h, n, 2 * n).astype(np.uint32)])
        dst = np.concatenate([dst, rng.integers(0, n, 2 * n).astype(np.uint32)])
        w = rng.random(len(src), dtype=np.float32)
    return src, dst, w, n, start


SSSP_CASES = [(k, d) for k in ("zero_chains", "parallel", "subnormal", "sink_start", "unreachable")
              for d in (0.1, 1e9)] + [("plain", d) for d in (1e-8, 1e-12, 1e-20, 1e-30, 1e-40)] + \
             [("subnormal", d) for d in (1e-44, 1e-40)] + [("zero_chains", 1e-30)]


@pytest.mark.parametrize("kind,delta", SSSP_CASES)
def test_sssp_shapes_bit_exact(gb, kind, delta):
    rng = np.random.default_rng(len(kind))
    src, dst, w, n, start = sssp_graph(kind, rng)
    delta = float(np.float32(delta))
    off, tgt, ww = oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED, w)
    want = oracle.sssp_bellman_ford(off, tgt, ww, start)
    if delta >= 0.1:     # the oracle keeps one bin per delta of distance
        assert (oracle.sssp_delta_stepping(off, tgt, ww, start, delta) == want).all()
    g = gb.DiGraph.from_numpy(np.stack([src, dst], 1), layout=gb.Layout.Sorted, weights=w, node_count=n)
    got = g.delta_stepping(start_node=start, delta=delta).distances()
    assert got.tobytes() == want.tobytes(), (kind, delta)
    if kind == "sink_start":
        assert (got == FLT_MAX).sum() == n - 1 and got[start] == 0.0
    if kind == "unreachable":
        assert (got[n // 2:] == FLT_MAX).all()
    if delta >= 1e9:
        assert want[want < FLT_MAX].max() < delta          # a single bucket


# ---- WCC -----------------------------------------------------------------------------------------
def wcc_graph(kind):
    n = 4001
    if kind == "no_edges":
        src = dst = np.zeros(0, np.uint32)
    elif kind == "self_loops":
        src = dst = np.arange(0, n, 3, dtype=np.uint32)
    elif kind == "pairs":              # n // 2 components of two vertices, far-apart ids
        a = np.arange(n // 2, dtype=np.uint32)
        src, dst = a, (n - 1 - a).astype(np.uint32)
    elif kind == "tied_giants":        # the two largest components have exactly the same size
        rng = np.random.default_rng(3)
        ids = rng.permutation(n).astype(np.uint32)
        c1, c2 = ids[:1500], ids[1500:3000]
        src = np.concatenate([c1[:-1], c2[:-1], ids[3000:3500:2]])
        dst = np.concatenate([c1[1:], c2[1:], ids[3001:3501:2]])
    elif kind == "giant_at_top":       # the giant component holds the highest ids; its minimum is n - 3000
        rng = np.random.default_rng(4)
        top = np.arange(n - 3000, n, dtype=np.uint32)
        src = rng.permutation(top)
        dst = np.roll(src, 1)
    return src.astype(np.uint32), dst.astype(np.uint32), n


@pytest.mark.parametrize("kind", ["no_edges", "self_loops", "pairs", "tied_giants", "giant_at_top"])
def test_wcc_shapes_bit_exact(gb, kind):
    src, dst, n = wcc_graph(kind)
    out = oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED)
    inc = oracle.csr_build(src, dst, n, oracle.INCOMING, oracle.SORTED)
    want = oracle.wcc_min_label(out[0], out[1])
    g = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    for kw in ({}, {"neighbor_rounds": 0}, {"neighbor_rounds": 1}, {"neighbor_rounds": 100}):
        assert (g.wcc(**kw).components() == want).all(), (kind, kw)
    if kind == "tied_giants":
        sizes = np.sort(np.unique(want, return_counts=True)[1])
        assert sizes[-1] == sizes[-2] == 1500


# ---- triangle count ------------------------------------------------------------------------------
def clique(k, base=0):
    a, b = np.triu_indices(k, 1)
    return (a + base).astype(np.uint32), (b + base).astype(np.uint32)


def list_pairs(lengths=(15, 16, 17, 33)):
    """for every (Lu, Lv): an edge u-v (v < u) whose item in k_tc cuts N(u) and N(v) to Lu and Lv entries: u
    has Lu neighbours (v among them), v has Lv besides u, about half of them shared.  The neighbours have ids
    below both endpoints, so every one counts toward the `<= v` prefixes."""
    src, dst, nxt = [], [], 0
    for lu in lengths:
        for lv in lengths:
            shared = min(lu - 1, lv) // 2
            common = list(range(nxt, nxt + shared))
            k = nxt + shared
            only_u = list(range(k, k + lu - 1 - shared))
            k += len(only_u)
            only_v = list(range(k, k + lv - shared))
            k += len(only_v)
            v, u = k, k + 1
            for x in common + only_u:
                src.append(u)
                dst.append(x)
            for x in common + only_v:
                src.append(v)
                dst.append(x)
            src.append(u)
            dst.append(v)
            for i in range(0, len(common) - 1, 2):     # a few edges among the shared neighbours too
                src.append(common[i])
                dst.append(common[i + 1])
            nxt = u + 1
    return np.array(src, np.uint32), np.array(dst, np.uint32), nxt


def tc_graph(kind):
    if kind == "K200":
        s, d = clique(200)
        return s, d, 200, oracle.SORTED
    if kind == "K60_multi":            # every edge twice and a self loop on every vertex: the multigraph sum,
        s, d = clique(60)              # with short lists of unequal length (walked lane by lane) beside it
        ps, pd, pn = list_pairs()
        s, d = np.concatenate([s, ps + 60]), np.concatenate([d, pd + 60])
        loops = np.arange(60 + pn, dtype=np.uint32)
        return np.concatenate([s, d, loops]), np.concatenate([d, s, loops]), 60 + pn, oracle.SORTED
    s, d, n = list_pairs()
    return s, d, n, oracle.SORTED


@pytest.mark.parametrize("kind", ["K200", "K60_multi", "list_lengths"])
def test_triangle_count_shapes_bit_exact(gb, kind):
    src, dst, n, layout = tc_graph(kind)
    off, tgt = oracle.csr_build(src, dst, n, oracle.UNDIRECTED, layout)
    want = oracle.triangle_count(off, tgt, threads=0)
    if kind == "K200":
        assert want == math.comb(200, 3)
    if kind == "list_lengths":
        deg = np.diff(off.astype(np.int64))
        assert {15, 16, 17, 33} <= set(deg.tolist())
    ug = gb.Graph.from_csr(off, tgt)
    assert ug.global_triangle_count().triangles == want, kind
    noff, ntgt, _ = oracle.make_degree_ordered(off, tgt)
    ug.make_degree_ordered()
    assert ug.global_triangle_count().triangles == oracle.triangle_count(noff, ntgt, threads=0), kind
    # the same through the device build from the edge list
    ue = gb.Graph.from_numpy(np.stack([src, dst], 1), layout=gb.Layout.Sorted, node_count=n)
    assert ue.global_triangle_count().triangles == want, kind


# ---- CSR build -----------------------------------------------------------------------------------
def test_unsorted_weighted_build_matches_oracle(gb):
    rng = np.random.default_rng(8)
    n = 3001
    src = rng.integers(0, n, 40000).astype(np.uint32)
    dst = rng.integers(0, n, 40000).astype(np.uint32)
    w = rng.random(len(src), dtype=np.float32)
    g = gb.DiGraph.from_numpy(np.stack([src, dst], 1), layout=gb.Layout.Unsorted, weights=w, node_count=n)
    off, tgt = g.csr("out")
    woff, wtgt, ww = oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.UNSORTED, w)
    assert (off == woff).all() and (tgt == wtgt).all()
    assert g.out_weights().tobytes() == ww.tobytes()        # each weight stays with its target, in row order


def test_ids_past_2_16(gb):
    n = (1 << 16) + 1
    hi = n - 1
    e = np.array([[0, hi], [hi, 0], [hi, hi], [0, 0], [hi, 1], [1, hi], [hi, 0]], np.uint32)
    src, dst = e[:, 0].copy(), e[:, 1].copy()
    for layout, lo in (("Unsorted", oracle.UNSORTED), ("Sorted", oracle.SORTED),
                       ("Deduplicated", oracle.DEDUPLICATED)):
        g = gb.DiGraph.from_numpy(e, layout=getattr(gb.Layout, layout), node_count=n)
        for which, direction in (("out", oracle.OUTGOING), ("in", oracle.INCOMING)):
            off, tgt = g.csr(which)
            woff, wtgt = oracle.csr_build(src, dst, n, direction, lo)
            assert (off == woff).all() and (tgt == wtgt).all(), (layout, which)
        ug = gb.Graph.from_numpy(e, layout=getattr(gb.Layout, layout), node_count=n)
        off, tgt = ug.csr()
        woff, wtgt = oracle.csr_build(src, dst, n, oracle.UNDIRECTED, lo)
        assert (off == woff).all() and (tgt == wtgt).all(), layout
