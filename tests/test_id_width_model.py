"""CPU checks behind test_gpu_id_width.py.

1. The expansion rule of id_width_fixtures: on the same fixtures scaled down (T placed in n of about 5000, around
   a stand-in for 2^31), the oracle on the whole graph equals the oracle on the compacted graph, mapped back,
   plus the closed form for the untouched ids.  The GPU tests rely on this rule at n = 2^31 + 1 and 2^32 - 1,
   where the oracle cannot run on the whole graph.
2. A scan of the kernels a graph with ids past 2^31 reaches: every grid- or warp-stride loop counts in 64 bits
   and stops at `< bound`.  A 32-bit counter bounded by a node count wraps below n once n is within one stride
   of 2^32 and never ends, and a `<= n` loop never ends at n = 2^32 - 1; neither can be run to show it.
"""
import re
from pathlib import Path

import numpy as np
import pytest

import oracle
from id_width_fixtures import (Fixture, expand_degree_order, expand_labels, expand_offsets,
                               in_degree_partition_ranges, mixed)

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "graph_b200" / "csrc"

# (n, half): the boundary one below, at and above the middle, and n just past it (the N1 shape)
SCALED = [(5000, 2048), (4099, 2048), (2049, 2048), (4096, 2048)]


def _fixtures():
    return [pytest.param(mixed(n, half, weighted=w), id=f"{'weighted' if w else 'mixed'}-n{n}-h{half}")
            for n, half in SCALED for w in (False, True)]


def _expand_csr(fx: Fixture, off_c, tgt_c):
    return expand_offsets(off_c, fx.T, fx.n), fx.ids(tgt_c)


@pytest.mark.parametrize("fx", _fixtures())
@pytest.mark.parametrize("layout", [oracle.UNSORTED, oracle.SORTED, oracle.DEDUPLICATED])
@pytest.mark.parametrize("direction", [oracle.OUTGOING, oracle.INCOMING, oracle.UNDIRECTED])
def test_csr_build_expands(fx, layout, direction):
    w = fx.weights if direction != oracle.UNDIRECTED else None
    full = oracle.csr_build(fx.src, fx.dst, fx.n, direction, layout, w)
    comp = oracle.csr_build(fx.csrc, fx.cdst, fx.k, direction, layout, w)
    off, tgt = _expand_csr(fx, comp[0], comp[1])
    np.testing.assert_array_equal(full[0], off)
    np.testing.assert_array_equal(full[1], tgt)
    if w is not None:
        np.testing.assert_array_equal(full[2], comp[2])


@pytest.mark.parametrize("fx", _fixtures())
def test_wcc_min_label_expands(fx):
    full_off, full_tgt = oracle.csr_build(fx.src, fx.dst, fx.n, oracle.OUTGOING, oracle.SORTED)
    off_c, tgt_c = oracle.csr_build(fx.csrc, fx.cdst, fx.k, oracle.OUTGOING, oracle.SORTED)
    want = oracle.wcc_min_label(full_off, full_tgt)
    np.testing.assert_array_equal(want, expand_labels(oracle.wcc_min_label(off_c, tgt_c), fx.T, fx.n))
    # some component has its minimum below half and another member at or above it
    lab = want[fx.T.astype(np.int64)]
    assert any((lab == l).any() and l < fx.half and (fx.T[lab == l] >= fx.half).any() for l in np.unique(lab))


@pytest.mark.parametrize("fx", _fixtures())
@pytest.mark.parametrize("layout", [oracle.UNSORTED, oracle.SORTED, oracle.DEDUPLICATED])
def test_triangle_count_expands(fx, layout):
    full = oracle.csr_build(fx.src, fx.dst, fx.n, oracle.UNDIRECTED, layout)
    comp = oracle.csr_build(fx.csrc, fx.cdst, fx.k, oracle.UNDIRECTED, layout)
    want = oracle.triangle_count(*full)
    assert want >= 1  # the triangle of the three highest ids, at least
    assert oracle.triangle_count(*comp) == want


@pytest.mark.parametrize("fx", _fixtures())
@pytest.mark.parametrize("layout", [oracle.SORTED, oracle.DEDUPLICATED])
def test_make_degree_ordered_expands(fx, layout):
    full = oracle.csr_build(fx.src, fx.dst, fx.n, oracle.UNDIRECTED, layout)
    comp = oracle.csr_build(fx.csrc, fx.cdst, fx.k, oracle.UNDIRECTED, layout)
    assert (np.diff(comp[0].astype(np.int64)) > 0).all(), "every touched id needs a positive degree"
    noff, ntgt, nid = oracle.make_degree_ordered(*full)
    eoff, etgt, enid = expand_degree_order(*oracle.make_degree_ordered(*comp), fx.T, fx.n)
    np.testing.assert_array_equal(noff, eoff)
    np.testing.assert_array_equal(ntgt, etgt)
    np.testing.assert_array_equal(nid, enid)


@pytest.mark.parametrize("fx", _fixtures())
@pytest.mark.parametrize("parts", [1, 2, 3, 7, 64])
def test_in_degree_partition_expands(fx, parts):
    full_in = oracle.csr_build(fx.src, fx.dst, fx.n, oracle.INCOMING, oracle.SORTED)[0]
    comp_in = oracle.csr_build(fx.csrc, fx.cdst, fx.k, oracle.INCOMING, oracle.SORTED)[0]
    got = in_degree_partition_ranges(comp_in, fx.T, fx.n, parts)
    want = oracle.in_degree_partition(full_in, parts)
    np.testing.assert_array_equal(got[:len(want)], want)
    assert (got[len(want):] == fx.n).all()


def test_fixtures_touch_both_sides_of_half():
    from id_width_fixtures import HALF, N1, N2
    for n in (N1, N2):
        fx = mixed(n, HALF)
        T = set(int(t) for t in fx.T)
        assert {0, HALF - 1, HALF, n - 2, n - 1} <= T
        assert int(fx.T.max()) == n - 1
    fx = mixed(N2, HALF)
    T = set(int(t) for t in fx.T)
    assert HALF + 1 in T
    # ids with bit 31 set whose low bits are those of touched ids below 2^31
    assert sum(1 for t in T if t >= HALF and (t - HALF) in T) >= 4
    hi = sorted(t for t in T if t >= HALF)
    clique = hi[:4]
    pairs = {(int(s), int(d)) for s, d in zip(fx.src, fx.dst)}
    assert all((u, v) in pairs for i, u in enumerate(clique) for v in clique[i + 1:])


# ---- loop counters -----------------------------------------------------------------------------------
# The files whose kernels a graph with ids past 2^31 reaches.  pagerank.cu, pr_layout.cu, pr_csr.cu and multi.cu are
# reached by PageRank alone, which refuses node counts of 2^31 - 1 and more (require_pr_node_count, pr_layout.cu).
SCANNED = ["graph.cu", "wcc.cu", "sssp.cu", "tc.cu", "load.cu"]
# a loop strides over the grid when its step is the grid size or the grid's warp or thread count
GRID_STEP = re.compile(r"gridDim|\bnwarps\b|\bnthreads\b|\bnw\b")
FOR = re.compile(r"\bfor\s*\(")


def _kernels(text: str):
    """(name, body) of every __global__ function of a CUDA source."""
    for m in re.finditer(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", text):
        i = text.index("{", m.end())
        depth, j = 0, i
        while True:
            depth += {"{": 1, "}": -1}.get(text[j], 0)
            if depth == 0:
                break
            j += 1
        yield m.group(1), text[i:j + 1]


def _for_headers(body: str):
    for m in FOR.finditer(body):
        depth, j = 0, m.end() - 1
        while True:
            depth += {"(": 1, ")": -1}.get(body[j], 0)
            if depth == 0:
                break
            j += 1
        yield body[m.end():j]


def stride_loop_faults(text: str):
    """The grid- and warp-stride loops of text's kernels whose counter is narrower than 64 bits or whose
    condition is `<=`: [(kernel, loop header)]."""
    bad = []
    for name, body in _kernels(text):
        for header in _for_headers(body):
            parts = header.split(";")
            if len(parts) != 3 or not GRID_STEP.search(parts[2]):
                continue
            init, cond = parts[0].strip(), parts[1]
            if not re.match(r"(const\s+)?(uint64_t|size_t|unsigned long long)\s", init) or "<=" in cond:
                bad.append((name, header.strip()))
    return bad


@pytest.mark.parametrize("src", SCANNED)
def test_stride_loops_count_in_64_bits(src):
    bad = stride_loop_faults((CSRC / src).read_text())
    assert not bad, f"{src}: 32-bit or `<=` grid-stride loops: {bad}"


def test_stride_loop_scan_finds_the_faults():
    text = """
    __global__ void k_a(uint32_t* p, uint32_t n) {
      for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) p[v] = v;
    }
    __global__ void __launch_bounds__(256) k_b(uint32_t* p, uint32_t n) {
      const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
      for (uint32_t v = threadIdx.x >> 5; v < n; v += nwarps) { for (uint32_t i = 0; i < 4; ++i) p[v] = i; }
    }
    __global__ void k_c(uint32_t* p, uint32_t n) {
      for (uint64_t v = blockIdx.x * (uint64_t)blockDim.x; v <= n; v += (uint64_t)gridDim.x * blockDim.x) p[v] = 0;
    }
    __global__ void k_ok(uint32_t* p, uint32_t n) {
      for (uint64_t v = blockIdx.x * (uint64_t)blockDim.x; v < n; v += (uint64_t)gridDim.x * blockDim.x) p[v] = 0;
      for (uint32_t i = threadIdx.x & 31; i < 64; i += 32) p[i] = 0;
    }
    """
    assert [k for k, _ in stride_loop_faults(text)] == ["k_a", "k_b", "k_c"]
