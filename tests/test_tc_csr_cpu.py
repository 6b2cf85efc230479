"""CPU-side checks of graph_b200.triangle_count_csr (one-shot triangle count of a host undirected CSR): the
chunk cut (tc_split, graph_b200/csrc/csr_split.h) compiled with g++ and checked on random, tiny, edgeless, hub-heavy and
non-monotone offsets; a restatement of the call's sorted-prefix rule, which counts chunk by chunk in row order
and switches from k_tc's term to the list-order term at the first chunk with an unsorted row, against
oracle.triangle_count on the tc_fixtures.py graphs; the C symbols with their ctypes declarations and header
lines; and the Python argument checks."""
import ctypes
import subprocess
from bisect import bisect_left, bisect_right
from pathlib import Path

import numpy as np
import pytest

import oracle
import tc_fixtures as fx

ROOT = Path(__file__).resolve().parent.parent


def test_split_cuts_rows_in_order(tmp_path):
    exe = tmp_path / "tc_split_check"
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'graph_b200' / 'csrc'}",
           str(ROOT / "tests" / "cpp" / "tc_split_check.cpp"), "-o", str(exe)]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "tc_split ok" in r.stdout, r.stdout + r.stderr


# ---- the sorted-prefix rule, restated --------------------------------------------------------------------
def k_tc_term(off, t, u, i) -> int:
    """k_tc's term of entry i = (u, v): the w <= v of N(v) found in N(u) cut to values <= v (sorted rows)"""
    v = t[i]
    if v > u:
        return 0
    ub, ue = off[u], bisect_right(t, v, off[u], off[u + 1])
    total = 0
    for j in range(off[v], bisect_right(t, v, off[v], off[v + 1])):
        p = bisect_left(t, t[j], ub, ue)
        total += p < ue and t[p] == t[j]
    return total


def list_term(off, t, cut, u, i) -> int:
    """k_tc_list's term of entry i < cut[u]: the reference loop, a put-back cursor over N(u), list order"""
    if i >= cut[u]:
        return 0
    v, it, ue, total = t[i], off[u], off[u + 1], 0
    for j in range(off[v], cut[v]):
        while it < ue and t[it] < t[j]:
            it += 1
        if it == ue:
            break
        total += t[it] == t[j]
    return total


def has_descent(off, t, r0, r1) -> bool:
    """k_tc_rows_unsorted over the rows [r0, r1) only"""
    return any(t[i - 1] > t[i] for u in range(r0, r1) for i in range(off[u] + 1, off[u + 1]))


def row_cut(off, t, u) -> int:
    return next((i for i in range(off[u], off[u + 1]) if t[i] > u), off[u + 1])


def chunked_count(off, tgt, rows):
    """the call's count over the row-aligned chunks [rows[k], rows[k + 1]), in order: a term of row u reads rows
    u and v <= u only, so no chunk reads a later one; (total, index of the first list-order chunk, or the chunk
    count when there is none)"""
    off, t = [int(x) for x in off], [int(x) for x in tgt]
    cut, total, first_list = [], 0, None
    for k in range(len(rows) - 1):
        r0, r1 = rows[k], rows[k + 1]
        cut += [row_cut(off, t, u) for u in range(r0, r1)]
        if first_list is None and has_descent(off, t, r0, r1):
            first_list = k
        for u in range(r0, r1):
            for i in range(off[u], off[u + 1]):
                total += k_tc_term(off, t, u, i) if first_list is None else list_term(off, t, cut, u, i)
    return total, len(rows) - 1 if first_list is None else first_list


def row_cuts(n, how, rng):
    if how == "one chunk":
        return [0, n]
    if how == "every row":
        return list(range(n + 1))
    if how == "thirds":
        return sorted({0, n // 3, 2 * n // 3, n})
    inner = rng.choice(np.arange(1, n), size=min(n - 1, 7), replace=False) if n > 1 else []
    return [0, *sorted(int(x) for x in inner), n]


@pytest.mark.parametrize("how", ["one chunk", "every row", "thirds", "random"])
@pytest.mark.parametrize("name", sorted(fx.FIXTURES))
def test_chunked_count_is_the_whole_graph_count(name, how):
    f = fx.FIXTURES[name]()
    if how == "every row" and f.n > 300:
        pytest.skip("one chunk per row is checked on the small fixtures")
    rows = row_cuts(f.n, how, np.random.default_rng(len(name)))
    total, first_list = chunked_count(f.off, f.tgt, rows)
    assert total == oracle.triangle_count(f.off, f.tgt), (name, how)
    assert (first_list == len(rows) - 1) == f.sorted_rows, (name, how)


def test_switch_lands_where_the_first_unsorted_row_is():
    """one unsorted row moved through the chunks: the list path starts at its chunk, and the sum stays put"""
    rows = fx.rmat_sorted_rows(8)
    n = len(rows)
    cuts = [0, 64, 128, 192, n]
    for where, u in ((0, 3), (1, 100), (2, 150), (3, n - 1)):
        u = next(x for x in range(u, n) if len(set(rows[x])) > 1)
        bad = [list(r) for r in rows]
        bad[u] = bad[u][::-1]
        f = fx.from_csr(bad)
        total, first_list = chunked_count(f.off, f.tgt, cuts)
        assert first_list == where
        assert total == oracle.triangle_count(f.off, f.tgt)


def test_multigraph_and_hub():
    s, d = fx.multi_clique_edges(12, 3)
    off, tgt = oracle.csr_build(s, d, 12, oracle.UNDIRECTED, oracle.SORTED)
    assert chunked_count(off, tgt, [0, 11, 12])[0] == fx.multi_clique_count(12, 3)
    star = fx.star_last_row()
    assert chunked_count(star.off, star.tgt, [0, 20, 39, 40])[0] == oracle.triangle_count(star.off, star.tgt)


# ---- the interface -------------------------------------------------------------------------------------------
OFF = np.array([0, 1, 2, 2], np.uint32)
TGT = np.array([1, 0], np.uint32)


def test_symbols_are_exported_and_declared():
    import graph_b200 as gb
    import graph_b200._capi as capi
    lib = ctypes.CDLL(str(capi.LIB_PATH))
    header = (ROOT / "include" / "graph_b200.h").read_text()
    for name, nargs, decl in (
            ("gb_triangle_count_csr_u32", 5, "gb_status gb_triangle_count_csr_u32(int device, uint32_t node_count,"),
            ("gb_triangle_count_csr_info", 1, "gb_status gb_triangle_count_csr_info(gb_tc_csr_info* info);")):
        assert hasattr(lib, name)
        res, args = capi.SIGNATURES[name]
        assert res is ctypes.c_int and len(args) == nargs
        assert decl in header
    assert ctypes.sizeof(capi.TcCsrInfo) == 7 * 8 + 2 * 4 + 2 * 8
    assert "global_triangle_count_csr(" in (ROOT / "include" / "graph_b200.hpp").read_text()
    assert "triangle_count_csr" in gb.__all__


def test_missing_device_is_reported():
    import torch
    if torch.cuda.is_available():
        pytest.skip("this box has a GPU")
    import graph_b200 as gb
    with pytest.raises(gb.GraphB200Error, match="no CUDA device"):
        gb.triangle_count_csr(OFF, TGT)


def test_arrays_must_be_contiguous_uint32():
    import graph_b200 as gb
    with pytest.raises(TypeError):
        gb.triangle_count_csr(OFF.astype(np.int64), TGT)
    with pytest.raises(TypeError):
        gb.triangle_count_csr(OFF, TGT.astype(np.int32))
    with pytest.raises(TypeError):
        gb.triangle_count_csr(OFF, np.array([1, 9, 0, 9], np.uint32)[::2])
    with pytest.raises(TypeError):
        gb.triangle_count_csr(OFF.tolist(), TGT)


def test_short_arrays_are_rejected():
    import graph_b200 as gb
    with pytest.raises(ValueError, match="targets hold 1 entries"):
        gb.triangle_count_csr(OFF, TGT[:1])
    with pytest.raises(ValueError, match="offsets need"):
        gb.triangle_count_csr(np.array([0], np.uint32), TGT)
