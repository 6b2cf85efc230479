"""graph_b200.triangle_count_csr (gb_triangle_count_csr_u32) on the H100: the count of a host CSR streamed in
row-aligned chunks must be oracle.triangle_count on the same CSR and what Graph.from_csr(...).global_triangle_count()
gives, on sorted and unsorted rows, with the first unsorted row in the first, a middle and the last chunk (the
reported chunk counts show which kernel path each chunk took), on multigraphs, a hub spanning many chunk budgets,
n = 1, no edges, a total above 2^32, RMAT-13 Unsorted and RMAT-20 Sorted, pinned and pageable inputs, and dozens
of chunks forced with GB_TC_FEED_ENTRIES.  Invalid input raises the error Graph.from_csr raises and leaves no
device memory behind."""
import numpy as np
import pytest

import oracle
import tc_fixtures as fx

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


def chunk_rows(off, c):
    """tc_split (csr_split.h) restated: greedy row-aligned chunks of at most c entries; a longer row stands alone
    with the empty rows next to it"""
    off = [int(x) for x in off]
    n, rows, r = len(off) - 1, [0], 0
    while r < n:
        p = int(np.searchsorted(off, off[r] + c, side="right")) - 1   # the last boundary within the budget
        p = max(p, r)
        if p < n and off[p] == off[r]:          # a hub
            p += 1
            while p < n and off[p + 1] == off[p]:
                p += 1
        rows.append(p)
        r = p
    return rows


def run(gb, off, tgt, monkeypatch=None, entries=None):
    """triangle_count_csr, checked against the oracle and the twin; returns the call's info"""
    if entries is not None:
        monkeypatch.setenv("GB_TC_FEED_ENTRIES", str(entries))
    r = gb.triangle_count_csr(off, tgt)
    if entries is not None:
        monkeypatch.delenv("GB_TC_FEED_ENTRIES")
    want = oracle.triangle_count(off, tgt, threads=0)
    assert r.triangles == want
    assert gb.Graph.from_csr(off, tgt).global_triangle_count().triangles == want
    info = r.info
    m = int(off[-1])
    assert info["h2d_bytes"] == 4 * len(off) + 4 * m
    budget = max(-(-m // 16), 1 << 20) if entries is None else entries
    assert info["chunk_entries"] == max(budget, -(-m // 4096))
    rows = chunk_rows(off, info["chunk_entries"])
    assert info["chunks"] == len(rows) - 1
    assert info["first_list_chunk"] == first_unsorted_chunk(off, tgt, rows)
    assert info["sorted_chunks"] == min(info["first_list_chunk"], info["chunks"] - (m == 0))
    assert info["sorted_chunks"] + info["list_chunks"] == info["chunks"] - (m == 0)
    return info


def first_unsorted_chunk(off, tgt, rows):
    """the chunk of the first descent inside a row (k_tc_rows_unsorted's rule), len(rows) - 1 when none"""
    off, tgt = off.astype(np.int64), tgt.astype(np.int64)
    starts = np.zeros(len(tgt) + 1, bool)
    starts[off] = True
    i = np.flatnonzero((tgt[1:] < tgt[:-1]) & ~starts[1:len(tgt)]) + 1
    if len(i) == 0:
        return len(rows) - 1
    u = int(np.searchsorted(off, i[0], side="right")) - 1
    return int(np.searchsorted(rows, u, side="right")) - 1


def rmat_csr(scale, layout):
    s, d = oracle.rmat_edges(scale, seed=42)
    return oracle.csr_build(s, d, 1 << scale, oracle.UNDIRECTED, layout)


@pytest.fixture(scope="module")
def rmat12():
    return rmat_csr(12, oracle.SORTED)


@pytest.mark.parametrize("entries", [None, 4])
@pytest.mark.parametrize("name", sorted(fx.FIXTURES))
def test_fixture(gb, monkeypatch, name, entries):
    f = fx.FIXTURES[name]()
    info = run(gb, f.off, f.tgt, monkeypatch, entries)
    assert (info["list_chunks"] == 0) == f.sorted_rows


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_first_unsorted_row_picks_the_switch(gb, monkeypatch, rmat12, where):
    off, tgt = (a.copy() for a in rmat12)
    c = int(off[-1]) // 9
    rows = chunk_rows(off, c)
    k = {"first": 0, "middle": (len(rows) - 1) // 2, "last": len(rows) - 2}[where]
    deg = np.diff(off.astype(np.int64))
    u = next(u for u in range(rows[k], rows[k + 1]) if len(set(tgt[off[u]:off[u + 1]].tolist())) > 1)
    tgt[off[u]:off[u + 1]] = tgt[off[u]:off[u + 1]][::-1].copy()
    assert deg[u] > 1
    info = run(gb, off, tgt, monkeypatch, c)
    K = info["chunks"]
    assert K == len(rows) - 1 >= 8
    assert info["first_list_chunk"] == k
    assert (info["sorted_chunks"], info["list_chunks"]) == (k, K - k)


def test_sorted_rows_take_k_tc_everywhere(gb, monkeypatch, rmat12):
    off, tgt = rmat12
    info = run(gb, off, tgt, monkeypatch, int(off[-1]) // 30)
    assert info["chunks"] >= 30 and info["list_chunks"] == 0 and info["first_list_chunk"] == info["chunks"]


@pytest.mark.parametrize("entries", [None, 7, 1000])
def test_multigraph_with_self_loops_and_parallel_edges(gb, monkeypatch, entries):
    rng = np.random.default_rng(5)
    s, d = rng.integers(0, 60, 900), rng.integers(0, 60, 900)
    s = np.concatenate([s, np.arange(60), np.arange(0, 60, 3)])
    d = np.concatenate([d, np.arange(60), np.arange(0, 60, 3)])
    for layout in (oracle.SORTED, oracle.UNSORTED):
        off, tgt = oracle.csr_build(s, d, 60, oracle.UNDIRECTED, layout)
        run(gb, off, tgt, monkeypatch, entries)
    s, d = fx.multi_clique_edges(40, 3)
    off, tgt = oracle.csr_build(s, d, 40, oracle.UNDIRECTED, oracle.SORTED)
    assert run(gb, off, tgt, monkeypatch, entries) is not None
    assert gb.triangle_count_csr(off, tgt).triangles == fx.multi_clique_count(40, 3)


def test_hub_spans_many_chunk_budgets(gb, monkeypatch):
    """a star on row 500 with 5000 leaves and chords among them: the hub is 20 budgets long and stands alone"""
    leaves = np.array([x for x in range(1001) if x != 500])
    rng = np.random.default_rng(9)
    s = np.concatenate([np.full(5000, 500), rng.integers(0, 1001, 3000)])
    d = np.concatenate([rng.choice(leaves, 5000), rng.integers(0, 1001, 3000)])
    for layout in (oracle.SORTED, oracle.UNSORTED):
        off, tgt = oracle.csr_build(s, d, 1001, oracle.UNDIRECTED, layout)
        rows = chunk_rows(off, 250)
        k = next(k for k in range(len(rows) - 1) if rows[k] <= 500 < rows[k + 1])
        assert int(off[rows[k + 1]] - off[rows[k]]) == int(off[501] - off[500]) > 20 * 250
        run(gb, off, tgt, monkeypatch, 250)


@pytest.mark.parametrize("entries", [None, 1])
def test_one_node(gb, monkeypatch, entries):
    run(gb, np.array([0, 3], np.uint32), np.zeros(3, np.uint32), monkeypatch, entries)
    info = run(gb, np.array([0, 0], np.uint32), np.zeros(0, np.uint32), monkeypatch, entries)
    assert info["chunks"] == 1 and info["kernel_launches"] == 1


def test_no_edges(gb, monkeypatch):
    off = np.zeros(1001, np.uint32)
    for entries in (None, 1):
        info = run(gb, off, np.zeros(0, np.uint32), monkeypatch, entries)
        assert info["chunks"] == 1 and info["sorted_chunks"] == info["list_chunks"] == 0


def test_total_above_2_32(gb, monkeypatch):
    n, reps = 1200, 4
    s, d = fx.multi_clique_edges(n, reps)
    off, tgt = oracle.csr_build(s, d, n, oracle.UNDIRECTED, oracle.SORTED)
    want = fx.multi_clique_count(n, reps)
    assert want == 4_596_486_400 > 2 ** 32
    assert gb.triangle_count_csr(off, tgt).triangles == want
    monkeypatch.setenv("GB_TC_FEED_ENTRIES", str(reps * (n - 1) * 50))
    r = gb.triangle_count_csr(off, tgt)
    assert r.triangles == want and r.info["chunks"] == 24


def test_rmat13_unsorted(gb, monkeypatch):
    off, tgt = rmat_csr(13, oracle.UNSORTED)
    info = run(gb, off, tgt)
    assert info["first_list_chunk"] == 0 and info["list_chunks"] == info["chunks"]
    info = run(gb, off, tgt, monkeypatch, int(off[-1]) // 40)
    assert info["chunks"] >= 40 and info["first_list_chunk"] == 0


def test_rmat20_sorted(gb):
    off, tgt = rmat_csr(20, oracle.SORTED)
    info = run(gb, off, tgt)
    assert info["chunks"] >= 16 and info["list_chunks"] == 0


def pinned_copy(a):
    import torch
    p = torch.empty(len(a), dtype=torch.int32, pin_memory=True).numpy().view(np.uint32)
    p[:] = a
    return p


def test_pinned_and_pageable_inputs_agree(gb, monkeypatch, rmat12):
    off, tgt = rmat12
    for entries in (None, int(off[-1]) // 24):
        a = run(gb, off, tgt, monkeypatch, entries)
        b = run(gb, pinned_copy(off), pinned_copy(tgt), monkeypatch, entries)
        assert (a["pinned"], b["pinned"]) == (0, 1)
        assert a["chunks"] == b["chunks"] and a["h2d_bytes"] == b["h2d_bytes"]
    unsorted = rmat_csr(12, oracle.UNSORTED)
    assert run(gb, *(pinned_copy(x) for x in unsorted))["pinned"] == 1


# ---- errors ----------------------------------------------------------------------------------------------------
def free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def raises_like_from_csr(gb, off, tgt, monkeypatch, entries):
    """the error of Graph.from_csr, and no device memory kept: a leaked target array (4 MB here) would show"""
    with pytest.raises(ValueError) as want:
        gb.Graph.from_csr(off, tgt)
    monkeypatch.setenv("GB_TC_FEED_ENTRIES", str(entries))
    with pytest.raises(ValueError):     # the first call may grow the memory pool
        gb.triangle_count_csr(off, tgt)
    before = free_bytes()
    for _ in range(3):
        with pytest.raises(ValueError) as got:
            gb.triangle_count_csr(off, tgt)
        assert str(got.value) == str(want.value)
    assert free_bytes() == before
    monkeypatch.delenv("GB_TC_FEED_ENTRIES")
    return str(got.value)


@pytest.mark.parametrize("where", [0.0, 0.5, 0.999])
def test_target_out_of_range(gb, monkeypatch, where):
    off, tgt = rmat_csr(15, oracle.SORTED)
    tgt = tgt.copy()
    tgt[int(where * len(tgt))] = len(off) - 1
    tgt[-1] = 0xFFFFFFFF
    msg = raises_like_from_csr(gb, off, tgt, monkeypatch, len(tgt) // 30)
    assert "2 targets >= node_count" in msg
    for pinned in (False, True):
        args = (pinned_copy(off), pinned_copy(tgt)) if pinned else (off, tgt)
        with pytest.raises(ValueError, match="targets >= node_count"):
            gb.triangle_count_csr(*args)


def test_offsets_not_monotone(gb, monkeypatch):
    off, tgt = rmat_csr(15, oracle.SORTED)
    off = off.copy()
    off[1000] = off[2000]
    assert "not monotone" in raises_like_from_csr(gb, off, tgt, monkeypatch, len(tgt) // 30)
    off[0] = 1
    with pytest.raises(ValueError, match=r"offsets\[0\] must be 0"):
        gb.triangle_count_csr(off, tgt)


def test_short_targets_and_wrong_dtype(gb):
    off, tgt = rmat_csr(10, oracle.SORTED)
    before = free_bytes()
    with pytest.raises(ValueError, match="targets hold"):
        gb.triangle_count_csr(off, tgt[:-1])
    for bad in ((off.astype(np.int64), tgt), (off, tgt.astype(np.int32)), (off, tgt.astype(np.uint64))):
        with pytest.raises(TypeError):
            gb.triangle_count_csr(*bad)
    assert free_bytes() == before
