"""One-shot WCC of a host out-CSR (gb_wcc_csr_u32 / graph_b200.wcc_csr): the targets stream through a ring of
device buffers in chunks of GB_WCC_FEED_EDGES edges and every edge is linked as it lands.  Every result is
compared bit for bit with the oracle's minimum-id labels, and on R-MAT also with DiGraph.wcc() on the twin."""
import ctypes as C

import numpy as np
import pytest

import oracle

pytestmark = pytest.mark.gpu

GB_ERR_INVALID = 1
SENTINEL = 0xDEADBEEF


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


def csr_of(src, dst, n, layout=oracle.SORTED, direction=oracle.OUTGOING):
    return oracle.csr_build(np.asarray(src, np.uint32), np.asarray(dst, np.uint32), n, direction, layout)


def labels(gb, off, tgt, **kw):
    return gb.wcc_csr(off, tgt, **kw).components()


def raw_call(off, tgt, comp, n=None):
    """gb_wcc_csr_u32 straight through ctypes: (status, last error message)."""
    from graph_b200._capi import WccConfig, lib
    P = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    cfg = WccConfig(16384, 2, 1024)
    n = len(off) - 1 if n is None else n
    st = lib.gb_wcc_csr_u32(0, n, P(off), P(tgt), C.byref(cfg), P(comp))
    return st, (lib.gb_last_error() or b"").decode()


def check_against_oracle(gb, off, tgt, **kw):
    want = oracle.wcc_min_label(off, tgt)
    got = labels(gb, off, tgt, **kw)
    assert got.dtype == np.uint32 and got.tobytes() == want.tobytes()
    return got


@pytest.fixture(scope="module")
def rmat16():
    src, dst = oracle.rmat_edges(16, seed=42)
    n = 1 << 16
    return src, dst, n, csr_of(src, dst, n)


# ---- R-MAT against the oracle and the twin ---------------------------------------------------------------
@pytest.mark.parametrize("layout", ["Sorted", "Unsorted"])
@pytest.mark.parametrize("seed", [42, 7])
@pytest.mark.parametrize("scale", [10, 16, 20])
def test_rmat_matches_oracle_and_twin(gb, scale, seed, layout):
    lay = {"Sorted": oracle.SORTED, "Unsorted": oracle.UNSORTED}[layout]
    src, dst = oracle.rmat_edges(scale, seed=seed)
    n = 1 << scale
    out = csr_of(src, dst, n, lay)
    inc = csr_of(src, dst, n, lay, oracle.INCOMING)
    got = check_against_oracle(gb, *out)
    twin = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1]).wcc().components()
    assert got.tobytes() == twin.tobytes()
    # the in-CSR lists the same edges: weak connectivity gives the same labels
    assert labels(gb, *inc).tobytes() == got.tobytes()
    # the config changes the reference's work, never the labels
    for kw in ({"neighbor_rounds": 0}, {"chunk_size": 1, "sampling_size": 0}):
        assert labels(gb, *out, **kw).tobytes() == got.tobytes()


# ---- chunking: GB_WCC_FEED_EDGES sets the chunk size C in edges --------------------------------------------
def feed(monkeypatch, c):
    monkeypatch.setenv("GB_WCC_FEED_EDGES", str(c))


def test_one_chunk(gb, rmat16, monkeypatch):
    off, tgt = rmat16[3]
    feed(monkeypatch, 4 * len(tgt))
    check_against_oracle(gb, off, tgt)


def test_fewer_chunks_than_buffers(gb, rmat16, monkeypatch):
    off, tgt = rmat16[3]
    m = len(tgt)
    feed(monkeypatch, (m // 2 + 4) & ~3)  # two chunks, three buffers
    check_against_oracle(gb, off, tgt)


def test_many_chunks_reuse_the_buffers(gb, rmat16, monkeypatch):
    off, tgt = rmat16[3]
    feed(monkeypatch, 4096)  # 256 chunks through three buffers
    check_against_oracle(gb, off, tgt)


def test_chunk_size_that_does_not_divide_m(gb, rmat16, monkeypatch):
    off, tgt = rmat16[3]
    assert len(tgt) % 1000 != 0
    feed(monkeypatch, 1000)
    check_against_oracle(gb, off, tgt)


def test_chunk_boundary_inside_a_hub_row(gb, rmat16, monkeypatch):
    off, tgt = rmat16[3]
    deg = np.diff(off.astype(np.int64))
    hub = int(np.argmax(deg))
    c = (int(off[hub]) // 4 + 1) * 4   # the first multiple of 4 past the hub's first edge
    assert off[hub] < c < off[hub + 1]
    feed(monkeypatch, c)
    check_against_oracle(gb, off, tgt)
    # a hub that spans many chunks and many warps
    feed(monkeypatch, 64)
    check_against_oracle(gb, off, tgt)


@pytest.mark.parametrize("c", [8, 12, 4])
def test_chunk_boundary_inside_a_run_of_empty_rows(gb, monkeypatch, c):
    # rows 0 and n - 1 hold 8 edges each, the 10^5 rows between are empty: C = 8 puts the boundary at the
    # run (off[1] == ... == off[n - 1] == 8), C = 12 puts the run inside a chunk, C = 4 does both
    n = 100002
    src = np.array([0] * 8 + [n - 1] * 8, np.uint32)
    dst = np.array([1, 2, 3, 4, 5, 6, 7, n - 1, 9, 10, 11, 12, 13, 14, 15, n - 2], np.uint32)
    off, tgt = csr_of(src, dst, n)
    feed(monkeypatch, c)
    got = check_against_oracle(gb, off, tgt)
    assert got[n - 1] == 0 and got[9] == 0 and got[n - 3] == n - 3


def test_smallest_chunk(gb, monkeypatch):
    src, dst = oracle.rmat_edges(12, seed=3)
    n = 1 << 12
    off, tgt = csr_of(src, dst, n, oracle.UNSORTED)
    feed(monkeypatch, 4)
    check_against_oracle(gb, off, tgt)
    feed(monkeypatch, 1)  # rounded up to the smallest chunk
    check_against_oracle(gb, off, tgt)


# ---- shapes ----------------------------------------------------------------------------------------------
def test_no_edges_and_null_targets(gb):
    off = np.zeros(6, np.uint32)
    comp = np.full(5, SENTINEL, np.uint32)
    st, msg = raw_call(off, None, comp)
    assert st == 0, msg
    assert (comp == np.arange(5, dtype=np.uint32)).all()
    assert (labels(gb, off, np.zeros(0, np.uint32)) == np.arange(5)).all()


def test_one_node_with_a_self_loop(gb):
    assert labels(gb, np.array([0, 1], np.uint32), np.array([0], np.uint32)).tolist() == [0]


def test_only_self_loops(gb):
    n = 1000
    off = np.arange(n + 1, dtype=np.uint32)
    assert (check_against_oracle(gb, off, np.arange(n, dtype=np.uint32)) == np.arange(n)).all()


def test_every_edge_three_times(gb, monkeypatch):
    src, dst = oracle.rmat_edges(10, seed=42)
    n = 1 << 10
    off, tgt = csr_of(np.repeat(src, 3), np.repeat(dst, 3), n, oracle.UNSORTED)
    check_against_oracle(gb, off, tgt)
    feed(monkeypatch, 12)
    check_against_oracle(gb, off, tgt)


@pytest.mark.parametrize("c", [None, 4096])
def test_star_with_the_hub_last(gb, monkeypatch, c):
    leaves = 100000
    n = leaves + 1
    off = np.zeros(n + 1, np.uint32)
    off[n] = leaves
    tgt = np.arange(leaves, dtype=np.uint32)  # row n - 1 -> every other node
    if c:
        feed(monkeypatch, c)
    assert (check_against_oracle(gb, off, tgt) == 0).all()


@pytest.mark.parametrize("c", [None, 4096])
def test_path_in_reverse_id_order(gb, monkeypatch, c):
    # row i links i - 1: every link hooks a root under the next lower one, a parent chain n deep
    n = 1 << 20
    off = np.concatenate([[0], np.arange(n, dtype=np.uint32)]).astype(np.uint32)
    tgt = np.arange(n - 1, dtype=np.uint32)
    if c:
        feed(monkeypatch, c)
    assert (check_against_oracle(gb, off, tgt) == 0).all()


def test_components_with_the_last_ids_as_minima(gb):
    n = 5000
    src = np.concatenate([np.arange(1, n - 2), [n - 2, n - 1]]).astype(np.uint32)
    dst = np.concatenate([np.arange(0, n - 3), [n - 2, n - 1]]).astype(np.uint32)
    got = check_against_oracle(gb, *csr_of(src, dst, n))
    assert (got[:n - 2] == 0).all() and got[n - 2] == n - 2 and got[n - 1] == n - 1


def test_every_target_is_the_last_id(gb, monkeypatch):
    n = 70000
    off = np.arange(n + 1, dtype=np.uint32)
    tgt = np.full(n, n - 1, np.uint32)
    assert (check_against_oracle(gb, off, tgt) == 0).all()
    feed(monkeypatch, 16)
    assert (check_against_oracle(gb, off, tgt) == 0).all()


def test_empty_leading_and_trailing_rows(gb, monkeypatch):
    n = 3000
    rng = np.random.default_rng(5)
    src = rng.integers(1000, 2000, 4000).astype(np.uint32)
    dst = rng.integers(1000, 2000, 4000).astype(np.uint32)
    off, tgt = csr_of(src, dst, n)
    assert off[1000] == 0 and off[2000] == len(tgt)
    check_against_oracle(gb, off, tgt)
    feed(monkeypatch, 100)
    check_against_oracle(gb, off, tgt)


def test_ids_past_2_16(gb, monkeypatch):
    n = (1 << 17) + 3
    rng = np.random.default_rng(11)
    src = rng.integers(1 << 16, n, 300000).astype(np.uint32)
    dst = rng.integers(0, n, 300000).astype(np.uint32)
    off, tgt = csr_of(src, dst, n, oracle.UNSORTED)
    check_against_oracle(gb, off, tgt)
    feed(monkeypatch, 10000)
    check_against_oracle(gb, off, tgt)


# ---- inputs ----------------------------------------------------------------------------------------------
def test_pinned_and_pageable_inputs_agree(gb, rmat16, monkeypatch):
    import torch
    off, tgt = rmat16[3]
    pinned = [torch.empty(len(a), dtype=torch.int32, pin_memory=True).numpy().view(np.uint32) for a in (off, tgt)]
    pinned[0][:] = off
    pinned[1][:] = tgt
    for c in (None, 8192):
        if c:
            feed(monkeypatch, c)
        a = labels(gb, *pinned)
        b = labels(gb, off, tgt)
        assert a.tobytes() == b.tobytes() == oracle.wcc_min_label(off, tgt).tobytes()
        assert labels(gb, *pinned).tobytes() == a.tobytes()  # two calls in a row


def test_invalid_input_leaves_components_untouched(gb, rmat16, monkeypatch):
    off, tgt = rmat16[3]
    n = len(off) - 1
    want = oracle.wcc_min_label(off, tgt)
    feed(monkeypatch, 8192)  # 128 chunks

    def rejected(o, t, match):
        comp = np.full(n, SENTINEL, np.uint32)
        st, msg = raw_call(o, t, comp)
        assert st == GB_ERR_INVALID and match in msg, msg
        assert (comp == SENTINEL).all()
        comp = np.empty(n, np.uint32)
        st, msg = raw_call(off, tgt, comp)  # a valid call right after succeeds
        assert st == 0 and comp.tobytes() == want.tobytes(), msg

    bad = off.copy()
    bad[0] = 1
    rejected(bad, tgt, "offsets[0] must be 0")
    bad = off.copy()
    bad[5] = off[6] + 1
    rejected(bad, tgt, "offsets are not monotone (1 rows)")
    m = len(tgt)
    for e in (0, m // 2 + 1, m - 1):  # first, a middle and the last chunk
        t = tgt.copy()
        t[e] = n + e % 3
        rejected(off, t, f"holds 1 targets >= node_count {n}")
    t = tgt.copy()
    t[[3, 8191, 8192, m - 2]] = 0xFFFFFFFF
    rejected(off, t, f"holds 4 targets >= node_count {n}")
    with pytest.raises(ValueError, match="targets >= node_count"):
        gb.wcc_csr(off, t)


def test_null_arguments(gb):
    off = np.array([0, 1, 2], np.uint32)
    tgt = np.array([1, 0], np.uint32)
    comp = np.full(2, SENTINEL, np.uint32)
    assert raw_call(off, None, comp)[0] == GB_ERR_INVALID
    assert raw_call(off, tgt, None)[0] == GB_ERR_INVALID
    assert raw_call(None, tgt, comp, n=2)[0] == GB_ERR_INVALID
    assert raw_call(off, tgt, comp, n=0)[0] == GB_ERR_INVALID
    from graph_b200._capi import lib
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib.gb_wcc_csr_u32(0, 2, P(off), P(tgt), None, P(comp)) == GB_ERR_INVALID
    assert (comp == SENTINEL).all()


# ---- the BASELINE WCC size ----------------------------------------------------------------------------
def test_rmat24_matches_oracle_and_twin(gb):
    g = gb.DiGraph.rmat(24, seed=42, layout=gb.Layout.Sorted)
    ooff, otgt = g.csr("out")
    got = labels(gb, ooff, otgt)
    assert got.tobytes() == g.wcc().components().tobytes()
    assert got.tobytes() == oracle.wcc_min_label(ooff, otgt).tobytes()
