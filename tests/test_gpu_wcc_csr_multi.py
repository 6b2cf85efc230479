"""One-shot WCC of a host out-CSR over the devices of a communicator (gb_wcc_csr_multi_u32 / Comm.wcc_csr).
The edges are cut into ndev x GB_WCC_MULTI_PARTS parts, each streamed and linked into its own forest, and the
forests merge in tree rounds.  On one GPU, GB_WCC_MULTI_PARTS > 1 runs every multi-part path (several parts,
row slices, merge rounds) on virtual parts.  Every result is compared bit for bit with the oracle's minimum-id
labels and with the single-device graph_b200.wcc_csr."""
import ctypes as C

import numpy as np
import pytest

import oracle

pytestmark = pytest.mark.gpu

GB_ERR_INVALID = 1
SENTINEL = 0xDEADBEEF
PARTS = [1, 2, 3, 8]


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


@pytest.fixture(scope="module")
def comm(gb):
    return gb.Comm([0])


def csr_of(src, dst, n, layout=oracle.SORTED):
    return oracle.csr_build(np.asarray(src, np.uint32), np.asarray(dst, np.uint32), n, oracle.OUTGOING, layout)


def parts(monkeypatch, v):
    monkeypatch.setenv("GB_WCC_MULTI_PARTS", str(v))


def feed(monkeypatch, c):
    monkeypatch.setenv("GB_WCC_FEED_EDGES", str(c))


def edge_cut(m, p, P):
    """E_p of the split: floor(m p / P) rounded down to a multiple of 4, E_P = m."""
    return m if p == P else (m * p // P) & ~3


def check_parts(gb, comm, monkeypatch, off, tgt, part_counts=PARTS):
    want = oracle.wcc_min_label(off, tgt)
    for v in part_counts:
        parts(monkeypatch, v)
        got = comm.wcc_csr(off, tgt).components()
        assert got.dtype == np.uint32 and got.tobytes() == want.tobytes(), f"{v} parts"
    return want


def raw_call(comm, off, tgt, comp, n=None):
    """gb_wcc_csr_multi_u32 straight through ctypes: (status, last error message)."""
    from graph_b200._capi import WccConfig, lib
    P = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    cfg = WccConfig(16384, 2, 1024)
    n = len(off) - 1 if n is None else n
    st = lib.gb_wcc_csr_multi_u32(comm._c if comm is not None else None, n, P(off), P(tgt), C.byref(cfg), P(comp))
    return st, (lib.gb_last_error() or b"").decode()


# ---- R-MAT against the oracle and the single-device call ---------------------------------------------------
@pytest.mark.parametrize("layout", ["Sorted", "Unsorted"])
@pytest.mark.parametrize("seed", [42, 7])
@pytest.mark.parametrize("scale", [10, 16, 20])
def test_rmat_matches_oracle_and_single_device(gb, comm, monkeypatch, scale, seed, layout):
    lay = {"Sorted": oracle.SORTED, "Unsorted": oracle.UNSORTED}[layout]
    src, dst = oracle.rmat_edges(scale, seed=seed)
    off, tgt = csr_of(src, dst, 1 << scale, lay)
    want = check_parts(gb, comm, monkeypatch, off, tgt)
    assert gb.wcc_csr(off, tgt).components().tobytes() == want.tobytes()


@pytest.mark.parametrize("c", [4, 128])
@pytest.mark.parametrize("scale", [10, 12])
def test_small_chunks(gb, comm, monkeypatch, scale, c):
    src, dst = oracle.rmat_edges(scale, seed=3)
    off, tgt = csr_of(src, dst, 1 << scale, oracle.UNSORTED)
    feed(monkeypatch, c)
    check_parts(gb, comm, monkeypatch, off, tgt)


# ---- adversarial shapes ------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [None, 4096])
def test_path_in_reverse_id_order(gb, comm, monkeypatch, c):
    # row i links i - 1: every part holds a stretch of one chain, and the merges join the stretches
    n = 1 << 20
    off = np.concatenate([[0], np.arange(n, dtype=np.uint32)]).astype(np.uint32)
    tgt = np.arange(n - 1, dtype=np.uint32)
    if c:
        feed(monkeypatch, c)
    assert (check_parts(gb, comm, monkeypatch, off, tgt) == 0).all()


@pytest.mark.parametrize("c", [None, 64])
def test_one_hub_row_spans_every_part(gb, comm, monkeypatch, c):
    n = 3000
    off = np.zeros(n + 1, np.uint32)
    off[1501:] = 100000  # row 1500 -> 100000 targets, spread over the ids below 1000 and above 2000
    rng = np.random.default_rng(1)
    tgt = np.where(rng.random(100000) < 0.5, rng.integers(0, 1000, 100000),
                   rng.integers(2000, n, 100000)).astype(np.uint32)
    if c:
        feed(monkeypatch, c)
    got = check_parts(gb, comm, monkeypatch, off, tgt)
    assert got[1500] == 0 and got[1000] == 1000


@pytest.mark.parametrize("m", [0, 1, 3, 5, 13, 31])
def test_fewer_edges_than_four_per_part(gb, comm, monkeypatch, m):
    n = 40
    rng = np.random.default_rng(m)
    off, tgt = csr_of(rng.integers(0, n, m), rng.integers(0, n, m), n, oracle.UNSORTED)
    check_parts(gb, comm, monkeypatch, off, tgt)


def test_no_edges_null_targets_and_one_node(gb, comm, monkeypatch):
    for v in PARTS:
        parts(monkeypatch, v)
        comp = np.full(5, SENTINEL, np.uint32)
        st, msg = raw_call(comm, np.zeros(6, np.uint32), None, comp)
        assert st == 0 and (comp == np.arange(5, dtype=np.uint32)).all(), msg
        assert comm.wcc_csr(np.array([0, 0], np.uint32), np.zeros(0, np.uint32)).components().tolist() == [0]
        assert comm.wcc_csr(np.array([0, 1], np.uint32), np.array([0], np.uint32)).components().tolist() == [0]
        assert comm.wcc_csr(np.array([0, 9], np.uint32), np.zeros(9, np.uint32)).components().tolist() == [0]


def test_all_edges_in_the_last_two_rows(gb, comm, monkeypatch):
    # every part's row slice is one or two rows wide
    n = 50000
    rng = np.random.default_rng(2)
    src = np.concatenate([np.full(3000, n - 2), np.full(5000, n - 1)]).astype(np.uint32)
    dst = rng.integers(0, n, len(src)).astype(np.uint32)
    off, tgt = csr_of(src, dst, n, oracle.UNSORTED)
    check_parts(gb, comm, monkeypatch, off, tgt)
    feed(monkeypatch, 12)
    check_parts(gb, comm, monkeypatch, off, tgt)


@pytest.mark.parametrize("shift", [0, 2])
def test_long_runs_of_empty_rows_at_part_borders(gb, comm, monkeypatch, shift):
    # 8 rows of 400 edges, each followed by 20000 empty rows: with 8 parts every cut E_p = 400 p falls at the
    # start of a run (shift 0), or two edges before the end of a row, in a row next to a run (shift 2)
    blocks, run = 8, 20000
    n = blocks * (run + 1) + 1
    rows = np.arange(blocks) * (run + 1)
    deg = np.zeros(n, np.int64)
    deg[rows] = 400
    deg[rows[0]] += shift
    deg[-1] = 0
    off = np.concatenate([[0], np.cumsum(deg)]).astype(np.uint32)
    m = int(off[-1])
    rng = np.random.default_rng(4)
    tgt = rng.integers(0, n, m).astype(np.uint32)
    tgt[:400] = rows[1]  # the first hub links the second, so that a merge joins a component across a cut
    want = check_parts(gb, comm, monkeypatch, off, tgt, part_counts=[1, 2, 7, 8, 9])
    assert want[rows[1]] == 0
    feed(monkeypatch, 100)
    check_parts(gb, comm, monkeypatch, off, tgt, part_counts=[8])


# ---- errors leave the output untouched ------------------------------------------------------------------
@pytest.fixture(scope="module")
def rmat16():
    src, dst = oracle.rmat_edges(16, seed=42)
    off, tgt = csr_of(src, dst, 1 << 16)
    return off, tgt, oracle.wcc_min_label(off, tgt)


def test_invalid_input_leaves_components_untouched(gb, comm, monkeypatch, rmat16):
    off, tgt, want = rmat16
    n, m, P = len(off) - 1, len(tgt), 4
    parts(monkeypatch, P)
    feed(monkeypatch, 8192)

    def rejected(o, t, match):
        comp = np.full(n, SENTINEL, np.uint32)
        st, msg = raw_call(comm, o, t, comp)
        assert st == GB_ERR_INVALID and match in msg, msg
        assert (comp == SENTINEL).all()
        comp = np.empty(n, np.uint32)
        st, msg = raw_call(comm, off, tgt, comp)  # a valid call right after succeeds
        assert st == 0 and comp.tobytes() == want.tobytes(), msg

    e2, e3 = edge_cut(m, 2, P), edge_cut(m, 3, P)
    for e in (e2, (e2 + e3) // 2, e3 - 1):  # a target >= n only in part 2: its first, a middle and last edge
        t = tgt.copy()
        t[e] = n + e % 3
        rejected(off, t, f"CSR holds 1 targets >= node_count {n}")
    # a decreasing offset inside part 2's rows: the row of its middle edge starts after the next one
    r = int(np.searchsorted(off, (e2 + e3) // 2, side="right")) - 1
    assert off[r] <= (e2 + e3) // 2 < off[r + 1] and r + 1 < n
    bad = off.copy()
    bad[r] = off[r + 1] + 1
    rejected(bad, tgt, "offsets are not monotone (1 rows)")
    bad = off.copy()
    bad[0] = 1
    rejected(bad, tgt, "offsets[0] must be 0")
    t = tgt.copy()
    t[[3, e2 + 1, m - 2]] = 0xFFFFFFFF
    rejected(off, t, f"CSR holds 3 targets >= node_count {n}")
    out = np.full(n, SENTINEL, np.uint32)
    with pytest.raises(ValueError, match="targets >= node_count"):
        comm.wcc_csr(off, t, out=out)
    assert (out == SENTINEL).all()


def test_null_arguments(gb, comm):
    from graph_b200._capi import lib
    off = np.array([0, 1, 2], np.uint32)
    tgt = np.array([1, 0], np.uint32)
    comp = np.full(2, SENTINEL, np.uint32)
    for args, match in (((None, off, tgt, comp), "comm is NULL"), ((comm, off, None, comp), "targets is NULL"),
                        ((comm, off, tgt, None), "components is NULL"),
                        ((comm, None, tgt, comp, 2), "offsets is NULL"), ((comm, off, tgt, comp, 0), "node_count")):
        st, msg = raw_call(*args)
        assert st == GB_ERR_INVALID and match in msg, msg
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib.gb_wcc_csr_multi_u32(comm._c, 2, P(off), P(tgt), None, P(comp)) == GB_ERR_INVALID
    assert (comp == SENTINEL).all()


def test_python_argument_checks(gb, comm):
    off = np.array([0, 1, 2, 2], np.uint32)
    tgt = np.array([1, 0], np.uint32)
    with pytest.raises(TypeError):
        comm.wcc_csr(off.astype(np.int64), tgt)
    with pytest.raises(TypeError):
        comm.wcc_csr(off, tgt, 16384)
    with pytest.raises(ValueError, match="targets hold 1 entries"):
        comm.wcc_csr(off, tgt[:1])
    with pytest.raises(TypeError):
        comm.wcc_csr(off, tgt, out=np.zeros(3, np.int32))
    with pytest.raises(ValueError, match="node_count = 3"):
        comm.wcc_csr(off, tgt, out=np.zeros(4, np.uint32))
    with pytest.raises(ValueError, match="node_count = 3"):
        gb.wcc_csr(off, tgt, out=np.zeros(2, np.uint32))


# ---- inputs and outputs ------------------------------------------------------------------------------------
def test_pinned_pageable_and_out_agree(gb, comm, monkeypatch, rmat16):
    import torch
    off, tgt, want = rmat16
    n = len(off) - 1
    pinned = [torch.empty(len(a), dtype=torch.int32, pin_memory=True).numpy().view(np.uint32) for a in (off, tgt)]
    pinned[0][:] = off
    pinned[1][:] = tgt
    out = torch.empty(n, dtype=torch.int32, pin_memory=True).numpy().view(np.uint32)
    for v in (1, 3):
        parts(monkeypatch, v)
        for c in (None, 8192):
            if c:
                feed(monkeypatch, c)
            a = comm.wcc_csr(*pinned).components()
            b = comm.wcc_csr(off, tgt).components()
            out[:] = SENTINEL
            r = comm.wcc_csr(*pinned, out=out).components()
            assert a.tobytes() == b.tobytes() == r.tobytes() == out.tobytes() == want.tobytes()
            assert np.shares_memory(r, out) and out.flags.writeable
            out[:] = SENTINEL
            assert gb.wcc_csr(off, tgt, out=out).components().tobytes() == want.tobytes()
            assert out.tobytes() == want.tobytes()


def test_page_rank_on_the_same_comm_is_unchanged(gb, comm, monkeypatch, rmat16):
    g = gb.DiGraph.rmat(14, seed=42, layout=gb.Layout.Sorted)
    before = comm.page_rank([g], max_iterations=20, tolerance=0.0)
    off, tgt, want = rmat16
    for v in (1, 3):
        parts(monkeypatch, v)
        assert comm.wcc_csr(off, tgt).components().tobytes() == want.tobytes()
        after = comm.page_rank([g], max_iterations=20, tolerance=0.0)
        assert after.ran_iterations == before.ran_iterations
        assert after.scores().tobytes() == before.scores().tobytes()


# ---- two or more devices -----------------------------------------------------------------------------------
@pytest.mark.parametrize("v", [1, 2])
def test_two_devices_match_oracle(gb, monkeypatch, v):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    src, dst = oracle.rmat_edges(20, seed=42)
    off, tgt = csr_of(src, dst, 1 << 20)
    parts(monkeypatch, v)
    got = gb.Comm([0, 1]).wcc_csr(off, tgt).components()
    assert got.tobytes() == oracle.wcc_min_label(off, tgt).tobytes()
