"""graph_b200.sssp_csr (gb_sssp_csr_u32) on the H100: delta-stepping over a host weighted out-CSR whose rows land
chunk by chunk, from the start's chunk on, while the bucket loop runs.  Every run must be bit-equal to the twin
(DiGraph.from_csr with the transpose built here, then delta_stepping) on the same arrays and to
oracle.sssp_bellman_ford, and must pass the certificate of test_gpu_sssp.py, restated below.  The graphs are every
sssp_fixtures.py graph and the one-shot fixtures of sssp_csr_fixtures.py (a backward chain, a late improver that
needs lower = 0 after a park, a hub row many chunk budgets long), cut into one, a few and dozens of chunks
(GB_SSSP_FEED_ENTRIES), landing as fast as the bus brings them or one chunk every 1 or 3 passes
(GB_SSSP_FEED_STEP), from pinned and pageable arrays, with the start in the first, a middle and the last chunk;
then RMAT-16 and RMAT-20 at several deltas.  Invalid input raises the twin's message and status, leaves the
distances untouched and leaves no device memory behind."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
import sssp_csr_fixtures as cfx
import sssp_fixtures as fx

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import sssp_model as sm  # noqa: E402

pytestmark = pytest.mark.gpu

FLT_MAX = fx.FLT_MAX


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


def certify(off, tgt, w, start, d):
    """the certificate of the f32 shortest-path distances d (test_gpu_sssp.py): the start is at +0, no edge
    improves a distance in f32, and the reached vertices are those reached from the start over tight edges"""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import breadth_first_order
    n = len(off) - 1
    assert d.dtype == np.float32 and len(d) == n
    assert d[start] == 0.0 and not np.signbit(d[start])
    assert np.isfinite(d).all() and (d >= 0).all()
    src = np.repeat(np.arange(n, dtype=np.int64), np.diff(off.astype(np.int64)))
    tgt = tgt.astype(np.int64)
    live = d[src] < FLT_MAX
    with np.errstate(over="ignore"):
        via = d[src] + w
    bad = live & ~(d[tgt] <= via)
    assert not bad.any(), f"{int(bad.sum())} edges improve a distance, first {np.flatnonzero(bad)[:5]}"
    tight = live & (d[tgt] == via) & (d[tgt] < FLT_MAX)
    adj = csr_matrix((np.ones(int(tight.sum()), np.int8), (src[tight], tgt[tight])), shape=(n, n))
    order = breadth_first_order(adj, start, directed=True, return_predecessors=False)
    on_tight = np.zeros(n, bool)
    on_tight[order] = True
    assert (on_tight == (d < FLT_MAX)).all()
    return int((d < FLT_MAX).sum())


def transpose(off, tgt):
    n = len(off) - 1
    src = np.repeat(np.arange(n, dtype=np.uint32), np.diff(off.astype(np.int64)))
    return oracle.csr_build(src, tgt, n, oracle.INCOMING, oracle.SORTED)


def twin(gb, off, tgt, w, start, delta, bf=True):
    """the twin's distances on the same out-CSR, checked once against oracle.sssp_bellman_ford (bf): every run is
    compared with them bit for bit"""
    io, it = transpose(off, tgt)
    d = gb.DiGraph.from_csr(off, tgt, io, it, out_weights=w).delta_stepping(start_node=start, delta=delta).distances()
    if bf:
        assert d.tobytes() == oracle.sssp_bellman_ford(off, tgt, w, start).tobytes()
    return d


def pinned_copy(a):
    import torch
    p = torch.empty(len(a), dtype=torch.int32, pin_memory=True).numpy().view(a.dtype)
    p[:] = a
    return p


def budget(m, entries):
    c = max(-(-m // 16), 1 << 20) if entries is None else entries
    return max(c, -(-m // 4096))


def run(gb, monkeypatch, off, tgt, w, start, delta, want, entries=None, step=None, pinned=False):
    """sssp_csr under the given chunk budget and landing step, checked against `want` (the twin's distances, which
    twin() checked against the oracle) and the certificate; returns the call's info"""
    for name, v in (("GB_SSSP_FEED_ENTRIES", entries), ("GB_SSSP_FEED_STEP", step)):
        if v is None:
            monkeypatch.delenv(name, raising=False)
        else:
            monkeypatch.setenv(name, str(v))
    args = (off, tgt, w)
    if pinned:
        args = tuple(pinned_copy(a) for a in args)
    r = gb.sssp_csr(*args, start_node=start, delta=delta)
    monkeypatch.delenv("GB_SSSP_FEED_ENTRIES", raising=False)
    monkeypatch.delenv("GB_SSSP_FEED_STEP", raising=False)
    d = r.distances()
    assert d.tobytes() == want.tobytes(), int((d.view(np.uint32) != want.view(np.uint32)).sum())
    certify(off, tgt, w, start, d)
    info = r.info
    m = int(off[-1])
    assert info["h2d_bytes"] == 4 * len(off) + 8 * m
    c = budget(m, entries)
    rows = sm.chunk_rows(off, c)
    assert info["chunk_entries"] == c and info["chunks"] == len(rows) - 1
    assert info["start_chunk"] == sm.start_chunk(rows, start)
    assert info["pinned"] == int(pinned and m > 0)
    assert info["passes"] >= 1 and info["passes_before_last_landed"] <= info["passes"]
    if info["chunks"] == 1:
        assert info["parked"] == 0 and info["passes_before_last_landed"] == 0
    return info


GRAPHS = {name: (lambda make=fx.FIXTURES[name]: make(), None) for name in fx.REPLAYED}
GRAPHS.update({name: (make, entries) for name, (make, entries) in cfx.FIXTURES.items()})
_cache = {}


def graph(gb, name):
    if name not in _cache:
        make, entries = GRAPHS[name]
        f = make()
        off, tgt, w = oracle.csr_build(f.src, f.dst, f.n, oracle.OUTGOING, oracle.SORTED, f.w)
        _cache[name] = (f, off, tgt, w, entries, twin(gb, off, tgt, w, f.start, f.delta))
    return _cache[name]


def sizes(m, own):
    """one chunk, a few, dozens (or the fixture's own budget)"""
    out = {"one": max(m, 1), "few": max(1, -(-m // 3)), "dozens": max(1, -(-m // 40))}
    if own is not None:
        out["dozens"] = own
    return out


@pytest.mark.parametrize("step", [None, 1, 3])
@pytest.mark.parametrize("chunks", ["one", "few", "dozens"])
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_fixture(gb, monkeypatch, name, chunks, step):
    f, off, tgt, w, own, want = graph(gb, name)
    entries = sizes(int(off[-1]), own)[chunks]
    for pinned in (False, True):
        info = run(gb, monkeypatch, off, tgt, w, f.start, f.delta, want, entries, step, pinned)
        if step is not None and chunks == "dozens" and name in ("backward_chain", "late_improver"):
            assert info["parked"] > 0 and info["passes_before_last_landed"] > 0, info
            assert info["unpark_rounds"] > 0


def test_late_improver_relaxes_the_chain_again(gb, monkeypatch):
    f, off, tgt, w, own, want = graph(gb, "late_improver")
    assert want[1] == np.float32(np.float32(0.1) + np.float32(0.1)) and (want[2:10] < 1.5).all()
    for step in (1, 3):
        info = run(gb, monkeypatch, off, tgt, w, f.start, f.delta, want, own, step)
        assert info["parked"] >= 1 and info["unpark_rounds"] >= 1    # p at least


def test_hub_row_stands_alone(gb, monkeypatch):
    f, off, tgt, w, own, want = graph(gb, "hub_row")
    rows = sm.chunk_rows(off, own)
    k = next(k for k in range(len(rows) - 1) if rows[k] <= 500 < rows[k + 1])
    assert int(off[rows[k + 1]] - off[rows[k]]) == int(off[501] - off[500]) > 5 * own
    for step in (None, 1):
        run(gb, monkeypatch, off, tgt, w, f.start, f.delta, want, own, step)


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("name", ["dense128", "mixed_hub", "int_one"])
def test_start_in_any_chunk(gb, monkeypatch, name, where):
    f, off, tgt, w, _, _ = graph(gb, name)
    entries = max(1, int(off[-1]) // 24)
    rows = sm.chunk_rows(off, entries)
    k = {"first": 0, "middle": (len(rows) - 1) // 2, "last": len(rows) - 2}[where]
    start = (rows[k] + rows[k + 1]) // 2
    want = twin(gb, off, tgt, w, start, f.delta)
    for step in (None, 1, 3):
        for pinned in (False, True):
            info = run(gb, monkeypatch, off, tgt, w, start, f.delta, want, entries, step, pinned)
            assert info["start_chunk"] == k


def test_one_node_and_no_edges(gb, monkeypatch):
    off1 = np.array([0, 2], np.uint32)
    tgt1 = np.zeros(2, np.uint32)
    w1 = np.array([1.0, 0.0], np.float32)
    want = twin(gb, off1, tgt1, w1, 0, 1.0)
    assert want.tolist() == [0.0]
    for entries in (None, 1):
        run(gb, monkeypatch, off1, tgt1, w1, 0, 1.0, want, entries)
    off0 = np.zeros(101, np.uint32)
    none_t, none_w = np.zeros(0, np.uint32), np.zeros(0, np.float32)
    want = twin(gb, off0, none_t, none_w, 7, 1.0)
    assert want[7] == 0.0 and (np.delete(want, 7) == FLT_MAX).all()
    for entries in (None, 1):
        info = run(gb, monkeypatch, off0, none_t, none_w, 7, 1.0, want, entries)
        assert info["chunks"] == 1 and info["passes"] == 1
    d = gb.sssp_csr(off0, none_t, None, start_node=7, delta=1.0).distances()   # weights may be None: no edges
    assert d.tobytes() == want.tobytes()


# ---- RMAT --------------------------------------------------------------------------------------------------------
def rmat_csr(scale):
    s, d = oracle.rmat_edges(scale, seed=42)
    w = oracle.rmat_weights(42, 0, len(s))
    off, tgt, w = oracle.csr_build(s, d, 1 << scale, oracle.OUTGOING, oracle.SORTED, w)
    start = int(np.argmax(np.diff(off.astype(np.int64))))
    return off, tgt, w, start


@pytest.mark.parametrize("scale,deltas", [(16, (1e-30, 0.01, 0.1, 1.0)), (20, (0.01, 0.1))])
def test_rmat(gb, monkeypatch, scale, deltas):
    off, tgt, w, start = rmat_csr(scale)
    m = int(off[-1])
    for delta in deltas:
        want = twin(gb, off, tgt, w, start, delta, bf=scale <= 16)
        for entries, step, pinned in ((None, None, True), (None, None, False), (m // 40, None, True),
                                      (m // 40, 1, False)):
            run(gb, monkeypatch, off, tgt, w, start, delta, want, entries, step, pinned)
        assert certify(off, tgt, w, start, want) > (1 << (scale - 1))


# ---- errors ------------------------------------------------------------------------------------------------------
def free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def fails_like_twin(gb, monkeypatch, off, tgt, w, start, delta, entries, status, io_it=None):
    """gb_sssp_csr_u32 fails with the status and message of DiGraph.from_csr + delta_stepping on the same out-CSR
    (the in-CSR is the transpose of the valid graph when the out-CSR cannot have one), writes nothing to the
    distances and keeps no device memory"""
    from graph_b200._capi import SsspConfig, lib
    io, it = io_it if io_it is not None else transpose(off, tgt)
    with pytest.raises(ValueError) as want:
        gb.DiGraph.from_csr(off, tgt, io, it, out_weights=w).delta_stepping(start_node=start, delta=delta)
    monkeypatch.setenv("GB_SSSP_FEED_ENTRIES", str(entries))
    n = len(off) - 1
    cfg = SsspConfig(start, delta)
    ptr = (lambda a: None if a is None else a.ctypes.data_as(C.c_void_p))

    def call(dist):
        return lib.gb_sssp_csr_u32(0, n, ptr(off), ptr(tgt), ptr(w), C.byref(cfg), ptr(dist))
    sentinel = np.full(n, 1234.5, np.float32)
    call(sentinel.copy())                 # the first call may grow the memory pool
    before = free_bytes()
    for step in (None, 1):
        if step is None:
            monkeypatch.delenv("GB_SSSP_FEED_STEP", raising=False)
        else:
            monkeypatch.setenv("GB_SSSP_FEED_STEP", str(step))
        dist = sentinel.copy()
        got = call(dist)
        assert got == status
        assert lib.gb_last_error().decode() == str(want.value)
        assert dist.tobytes() == sentinel.tobytes()
    assert free_bytes() == before
    monkeypatch.delenv("GB_SSSP_FEED_ENTRIES")
    monkeypatch.delenv("GB_SSSP_FEED_STEP", raising=False)
    return str(want.value)


@pytest.fixture(scope="module")
def rmat12():
    return rmat_csr(12)


def test_null_weights(gb, monkeypatch, rmat12):
    from graph_b200._capi import GB_ERR_UNSUPPORTED
    off, tgt, w, start = rmat12
    msg = fails_like_twin(gb, monkeypatch, off, tgt, None, start, 0.1, int(off[-1]) // 30, GB_ERR_UNSUPPORTED)
    assert msg.startswith("sssp needs f32 edge values")


@pytest.mark.parametrize("where", [0.0, 0.5, 0.999])
def test_target_out_of_range(gb, monkeypatch, rmat12, where):
    from graph_b200._capi import GB_ERR_INVALID
    off, tgt, w, start = rmat12
    io_it = transpose(off, tgt)
    tgt = tgt.copy()
    tgt[int(where * len(tgt))] = len(off) - 1
    tgt[-1] = 0xFFFFFFFF
    msg = fails_like_twin(gb, monkeypatch, off, tgt, w, start, 0.1, len(tgt) // 30, GB_ERR_INVALID, io_it)
    assert "out CSR holds 2 targets >= node_count" in msg
    for pinned in (False, True):
        args = tuple(pinned_copy(a) for a in (off, tgt, w)) if pinned else (off, tgt, w)
        with pytest.raises(ValueError, match="targets >= node_count"):
            gb.sssp_csr(*args, start_node=start, delta=0.1)


def test_offsets_not_monotone(gb, monkeypatch, rmat12):
    from graph_b200._capi import GB_ERR_INVALID
    off, tgt, w, start = rmat12
    io_it = transpose(off, tgt)
    off = off.copy()
    off[1000] = off[2000]
    msg = fails_like_twin(gb, monkeypatch, off, tgt, w, start, 0.1, len(tgt) // 30, GB_ERR_INVALID, io_it)
    assert "out offsets are not monotone" in msg


@pytest.mark.parametrize("start,delta", [(1 << 12, 0.1), (0, 0.0), (0, -1.0), (0, float("inf")),
                                         (0, float("nan"))])
def test_bad_config(gb, monkeypatch, rmat12, start, delta):
    from graph_b200._capi import GB_ERR_INVALID
    off, tgt, w, _ = rmat12
    msg = fails_like_twin(gb, monkeypatch, off, tgt, w, start, delta, len(tgt) // 30, GB_ERR_INVALID)
    assert ("start_node" in msg) == (start != 0)
