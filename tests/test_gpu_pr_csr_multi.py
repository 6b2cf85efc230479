"""One-shot PageRank of a host CSR over the devices of a communicator (gb_page_rank_csr_multi_u32 /
gb_pr_shards_csr_u32 / Comm.page_rank_csr).  Each part of the in-CSR is uploaded by one rank's device, every rank
gathers the rows it owns into a local in-CSR (k_pr_gather_rows) and builds its shard from it.  On one GPU,
ranks_per_device > 1 runs every multi-part path on virtual ranks: each shard must equal gb_pr_shard_create on a
full twin (plan shape, statistics, and six sweeps with fused peer stores through tests/virtual_ranks.py, bit for
bit), and Comm.page_rank_csr must equal Comm.page_rank with a twin."""
import ctypes as C

import numpy as np
import pytest

import oracle
import pr_path_fixtures as fx
from virtual_ranks import VirtualRanks

pytestmark = pytest.mark.gpu

GB_ERR_INVALID = 1
SENTINEL = np.float32(-7.25)
SWEEPS = 6
PR_RTOL = 1e-6
RANKS = [1, 2, 3, 8]
# GB_PR_PART_CHUNK_EDGES per rank count: several target chunks per part, down to chunks of a few rows
CHUNKS = {1: None, 2: 4096, 3: 777, 8: 100000}


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


@pytest.fixture(scope="module")
def comm(gb):
    return gb.Comm([0])


def csrs(src, dst, n, layout=oracle.SORTED):
    src, dst = np.asarray(src, np.uint32), np.asarray(dst, np.uint32)
    return n, oracle.csr_build(src, dst, n, oracle.OUTGOING, layout), oracle.csr_build(src, dst, n, oracle.INCOMING,
                                                                                       layout)


def twin(gb, out, inc):
    return gb.DiGraph.for_page_rank(inc[0], inc[1], out[0])


def rel_err(got, want):
    return float(np.max(np.abs(got.astype(np.float64) - want) / want)) if len(want) else 0.0


def sweeps(vr):
    """init + SWEEPS sweeps with fused peer stores: (error shares per sweep, next vectors, score vectors)"""
    import torch
    vr.init()
    errs = [vr.step(peers=True) for _ in range(SWEEPS)]
    torch.cuda.synchronize()
    return (errs, [x.cpu().numpy().tobytes() for x in vr.x_next()],
            [s.cpu().numpy().tobytes() for s in vr.scores])


def check_shards(gb, comm, monkeypatch, n, out, inc, ranks=RANKS):
    """every shard of gb_pr_shards_csr_u32 equals the twin's shard of the same rank"""
    want = oracle.page_rank_jacobi(inc[0], inc[1], out[0], SWEEPS, 0.0, 0.85, acc64=True)[0]
    g = twin(gb, out, inc)
    for v in ranks:
        if CHUNKS[v]:
            monkeypatch.setenv("GB_PR_PART_CHUNK_EDGES", str(CHUNKS[v]))
        else:
            monkeypatch.delenv("GB_PR_PART_CHUNK_EDGES", raising=False)
        ref = VirtualRanks(g, v)
        new = VirtualRanks(g, v)
        new.ranks = comm.pr_shards_csr(inc[0], inc[1], out[0], ranks_per_device=v)
        assert len(new.ranks) == v
        for r, (a, b) in enumerate(zip(ref.ranks, new.ranks)):
            assert b.graph is None and (b.rank, b.world, b.n) == (r, v, n)
            assert b.plan_shape() == a.plan_shape(), (v, r)
            assert b.info() == a.info(), (v, r)
        got, exp = sweeps(new), sweeps(ref)
        assert got[0] == exp[0], (v, "error shares")
        assert got[1] == exp[1], (v, "next vectors")
        assert got[2] == exp[2], (v, "score vectors")
        scores = new.scores_host()
        assert scores.tobytes() == ref.scores_host().tobytes(), v
        assert rel_err(scores, want) <= PR_RTOL, v


# ---- 1. shards against twins --------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", ["Sorted", "Unsorted"])
@pytest.mark.parametrize("seed", [42, 7])
@pytest.mark.parametrize("scale", [10, 16, 20])
def test_rmat_shards_equal_twin_shards(gb, comm, monkeypatch, scale, seed, layout):
    fx.set_knobs(monkeypatch, "rmat")
    src, dst = oracle.rmat_edges(scale, seed=seed)
    lay = {"Sorted": oracle.SORTED, "Unsorted": oracle.UNSORTED}[layout]
    check_shards(gb, comm, monkeypatch, *csrs(src, dst, 1 << scale, lay))


@pytest.mark.parametrize("name", ["star_in", "repeated_source", "rmat18", "capped_finish", "few_active"])
def test_path_fixture_shards_equal_twin_shards(gb, comm, monkeypatch, name):
    """mega rows (star_in, repeated_source), hub-group finish CTAs (rmat18, capped_finish), fewer than 32 P
    active rows (few_active)"""
    fx.set_knobs(monkeypatch, name)
    _, _, n, out, inc = fx.graph(name)
    check_shards(gb, comm, monkeypatch, n, out, inc)


def hub_longer_than_parts():
    # row 1500 holds 100000 of the ~103000 in-edges: with 2 or more parts, the parts between its first and last
    # edge are empty
    n = 3000
    rng = np.random.default_rng(1)
    src = np.concatenate([rng.integers(0, n, 100000), rng.integers(0, n, 3000)])
    dst = np.concatenate([np.full(100000, 1500), rng.integers(0, n, 3000)])
    return src, dst, n


def high_ids():
    # ids past 2^24, and a few rows near 0
    n = (1 << 24) + 4096
    rng = np.random.default_rng(2)
    src = np.concatenate([rng.integers(n - 60000, n, 200000), rng.integers(0, 64, 100)])
    dst = np.concatenate([rng.integers(n - 60000, n, 200000), rng.integers(n - 10, n, 100)])
    return src, dst, n


SHAPES = {
    "no_edges": lambda: (np.zeros(0), np.zeros(0), 70),
    "one_node": lambda: (np.zeros(0), np.zeros(0), 1),
    "one_node_loop": lambda: ([0, 0], [0, 0], 1),
    "hub_longer_than_parts": hub_longer_than_parts,
    "high_ids": high_ids,
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_edge_shapes_shards_equal_twin_shards(gb, comm, monkeypatch, name):
    fx.set_knobs(monkeypatch, "shape")
    src, dst, n = SHAPES[name]()
    check_shards(gb, comm, monkeypatch, *csrs(src, dst, n))


# ---- 2. Comm([0]).page_rank_csr against Comm([0]).page_rank with a twin --------------------------------------
def rmat16():
    src, dst = oracle.rmat_edges(16, seed=42)
    return csrs(src, dst, 1 << 16)


def pinned(a):
    import torch
    p = torch.empty(max(len(a), 1), dtype=torch.int32, pin_memory=True).numpy().view(np.uint32)[:len(a)]
    p[:] = a
    return p


def same(a, b):
    return (a.scores().tobytes() == b.scores().tobytes() and a.ran_iterations == b.ran_iterations
            and a.error == b.error)


@pytest.mark.parametrize("name,maxit,tol", [("rmat16", 60, 1e-5), ("rmat16", 0, 1e-4), ("few_active", 60, 1e-5),
                                            ("few_active", 20, 0.0), ("no_edges", 60, 1e-5), ("no_edges", 5, 0.0)])
def test_page_rank_csr_equals_twin_path(gb, monkeypatch, name, maxit, tol):
    """two consecutive calls, then calls interleaved with page_rank on the same communicator (the barrier's
    sequence numbers carry over), from pageable and pinned arrays"""
    fx.set_knobs(monkeypatch, name)
    if name == "rmat16":
        n, out, inc = rmat16()
    elif name == "no_edges":
        n, out, inc = csrs([], [], 70)
    else:
        _, _, n, out, inc = fx.graph(name)
    g = twin(gb, out, inc)
    comm = gb.Comm([0])
    kw = dict(max_iterations=maxit, tolerance=tol)
    ref = comm.page_rank([g], **kw)
    _, wit, werr = oracle.page_rank_jacobi(inc[0], inc[1], out[0], maxit, tol, 0.85, acc64=True)
    assert ref.ran_iterations == wit
    host = (inc[0], inc[1], out[0])
    pin = tuple(pinned(a) for a in host)
    for _ in range(2):
        assert same(comm.page_rank_csr(*host, **kw), ref)
    for arrays in (pin, host, pin):
        assert same(comm.page_rank([g], **kw), ref)
        assert same(comm.page_rank_csr(*arrays, **kw), ref)
    assert same(comm.page_rank_csr(*pin, **kw), ref)


# ---- 3. errors -------------------------------------------------------------------------------------------------
def P(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def single_call(inc_off, inc_tgt, out_off, n):
    from graph_b200._capi import PageRankConfig, lib
    cfg = PageRankConfig(20, 0.0, 0.85, 2)
    scores = np.full(max(n, 1), SENTINEL, np.float32)
    it, err = C.c_uint64(0), C.c_double(0.0)
    st = lib.gb_page_rank_csr_u32(0, n, P(inc_off), P(inc_tgt), P(out_off), C.byref(cfg), P(scores), C.byref(it),
                                  C.byref(err))
    return st, (lib.gb_last_error() or b"").decode()


def multi_call(comm, inc_off, inc_tgt, out_off, n, maxit=20):
    from graph_b200._capi import PageRankConfig, lib
    cfg = PageRankConfig(maxit, 0.0, 0.85, 2)
    scores = np.full(max(n, 1), SENTINEL, np.float32)
    it, err = C.c_uint64(0), C.c_double(0.0)
    st = lib.gb_page_rank_csr_multi_u32(comm._c if comm is not None else None, n, P(inc_off), P(inc_tgt),
                                        P(out_off), C.byref(cfg), P(scores), C.byref(it), C.byref(err))
    return st, (lib.gb_last_error() or b"").decode(), scores


def shards_call(comm, v, inc_off, inc_tgt, out_off, n):
    """gb_pr_shards_csr_u32: (status, message); the shards are freed"""
    from graph_b200._capi import lib
    arr = (C.c_void_p * 16)()
    st = lib.gb_pr_shards_csr_u32(comm._c if comm is not None else None, v, n, P(inc_off), P(inc_tgt), P(out_off),
                                  arr)
    msg = (lib.gb_last_error() or b"").decode()
    made = [arr[i] for i in range(16) if arr[i]]
    for h in made:
        lib.gb_pr_shard_free(h)
    assert st == 0 or not made, "a failed call handed out shards"
    return st, msg


def part_rows(off, parts):
    """R_0 .. R_U of pr_split (csr_split.h) on monotone offsets"""
    m, n = int(off[-1]), len(off) - 1
    cuts = [0] + [int(np.searchsorted(off, m * u // parts, side="left")) for u in range(1, parts)] + [n]
    return [min(max(c, p), n) for c, p in zip(cuts, [0] + cuts[:-1])]


def test_errors_match_single_device_call(gb, comm):
    check_errors_match_single_device_call(comm)


def test_errors_match_streamed_single_device_call(gb, comm, monkeypatch):
    """rmat16 is below GB_PR_FEED_MIN_EDGES: lowered to 0, gb_page_rank_csr_u32 streams its targets in as it does
    from 2^22 edges up, and must reject every malformed input as the communicator calls do"""
    monkeypatch.setenv("GB_PR_FEED_MIN_EDGES", "0")
    check_errors_match_single_device_call(comm)


def check_errors_match_single_device_call(comm):
    n, out, inc = rmat16()
    io, it, oo = inc[0], inc[1], out[0]
    U = 4
    rows = part_rows(io, U)
    want_scores = comm.page_rank_csr(io, it, oo, max_iterations=20, tolerance=0.0).scores()

    def rejected(a, b, c, nn=n):
        st0, msg0 = single_call(a, b, c, nn)
        assert st0 == GB_ERR_INVALID, msg0
        st, msg, scores = multi_call(comm, a, b, c, nn)
        assert (st, msg) == (st0, msg0)
        assert (scores == SENTINEL).all()
        assert shards_call(comm, U, a, b, c, nn) == (st0, msg0)
        st, msg, scores = multi_call(comm, io, it, oo, n)  # the next good call succeeds
        assert st == 0 and scores.tobytes() == want_scores.tobytes(), msg
        return msg0

    assert "offset arrays are NULL" in rejected(None, it, oo)
    assert "offset arrays are NULL" in rejected(io, it, None)
    assert "in targets is NULL" in rejected(io, None, oo)
    assert "node_count must be > 0" in rejected(io, it, oo, 0)
    bad = oo.copy()
    bad[-1] -= 1
    assert "disagree on the edge count" in rejected(io, it, bad)
    for off, which in ((io, 0), (oo, 2)):
        bad = off.copy()
        bad[0] = 1
        args = [io, it, oo]
        args[which] = bad
        assert "offsets[0] must be 0" in rejected(*args)
    for u in range(U):
        r0, r1 = rows[u], rows[u + 1]
        assert r1 - r0 >= 3, rows
        r = (r0 + r1) // 2  # a decreasing offset inside part u: row r starts after row r + 1
        for which in (0, 2):
            args = [io, it, oo]
            bad = args[which].copy()
            bad[r] = bad[r + 1] + 1
            args[which] = bad
            assert "offsets are not monotone (1 rows)" in rejected(*args)
        e = (int(io[r0]) + int(io[r1])) // 2  # a target >= n inside part u
        t = it.copy()
        t[e] = n + u
        assert f"in CSR holds 1 targets >= node_count {n}" in rejected(io, t, oo)
    t = it.copy()
    t[[0, len(t) // 2, len(t) - 1]] = 0xFFFFFFFF
    assert f"in CSR holds 3 targets >= node_count {n}" in rejected(io, t, oo)


def test_invalid_comm_and_rank_counts(gb, comm):
    n, out, inc = csrs([0, 1], [1, 0], 2)
    args = (inc[0], inc[1], out[0], n)
    st, msg, scores = multi_call(None, *args)
    assert st == GB_ERR_INVALID and "comm is NULL" in msg and (scores == SENTINEL).all()
    assert shards_call(None, 1, *args)[0] == GB_ERR_INVALID
    assert shards_call(comm, 0, *args)[0] == GB_ERR_INVALID
    st, msg = shards_call(comm, 9, *args)
    assert st == GB_ERR_INVALID and "at most 8 ranks" in msg
    st, msg, scores = multi_call(comm, *args, maxit=0)  # tolerance 0: never terminates
    assert st == GB_ERR_INVALID and (scores == SENTINEL).all()
    assert shards_call(comm, 8, *args)[0] == 0
    st, msg, scores = multi_call(comm, *args)
    assert st == 0, msg


# ---- 4. two devices ----------------------------------------------------------------------------------------------
def test_two_devices_equal_twin_path(gb):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    src, dst = oracle.rmat_edges(18, seed=42)
    n, out, inc = csrs(src, dst, 1 << 18)
    graphs = []
    for d in (0, 1):
        gb.set_device(d)
        graphs.append(twin(gb, out, inc))
    gb.set_device(0)
    comm = gb.Comm([0, 1])
    for maxit, tol in ((20, 0.0), (60, 1e-5)):
        want, wit, werr = oracle.page_rank_jacobi(inc[0], inc[1], out[0], maxit, tol, 0.85, acc64=True)
        ref = comm.page_rank(graphs, max_iterations=maxit, tolerance=tol)
        got = comm.page_rank_csr(inc[0], inc[1], out[0], max_iterations=maxit, tolerance=tol)
        assert same(got, ref) and got.ran_iterations == wit
        assert rel_err(got.scores(), want) <= PR_RTOL
