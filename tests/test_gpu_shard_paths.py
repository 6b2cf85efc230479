"""The sharded PageRank and WCC paths on one GPU, with P virtual ranks (tests/virtual_ranks.py): the peer
stores of k_pr_sell / k_pr_finish (PEERS = true), the device barrier and rank-order error sum of k_pr_sync
with P > 1, shards that own few or no rows, the stop rule and sequence numbers of gb_page_rank_multi, and
the WCC shard phases on empty vertex ranges.  Every case runs the ranks one after another, so none depends
on two kernels being resident at once.  Each shard's launch shape is checked against the layout model
(tools/layout_model.py) before its numbers are."""
import os
import sys
import time

import numpy as np
import pytest

import oracle
import pr_path_fixtures as fx

pytestmark = pytest.mark.gpu

lm = fx.lm
PR_RTOL = 1e-6
ERR_ATOL = 2e-6          # as test_gpu_parity.py
SHARD_RTOL = 5e-7        # sharded vs single-GPU ranks, as test_shard_api_virtual_ranks_match_single_gpu
SWEEPS = 6
SHAPE_KEYS = ("hot_blocks", "n_cb", "n_fin", "n_fin_warp", "fin_u", "grid_sell", "grid_fin", "fin_hub_ctas",
              "n_mega", "dual", "last_hot_block")


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


_GRAPHS: dict = {}


def graph(name):
    """(n, out CSR, in CSR) of a fixture of pr_path_fixtures.py or of RMAT-15 (seed 11), Sorted layout"""
    if name in fx.FIXTURES:
        _, _, n, out, inc = fx.graph(name)
        return n, out, inc
    if name not in _GRAPHS:
        assert name == "rmat15"
        src, dst = oracle.rmat_edges(15, seed=11)
        n = 1 << 15
        _GRAPHS[name] = (n, oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED),
                         oracle.csr_build(src, dst, n, oracle.INCOMING, oracle.SORTED))
    return _GRAPHS[name]


def device_graph(gb, n, out, inc):
    return gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])


def shard_model(n, out, inc, block, P, p, sms, **knobs):
    plan = lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)),
                        lm.clamp_block(block or lm.CB_BLOCK_DEFAULT), lm.CB_TAU_DEFAULT, P=P, p=p)
    return plan, lm.launch_shape(plan, sms=sms, **knobs)


def assert_shard_shapes(vr, n, out, inc, block, sms, **knobs):
    """every shard's launch shape is the layout model's; returns the device shapes"""
    shapes = []
    for p, b in enumerate(vr.ranks):
        _, want = shard_model(n, out, inc, block, vr.world, p, sms, **knobs)
        got = b.plan_shape()
        assert {k: got[k] for k in SHAPE_KEYS} == {k: want[k] for k in SHAPE_KEYS}, (p, got, want)
        got["n_loc"] = b.stats["local_rows"]
        shapes.append(got)
    return shapes


def rel_err(got, want):
    return float(np.max(np.abs(got.astype(np.float64) - want) / want)) if len(want) else 0.0


# ---- 1. fused peer stores vs the host-copy exchange --------------------------------------------------------
# (graph, knobs): what the shards reach is asserted by check_peer_path
PEER_CASES = [
    ("rmat15", {}),
    ("rmat18", {}),
    ("rmat18", {"GB_PR_FIN_U": 4}),
    ("capped_finish", {"GB_PR_FIN_U": 2}),
    ("capped_finish", {"GB_PR_FIN_SPLIT": 1}),
    ("tail_r33", {}),
    ("few_active", {}),
]


def check_peer_path(name, env, shapes):
    """the sweep paths the case exists for, on the device shapes of its shards; returns a description"""
    lane_done = [s["n_loc"] - s["n_fin"] for s in shapes]     # rows completed by their k_pr_sell lane
    hub = [s["n_fin_warp"] for s in shapes]                   # rows of the hub-group branch of k_pr_finish
    tail = [s["n_fin"] - s["n_fin_warp"] for s in shapes]     # rows of its per-lane branch
    u = {s["fin_u"] for s in shapes if s["n_fin"]}
    if name == "rmat15":
        assert all(lane_done)
    elif name == "rmat18":
        assert any(hub) and all(tail) and all(lane_done) and u == {env.get("GB_PR_FIN_U", 2)}
    elif name == "capped_finish":
        assert hub[0] == 32 and all(tail) and not any(lane_done) and u == {2}
        if env.get("GB_PR_FIN_SPLIT") == 1:
            assert shapes[0]["fin_hub_ctas"] == 1
    elif name == "tail_r33":
        assert shapes[0]["hot_blocks"] > lm.SELL_FEW and tail[0] and all(lane_done)
        assert all(s["hot_blocks"] == 0 for s in shapes[1:])
    elif name == "few_active":
        assert hub[0] == shapes[0]["n_fin"] == 20 and all(s["n_loc"] == 0 for s in shapes[1:])
    return f"lane rows {lane_done}, hub rows {hub}, finish tail rows {tail}, fin_u {sorted(u)}"


def poison_next(vr):
    """NaN into the active rows of every rank's next vector: the coming sweep must store each of them again
    (a missed store would otherwise leave an equal value behind, e.g. the +inf of a row without out-edges)"""
    nxt = (vr.sweep + 1) & 1
    for x in vr.x:
        x[nxt][: vr.n_active] = float("nan")


_ORACLE: dict = {}


def oracle_pr(name, n, out, inc, sweeps, tol):
    key = (name, sweeps, tol)
    if key not in _ORACLE:
        _ORACLE.clear()
        _ORACLE[key] = oracle.page_rank_jacobi(inc[0], inc[1], out[0], sweeps, tol, 0.85, acc64=True)
    return _ORACLE[key]


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("name,env", PEER_CASES,
                         ids=[f"{c}-" + "-".join(f"{k}={v}" for k, v in e.items()) for c, e in PEER_CASES])
def test_peer_stores_equal_host_exchange(gb, sms, monkeypatch, name, env, world):
    import torch
    from virtual_ranks import VirtualRanks
    if name == "capped_finish" and sms != lm.H100_SMS:
        pytest.skip("the fixture is sized for 132 SMs")
    fx.set_knobs(monkeypatch, name, **env)
    block = fx.FIXTURES[name][1] if name in fx.FIXTURES else None
    n, out, inc = graph(name)
    g = device_graph(gb, n, out, inc)
    vr = VirtualRanks(g, world)
    knobs = {"fin_u": env.get("GB_PR_FIN_U", 0), "fin_split": env.get("GB_PR_FIN_SPLIT", 0)}
    print(check_peer_path(name, env, assert_shard_shapes(vr, n, out, inc, block, sms, **knobs)))
    # (a) host copies after every sweep: the reference for (b)
    vr.init()
    host = []
    for _ in range(SWEEPS):
        poison_next(vr)
        shares = vr.step(peers=False)
        x = vr.x_next()[0].cpu().numpy()
        assert not np.isnan(x).any()
        host.append((shares, x.tobytes()))
    host_scores = torch.stack(vr.scores).cpu().numpy()
    # (b) every rank stores its rows into the other ranks' x_next itself
    vr.init()
    total = 0.0
    for sweep in range(SWEEPS):
        poison_next(vr)
        shares = vr.step(peers=True)
        assert shares == host[sweep][0], sweep                 # the same f64 bits, rank by rank
        for r, x in enumerate(vr.x_next()):
            assert x.cpu().numpy().tobytes() == host[sweep][1], (sweep, r)
        total = 0.0
        for e in shares:
            total += e
    assert torch.stack(vr.scores).cpu().numpy().tobytes() == host_scores.tobytes()
    got = vr.scores_host()
    want = g.page_rank(max_iterations=SWEEPS, tolerance=0.0, mode="jacobi")
    assert rel_err(got, want.scores()) <= SHARD_RTOL
    assert abs(total - want.error) <= 1e-7 + 1e-6 * want.error
    ref, it, err = oracle_pr(name, n, out, inc, SWEEPS, 0.0)
    assert rel_err(got, ref) <= PR_RTOL
    assert abs(total - err) <= ERR_ATOL


# ---- 2. k_pr_sync: the device barrier and the rank-order error sum -----------------------------------------
BARRIER_WAIT_S = 30.0


def wait_bounded(what):
    """wait for the current stream for at most BARRIER_WAIT_S.  A barrier that does not return is broken:
    the test process ends at once, so that its CUDA context (and the spinning kernel) goes away."""
    import torch
    stream = torch.cuda.current_stream()
    t0 = time.monotonic()
    while not stream.query():
        if time.monotonic() - t0 > BARRIER_WAIT_S:
            sys.stderr.write(f"\nFAILED: {what} did not return within {BARRIER_WAIT_S:.0f} s (k_pr_sync is "
                             "waiting for an arrival that was already there); ending the test process\n")
            sys.stderr.flush()
            os._exit(1)
        time.sleep(1e-3)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_device_barrier_on_one_gpu(gb, monkeypatch, world):
    """The syncs run one at a time in rank order.  Before rank r's, r's control block gets the arrival
    (sweep_no + 1000: ahead, so a correct kernel never waits) and the true error share of every rank q > r
    that has not published yet; ranks q < r have published into it already."""
    import torch
    from virtual_ranks import VirtualRanks
    fx.set_knobs(monkeypatch, "rmat15")
    n, out, inc = graph("rmat15")
    vr = VirtualRanks(device_graph(gb, n, out, inc), world)
    dev = vr.ranks[0].device
    # one 192-byte block per rank: arrive[8] (u32), then errs[2][8] (f64)
    blocks = torch.zeros((world, 24), dtype=torch.float64, device=dev)
    arrive = blocks[:, :4].view(torch.int32)
    errs = blocks[:, 4:20]
    ptrs = [blocks[r].data_ptr() for r in range(world)]
    total_err = [torch.zeros(64, dtype=torch.float64, device=dev) for _ in range(world)]
    prev = [0.0] * world
    seq0 = 0
    for sweeps in (4, 3):           # a second run continues the sequence numbers, as gb_page_rank_multi does
        vr.init()
        for sweep in range(1, sweeps + 1):
            shares = vr.step(peers=world > 1)
            seq, slot = seq0 + sweep, sweep % 64
            bank = seq & 1
            for r, b in enumerate(vr.ranks):
                for q in range(r + 1, world):
                    arrive[r, q] = seq + 1000
                    errs[r, 8 * bank + q] = shares[q]
                b.sync(seq, vr.err[r], ptrs[r], ptrs, total_err[r], slot)
                wait_bounded(f"k_pr_sync of rank {r} of {world} at sweep {seq}")
            h = blocks.cpu().numpy()
            seen = h[:, :4].copy().view(np.uint32)
            e = h[:, 4:20].reshape(world, 2, 8)
            assert (seen[:, :world] == seq).all(), seen           # the publications overwrote the seeds
            assert (seen[:, world:] == 0).all()
            want = 0.0
            for s in shares:
                want += s
            for r in range(world):
                assert e[r, bank, :world].tolist() == shares, (r, seq)
                assert e[r, 1 - bank, :world].tolist() == prev, (r, seq)   # last sweep's bank untouched
                assert total_err[r][slot].item() == want, (r, seq)
            prev = shares
        seq0 += sweeps


# ---- 3. shards with few or no rows ------------------------------------------------------------------------
FEW_N = 6 * 1024 + 5            # not a multiple of 32 P for P = 3 or 8; 7 blocks of 1024
FEW_TOL = 1e-7


def few_rows(k, n=FEW_N):
    """k rows with in-edges (in-degrees 1..40, sources anywhere), all other rows without; k = 0: m = 0.
    With k <= 32 every row with edges lies in the first 32-row slice."""
    rng = np.random.default_rng(1000 + k)
    rows = rng.choice(n, k, replace=False).astype(np.uint32)
    dst = np.repeat(rows, rng.integers(1, 41, k))
    src = rng.integers(0, n, len(dst)).astype(np.uint32)
    return (n, oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED),
            oracle.csr_build(src, dst, n, oracle.INCOMING, oracle.SORTED))


FEW_CASES = [(P, k) for P in (3, 8) for k in (0, 1, 20, 31, 33, 32 * P - 1, 32 * P + 1)]


@pytest.mark.parametrize("world,k", FEW_CASES)
def test_shards_with_few_or_no_rows(gb, sms, monkeypatch, world, k):
    fx.set_knobs(monkeypatch, "few_rows", GB_PR_BLOCK=1024)
    from virtual_ranks import VirtualRanks
    n, out, inc = few_rows(k)
    g = device_graph(gb, n, out, inc)
    vr = VirtualRanks(g, world)
    assert vr.n_active == k
    local = [b.stats["local_rows"] for b in vr.ranks]
    assert local == [lm.deal_count(k, world, p) for p in range(world)] and sum(local) == k
    shapes = assert_shard_shapes(vr, n, out, inc, 1024, sms)
    for s in shapes:
        if s["n_loc"] == 0:
            assert s["grid_sell"] == 0 and s["grid_fin"] == 1 and s["hot_blocks"] == 0 and s["n_fin"] == 0
    assert any(s["n_loc"] == 0 for s in shapes) or k > 32 * (world - 1)
    # sweep 1: the closed-form error of the rows without in-edges is added once (rank 0), not per rank
    one = g.page_rank(max_iterations=1, tolerance=0.0, mode="jacobi")
    e1 = vr.run(1, peers=True)
    assert abs(e1 - one.error) <= 1e-7 + 1e-6 * one.error, (e1, one.error)
    assert rel_err(vr.scores_host(), one.scores()) <= SHARD_RTOL
    for sweeps, tol in ((SWEEPS, 0.0), (200, FEW_TOL)):
        want = g.page_rank(max_iterations=sweeps, tolerance=tol, mode="jacobi")
        total = vr.run(sweeps, tol, peers=True)
        assert vr.sweep == want.ran_iterations, (tol, vr.sweep, want.ran_iterations)
        assert rel_err(vr.scores_host(), want.scores()) <= SHARD_RTOL
        assert abs(total - want.error) <= 1e-7 + 1e-6 * want.error, (tol, total, want.error)
    import torch
    torch.cuda.synchronize()


# ---- 4. gb_page_rank_multi on one device ------------------------------------------------------------------
def comm_graph(name):
    if name == "rmat16":
        src, dst = oracle.rmat_edges(16, seed=42)
        n = 1 << 16
        return (n, oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED),
                oracle.csr_build(src, dst, n, oracle.INCOMING, oracle.SORTED))
    if name == "no_edges":
        return few_rows(0)
    return graph(name)


@pytest.mark.parametrize("name,maxit,tol", [("rmat16", 60, 1e-5), ("rmat16", 0, 1e-4), ("few_active", 60, 1e-5),
                                            ("few_active", 20, 0.0), ("no_edges", 60, 1e-5), ("no_edges", 5, 0.0)])
def test_page_rank_multi_one_device(gb, monkeypatch, name, maxit, tol):
    """two consecutive calls on one communicator: the second continues the barrier's sequence numbers"""
    fx.set_knobs(monkeypatch, name)
    n, out, inc = comm_graph(name)
    g = device_graph(gb, n, out, inc)
    want, it, err = oracle.page_rank_jacobi(inc[0], inc[1], out[0], maxit, tol, 0.85, acc64=True)
    comm = gb.Comm([0])
    first = None
    for call in range(2):
        pr = comm.page_rank([g], max_iterations=maxit, tolerance=tol)
        assert pr.ran_iterations == it, (call, pr.ran_iterations, it)
        assert rel_err(pr.scores(), want) <= PR_RTOL, call
        assert abs(pr.error - err) <= ERR_ATOL, (call, pr.error, err)
        if first is None:
            first = pr
        else:
            assert pr.scores().tobytes() == first.scores().tobytes() and pr.error == first.error


# ---- 5. WCC shard phases on empty vertex ranges ------------------------------------------------------------
def wcc_graph(n):
    if n == 4096:
        src, dst = oracle.rmat_edges(12, seed=3)
    else:   # n / 2 random edges and a self loop: several components, isolated vertices
        rng = np.random.default_rng(n)
        src = np.append(rng.integers(0, n, n // 2), n - 1).astype(np.uint32)
        dst = np.append(rng.integers(0, n, n // 2), n - 1).astype(np.uint32)
    return (n, oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED),
            oracle.csr_build(src, dst, n, oracle.INCOMING, oracle.SORTED))


@pytest.mark.parametrize("rounds,samples", [(2, 1024), (0, 1024), (2, 0), (1, 16)])
@pytest.mark.parametrize("n", [40, 100, 257, 4096])
def test_wcc_shard_phases_empty_ranges(gb, n, rounds, samples):
    from graph_b200.multigpu import vertex_ranges
    from virtual_ranks import wcc_virtual_ranks
    world = 8
    n, out, inc = wcc_graph(n)
    if n in (40, 100):
        assert any(vb == ve for vb, ve in vertex_ranges(n, world))
    want = oracle.wcc_min_label(out[0], out[1])
    g = device_graph(gb, n, out, inc)
    parents, labels = wcc_virtual_ranks(g, world, neighbor_rounds=rounds, sampling_size=samples)
    assert len(set(labels)) == 1 and labels[0][1] == (samples > 0)
    for r, p in enumerate(parents):
        assert (p.cpu().numpy().view(np.uint32) == want).all(), r


# ---- shard lifetime ---------------------------------------------------------------------------------------
def test_shard_freed_after_its_graph(gb):
    # regression: gb_pr_shard_free read the device of a graph that may be freed already (a garbage collector
    # finalizes a cycle holding both in any order); the failed cudaSetDevice left an error for the next call
    import ctypes as C
    import torch
    from graph_b200._capi import check, lib
    from virtual_ranks import VirtualRanks
    keep = VirtualRanks(gb.DiGraph.rmat(10, seed=2), 2)       # used after the frees
    g = gb.DiGraph.rmat(10, seed=1)
    shards = [C.c_void_p() for _ in range(4)]
    for r, sh in enumerate(shards):
        check(lib.gb_pr_shard_create(g._g, r, len(shards), C.byref(sh)))
    raw, g._g = g._g, None
    check(lib.gb_graph_free(raw))
    for sh in shards:
        check(lib.gb_pr_shard_free(sh))
    keep.run(3, peers=True)     # gb_pr_shard_init / _step end with a cudaGetLastError check
    torch.cuda.synchronize()
