"""The JACOBI PageRank sweep with its cold edges reduced through virtual blocks (pass A bins the source values
of every (source, partition) pair into V, pass B walks a column-block stream over V) instead of k_pr_sell.
GB_PR_VBLOCKS=1 builds them on the small graphs of tests/pr_path_fixtures.py that have cold edges
(tests/vblock_fixtures.py), which the automatic choice leaves on the SELL path (their source vectors fit in
L2); every case asserts that the path was built, with the layout model's partition, pair and edge counts.  Every case checks the ranks against the f64
oracle, that repeated runs give the same bits, that the streamed one-shot build gives the resident twin's
bits, and that the SELL path of the same graph agrees to the rounding of the reordered sums."""
import ctypes as C

import numpy as np
import pytest

import oracle
import pr_path_fixtures as fx
import vblock_fixtures as vf

pytestmark = pytest.mark.gpu

PR_RTOL = 1e-6
ERR_ATOL = 2e-6
SWEEPS = 10


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


def device_graph(gb, name):
    _, _, n, out, inc = fx.graph(name)
    return gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])


def run(g, sweeps=SWEEPS, tol=0.0):
    return g.page_rank(max_iterations=sweeps, tolerance=tol, mode="jacobi")


def assert_matches_oracle(pr, name, sweeps, tol):
    _, _, n, out, inc = fx.graph(name)
    want, it, err = oracle.page_rank_jacobi(inc[0], inc[1], out[0], sweeps, tol, 0.85, acc64=True)
    assert pr.ran_iterations == it, (name, pr.ran_iterations, it)
    rel = np.abs(pr.scores() - want) / want
    assert rel.max() <= PR_RTOL, (name, rel.max(), int(rel.argmax()))
    assert abs(pr.error - err) <= ERR_ATOL, (name, pr.error, err)


VB_KEYS = ("vblock_parts", "vblock_pairs", "vblock_edges")


def vblock_plan(g, name, tau=fx.lm.CB_TAU_DEFAULT):
    """the plan took the virtual blocks, with the model's counts, and k_pr_sell does not run"""
    info = g.page_rank_plan_info()
    assert info["vblock_parts"] > 0, (name, info)
    assert {k: info[k] for k in VB_KEYS} == vf.model_counts(name, tau=tau), name
    assert info["vblock_edges"] == info["local_edges"] - info["block_edges"]
    assert g.page_rank_plan_shape()["grid_sell"] == 0
    return info


@pytest.mark.parametrize("name", vf.VB_FIXTURES)
def test_vblocks_ranks_determinism_and_sell_agreement(gb, monkeypatch, name):
    fx.set_knobs(monkeypatch, name, GB_PR_VBLOCKS=2)
    sell = run(device_graph(gb, name))
    fx.set_knobs(monkeypatch, name, GB_PR_VBLOCKS=1)
    g = device_graph(gb, name)
    vblock_plan(g, name)
    pr = run(g)
    assert_matches_oracle(pr, name, SWEEPS, 0.0)
    assert run(g).scores().tobytes() == pr.scores().tobytes()
    rel = np.abs(pr.scores() - sell.scores()) / sell.scores()
    assert rel.max() <= PR_RTOL, (name, rel.max())
    pr = run(g, 60, 1e-5)
    assert_matches_oracle(pr, name, 60, 1e-5)


def test_vblocks_reach_partitions_and_rows_without_cold_edges(gb, monkeypatch):
    """rmat18 at its fixture block size: many partitions, hot rows with 1-4 and more blocks, rows whose every
    edge lies in a segment (a padding group in pass B)"""
    fx.set_knobs(monkeypatch, "rmat18", GB_PR_VBLOCKS=1)
    g = device_graph(gb, "rmat18")
    info = vblock_plan(g, "rmat18")
    assert info["vblock_parts"] > 1 and info["hot_blocks"] > 4
    assert info["vblock_pairs"] < info["vblock_edges"]  # some sources feed several rows of one partition
    assert g.page_rank_plan_shape()["n_fin"] == info["local_rows"]  # k_pr_finish completes every row
    assert_matches_oracle(run(g), "rmat18", SWEEPS, 0.0)


@pytest.mark.parametrize("name", ["rmat18", "tail_r1"])
def test_vblocks_streamed_one_shot_matches_resident(gb, monkeypatch, name):
    from graph_b200 import _capi
    from graph_b200._capi import check, lib
    fx.set_knobs(monkeypatch, name, GB_PR_VBLOCKS=1)
    g = device_graph(gb, name)
    vblock_plan(g, name)
    want = run(g)
    _, _, n, out, inc = fx.graph(name)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    monkeypatch.setenv("GB_PR_FEED_MIN_EDGES", "0")
    for chunks in (1, 7):
        monkeypatch.setenv("GB_PR_FEED_CHUNKS", str(chunks))
        cfg = _capi.PageRankConfig(SWEEPS, 0.0, 0.85, _capi.PR_JACOBI)
        scores = np.empty(n, np.float32)
        it, err = C.c_uint64(0), C.c_double(0.0)
        check(lib.gb_page_rank_csr_u32(0, n, P(inc[0]), P(inc[1]), P(out[0]), C.byref(cfg), P(scores), C.byref(it),
                                       C.byref(err)))
        assert it.value == SWEEPS and scores.tobytes() == want.scores().tobytes() and err.value == want.error, chunks


@pytest.mark.parametrize("peers", [False, True])
@pytest.mark.parametrize("world", [2, 5])
def test_vblocks_virtual_rank_shards(gb, monkeypatch, world, peers):
    """every rank builds the partitions of its own rows; with the host exchange or the fused peer stores the
    ranks' scores match the oracle"""
    from virtual_ranks import VirtualRanks
    name = "rmat18"
    fx.set_knobs(monkeypatch, name, GB_PR_VBLOCKS=1)
    g = device_graph(gb, name)
    _, _, n, out, inc = fx.graph(name)
    vr = VirtualRanks(g, world)
    for p, r in enumerate(vr.ranks):
        assert {k: r.stats[k] for k in VB_KEYS} == vf.model_counts(name, P=world, p=p)
        assert r.stats["vblock_parts"] > 0
    vr.run(SWEEPS, 0.0, peers=peers)
    want, _, _ = oracle.page_rank_jacobi(inc[0], inc[1], out[0], SWEEPS, 0.0, 0.85, acc64=True)
    rel = np.abs(vr.scores_host() - want) / want
    assert rel.max() <= PR_RTOL, rel.max()


def test_vblocks_without_hot_blocks(gb, monkeypatch):
    """GB_PR_TAU=0: no column block, every edge reduced through the virtual blocks, no k_pr_cb launch"""
    name, knobs = vf.NO_HOT
    fx.set_knobs(monkeypatch, name, GB_PR_VBLOCKS=1, **knobs)
    g = device_graph(gb, name)
    info = vblock_plan(g, name, tau=knobs["GB_PR_TAU"])
    assert info["hot_blocks"] == 0 and info["block_edges"] == 0
    pr = run(g)
    assert_matches_oracle(pr, name, SWEEPS, 0.0)
    assert run(g).scores().tobytes() == pr.scores().tobytes()


def test_row_with_more_than_b_cold_edges_keeps_sell(gb, monkeypatch):
    """star_in without column blocks: the hub row's 2e5 cold edges do not fit one virtual block, so the graph
    keeps the SELL path even under GB_PR_VBLOCKS=1: the same plan and bits as with the virtual blocks off.
    (Its hub row is one SELL lane's serial f32 sum of 2e5 edges, 4e-5 from the f64 oracle: the other rows are
    held to the usual 1e-6.)"""
    name, knobs = vf.FALLBACK
    fx.set_knobs(monkeypatch, name, GB_PR_VBLOCKS=2, **knobs)
    sell = run(device_graph(gb, name))
    fx.set_knobs(monkeypatch, name, GB_PR_VBLOCKS=1, **knobs)
    g = device_graph(gb, name)
    info = g.page_rank_plan_info()
    assert {k: info[k] for k in VB_KEYS} == {k: 0 for k in VB_KEYS}
    assert g.page_rank_plan_shape()["grid_sell"] > 0
    pr = run(g)
    assert pr.scores().tobytes() == sell.scores().tobytes() and pr.error == sell.error
    _, _, n, out, inc = fx.graph(name)
    want, it, _ = oracle.page_rank_jacobi(inc[0], inc[1], out[0], SWEEPS, 0.0, 0.85, acc64=True)
    rel = np.abs(pr.scores() - want) / want
    assert pr.ran_iterations == it and rel[1:].max() <= PR_RTOL and rel[0] <= 1e-4, (rel[1:].max(), rel[0])
