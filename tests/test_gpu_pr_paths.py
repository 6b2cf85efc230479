"""The JACOBI PageRank sweep on graphs built to reach its less common paths (tests/pr_path_fixtures.py):
the partial last column block (scalar tail of the block load), a rectangular staircase, a mega row cut by
chunk boundaries, a repeated source, fewer than 32 active rows, the hub-group CTAs of k_pr_finish, its
FIN_U = 4 instantiation, its role split, a capped finish grid, the GB_PR_TASK_CHUNKS variant, and x vectors
that are not 16-byte aligned.  Every case asserts that the device plan took the path (against the layout
model), that the ranks match the f64-accumulating oracle, and that runs and arithmetic-preserving variants
give the same bits."""
import ctypes as C

import numpy as np
import pytest

import oracle
import pr_path_fixtures as fx

pytestmark = pytest.mark.gpu

PR_RTOL = 1e-6
ERR_ATOL = 2e-6          # as test_gpu_parity.py
SWEEPS = 10
set_knobs = fx.set_knobs
SHAPE_KEYS = ("hot_blocks", "n_cb", "n_fin", "n_fin_warp", "fin_u", "grid_fin", "fin_hub_ctas", "n_mega", "dual",
              "last_hot_block")


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def oracle_pr(name, sweeps, tol):
    _, _, n, out, inc = fx.graph(name)
    return oracle.page_rank_jacobi(inc[0], inc[1], out[0], sweeps, tol, 0.85, acc64=True)


def device_graph(gb, name):
    _, _, n, out, inc = fx.graph(name)
    return gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])


def assert_shape(g, name, sms, P=1, p=0, **knobs):
    """(a): the device plan's launch shape and layout statistics are the model's"""
    plan, want, counts = fx.model(name, P=P, p=p, sms=sms, **knobs)
    shape, info = g.page_rank_plan_shape(), g.page_rank_plan_info()
    assert {k: shape[k] for k in SHAPE_KEYS} == {k: want[k] for k in SHAPE_KEYS}, name
    assert info["hot_blocks"] == want["hot_blocks"]
    assert {k: info[k] for k in counts} == counts, name
    return plan, {**want, **shape}, info


def assert_matches_oracle(pr, name, sweeps, tol):
    """(b): ranks within 1e-6 of the f64 oracle, same sweep count, error within ERR_ATOL"""
    want, it, err = oracle_pr(name, sweeps, tol)
    assert pr.ran_iterations == it, (name, pr.ran_iterations, it)
    rel = np.abs(pr.scores() - want) / want
    assert rel.max() <= PR_RTOL, (name, rel.max(), int(rel.argmax()))
    assert abs(pr.error - err) <= ERR_ATOL, (name, pr.error, err)


def run(g, sweeps=SWEEPS, tol=0.0):
    return g.page_rank(max_iterations=sweeps, tolerance=tol, mode="jacobi")


def assert_same_bits(a, b, what):
    """(d): same scores bit for bit; the error sums per-CTA partials, which the variants regroup"""
    assert a.ran_iterations == b.ran_iterations, what
    assert a.scores().tobytes() == b.scores().tobytes(), what
    assert abs(a.error - b.error) <= 1e-12 * abs(b.error), (what, a.error, b.error)


@pytest.mark.parametrize("name", list(fx.FIXTURES))
def test_fixture_path_ranks_and_determinism(gb, sms, monkeypatch, name):
    set_knobs(monkeypatch, name)
    g = device_graph(gb, name)
    plan, shape, info = assert_shape(g, name, sms)
    assert info["chunks"] == len(fx.chunks(name, sms))                # the chunk table of the model
    if sms == fx.lm.H100_SMS:
        fx.check_path(name, plan, shape)
    pr = run(g)
    assert_matches_oracle(pr, name, SWEEPS, 0.0)
    assert run(g).scores().tobytes() == pr.scores().tobytes()        # (c)
    # the stop rule evaluated on the device
    pr = run(g, 60, 1e-5)
    assert pr.ran_iterations < 60
    assert_matches_oracle(pr, name, 60, 1e-5)
    if name == "star_in":
        assert info["cut_segments"] > 0 and shape["n_fix"] > 0          # at the default knobs


@pytest.mark.parametrize("r", fx.TAIL_R)
def test_tail_block_loads_and_streamed_upload(gb, monkeypatch, r):
    import torch
    from graph_b200 import _capi
    from graph_b200._capi import check, lib
    from graph_b200.multigpu import CudaShardBackend
    name = f"tail_r{r}"
    set_knobs(monkeypatch, name)
    g = device_graph(gb, name)
    want = run(g)
    _, _, n, out, inc = fx.graph(name)
    # a one-rank shard whose x vectors start one float past a 16-byte boundary: no TMA, element-wise block loads
    b = CudaShardBackend(g, 0, 1)
    x = [torch.zeros(n + 4, dtype=torch.float32, device=b.device)[1:n + 1] for _ in range(2)]
    assert all(v.data_ptr() % 16 == 4 for v in x)
    scores = torch.empty(n, dtype=torch.float32, device=b.device)
    err = torch.zeros(1, dtype=torch.float64, device=b.device)
    b.init(0.85, x[0], x[1], scores)
    for sweep in range(1, SWEEPS + 1):
        b.step(0.85, sweep, x[(sweep - 1) & 1], x[sweep & 1], None, scores, err)
    assert b.finish(scores).cpu().numpy().tobytes() == want.scores().tobytes()
    assert abs(err.item() - want.error) <= 1e-12 * abs(want.error)
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


# GB_PR_FIN_U 2 vs 4 and the role split keep every row's f64 sum in the same block order: all bit-equal to
# the automatic plan
BIT_EQUAL = [
    ({"GB_PR_FIN_U": 4}, {"fin_u": 4}),
    ({"GB_PR_FIN_SPLIT": 1}, {"fin_split": 1}),
    ({"GB_PR_FIN_U": 4, "GB_PR_FIN_SPLIT": 1}, {"fin_u": 4, "fin_split": 1}),
    ({"GB_PR_FIN_SPLIT": 2}, {"fin_split": 2}),
]


@pytest.mark.parametrize("env,knobs", BIT_EQUAL, ids=lambda v: "-".join(f"{k}={x}" for k, x in v.items()) or "model")
def test_rmat18_finish_variants_bit_equal(gb, sms, monkeypatch, env, knobs):
    set_knobs(monkeypatch, "rmat18")
    want = run(device_graph(gb, "rmat18"))
    set_knobs(monkeypatch, "rmat18", **env)
    g = device_graph(gb, "rmat18")
    _, shape, _ = assert_shape(g, "rmat18", sms, **knobs)
    if "fin_split" in knobs and knobs["fin_split"] == 1:
        assert shape["fin_hub_ctas"] == shape["n_fin_warp"] // 32 > 0
    assert_same_bits(run(g), want, env)


def test_rmat18_task_chunks(gb, sms, monkeypatch):
    """GB_PR_TASK_CHUNKS regroups chunks into tasks; with the chunk size fixed, the segments are cut at the
    same places and the ranks are bit-equal.  Without it the default chunk size follows the task size."""
    set_knobs(monkeypatch, "rmat18", GB_PR_CHUNK=512)
    want = run(device_graph(gb, "rmat18"))
    for t in (64, 128):
        set_knobs(monkeypatch, "rmat18", GB_PR_CHUNK=512, GB_PR_TASK_CHUNKS=t)
        assert_same_bits(run(device_graph(gb, "rmat18")), want, t)
    set_knobs(monkeypatch, "rmat18", GB_PR_TASK_CHUNKS=128)
    g = device_graph(gb, "rmat18")
    assert g.page_rank_plan_info()["chunk_groups"] != 512
    assert_matches_oracle(run(g), "rmat18", SWEEPS, 0.0)


def test_capped_finish_grid(gb, sms, monkeypatch):
    """GB_PR_FIN_U=2 caps the finish grid on this graph (warps walk several row groups), with and without a
    forced role split; the rows' sums are those of the automatic FIN_U = 4 plan, bit for bit"""
    if sms != fx.lm.H100_SMS:
        pytest.skip("the fixture is sized for 132 SMs")
    set_knobs(monkeypatch, "capped_finish")
    want = run(device_graph(gb, "capped_finish"))
    for env, knobs, hub in (({"GB_PR_FIN_U": 2}, {"fin_u": 2}, 0),
                            ({"GB_PR_FIN_U": 2, "GB_PR_FIN_SPLIT": 1}, {"fin_u": 2, "fin_split": 1}, 1),
                            ({"GB_PR_FIN_SPLIT": 1}, {"fin_split": 1}, 1)):
        set_knobs(monkeypatch, "capped_finish", **env)
        g = device_graph(gb, "capped_finish")
        _, shape, _ = assert_shape(g, "capped_finish", sms, **knobs)
        assert shape["fin_hub_ctas"] == hub
        if knobs.get("fin_u") == 2:
            assert shape["grid_fin"] == 8 * sms
        assert_same_bits(run(g), want, env)


@pytest.mark.parametrize("world", [2, 3])
def test_split_on_virtual_rank_shards(gb, sms, monkeypatch, world):
    """the harness of test_shard_api_virtual_ranks_match_single_gpu with the role split forced on every
    shard of RMAT-18 (where production uses the split: a shard of a large graph)"""
    from virtual_ranks import VirtualRanks
    set_knobs(monkeypatch, "rmat18")
    g = device_graph(gb, "rmat18")
    sweeps, damping = 6, 0.85
    want = g.page_rank(max_iterations=sweeps, tolerance=0.0, damping_factor=damping, mode="jacobi")
    monkeypatch.setenv("GB_PR_FIN_SPLIT", "1")
    vr = VirtualRanks(g, world, damping)
    for r, b in enumerate(vr.ranks):
        shape = b.plan_shape()
        _, model, _ = fx.model("rmat18", P=world, p=r, sms=sms, fin_split=1)
        assert {k: shape[k] for k in SHAPE_KEYS} == {k: model[k] for k in SHAPE_KEYS}
        assert shape["fin_hub_ctas"] > 0
    total = vr.run(sweeps)
    got = vr.scores_host()
    assert np.max(np.abs(got - want.scores()) / want.scores()) <= 5e-7
    assert abs(total - want.error) <= 1e-7 + 1e-6 * want.error
