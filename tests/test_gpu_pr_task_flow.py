"""k_pr_cb's chunk flow: inside a source block the warps of a CTA claim the chunks of one task after another from
one shared cursor, and a CTA barrier is left only where the block changes.  The cases are blocks with several
consecutive tasks: hot-only, pass-A-only and mixed fused tasks (k_pr_cb<CB_FUSED>, GB_PR_VBLOCKS=1), and the SELL
path's tasks (k_pr_cb<CB_MAIN>); in each, some block's run of tasks is cut by a CTA range boundary, so that a
steal lands in the middle of it, and two cases have no more tasks than CTAs (every range holds one task).  On the
CPU the layout model (tools/layout_model.py: fused_tasks, hot_chunks) shows that each case reaches what it names.
On the GPU the plan's task counts are the model's, the ranks match the f64 oracle, repeated runs give the same
bits, and GB_PR_TASK_CHUNKS = 32 and 128 (at a fixed chunk size) give the same bits; and the virtual-rank shards at
2 and 5 ranks, with and without virtual blocks, match the oracle and repeat their bits."""
import numpy as np
import pytest

import oracle
import pr_path_fixtures as fx

lm = fx.lm

PR_RTOL = 1e-6
ERR_ATOL = 2e-6
SWEEPS = 10
VB = {"GB_PR_VBLOCKS": 1}
VB_KNOBS = ("GB_PR_VBLOCKS", "GB_PR_VB_WINDOW")


def cold_only(n=20001, d=128):
    """every in- and out-degree is d; at GB_PR_TAU=0 no pair gets a segment, and at B = 4096 each source block
    holds more than 32 pass-A chunks: blocks of several pass-A-only tasks"""
    rng = np.random.default_rng(5)
    src = np.tile(np.arange(n, dtype=np.uint32), d)
    dst = np.concatenate([rng.permutation(n).astype(np.uint32) for _ in range(d)])
    return src, dst, n


def hubs(n=100001, d=24, n_hubs=20):
    """every vertex sends an edge to each of n_hubs hub rows (segments in every block) and d edges to random other
    rows (cold at the default tau); at B = 4096 and a V window of 2048 slots each source block holds more than 32
    hot and more than 32 pass-A chunks: blocks of several mixed tasks"""
    rng = np.random.default_rng(3)
    v = np.arange(n, dtype=np.uint32)
    src = np.concatenate([np.tile(v, d), np.tile(v, n_hubs)])
    dst = np.concatenate([rng.integers(n_hubs, n, n * d).astype(np.uint32),
                          np.repeat(np.arange(n_hubs, dtype=np.uint32), n)])
    return src, dst, n


# case -> (graph builder, knobs, V window of the model or None, kernel)
CASES = {
    "hot_only": (fx.rmat18, {**VB, "GB_PR_BLOCK": 1024}, None, "fused"),
    "pass_a_only": (cold_only, {**VB, "GB_PR_BLOCK": 4096, "GB_PR_TAU": 0}, None, "fused"),
    "mixed": (hubs, {**VB, "GB_PR_BLOCK": 4096, "GB_PR_VB_WINDOW": 2048}, 2048, "fused"),
    "sell": (fx.rmat18, {"GB_PR_BLOCK": 1024}, None, "main"),
}

_GRAPH: dict = {}
_MODEL: dict = {}


def graph(case):
    """(n, out CSR, in CSR) of a case's graph, Sorted layout, one graph cached at a time"""
    if case not in _GRAPH:
        src, dst, n = CASES[case][0]()
        out = oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED)
        inc = oracle.csr_build(src, dst, n, oracle.INCOMING, oracle.SORTED)
        _GRAPH.clear()
        _GRAPH[case] = (n, out, inc)
    return _GRAPH[case]


def model(case):
    """k_pr_cb's tasks of a case by the layout model, as (block, hot chunks, pass-A chunks) per task (cached)"""
    if case not in _MODEL:
        _, env, window, kernel = CASES[case]
        n, out, inc = graph(case)
        tau = 1e30 if env.get("GB_PR_TAU") == 0 else lm.CB_TAU_DEFAULT
        plan = lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)),
                            lm.clamp_block(env["GB_PR_BLOCK"]), tau)
        built = lm.build(plan, inc[0], inc[1], np.arange(n))
        if kernel == "fused":
            vb = lm.vblocks(plan, built, **({"window": window} if window else {}))
            assert vb is not None, case
            tasks = [(b, nh, na) for _, nh, _, na, b in lm.fused_tasks(plan, built["goff"], vb)["tasks"]]
        else:
            tasks = [(j, nc, 0) for _, nc, j in lm.hot_chunks(plan, built["goff"])[1]]
        _MODEL[case] = tasks
    return _MODEL[case]


def block_runs(tasks):
    """[first, end) of every block's run of consecutive tasks"""
    runs, i = [], 0
    while i < len(tasks):
        k = i
        while k < len(tasks) and tasks[k][0] == tasks[i][0]:
            k += 1
        runs.append((i, k))
        i = k
    return runs


def range_bounds(n_tasks, sms=lm.H100_SMS):
    """the first task of every CTA's range (grid = min(tasks, SMs), as the layout build sizes it)"""
    R = min(n_tasks, sms)
    return {n_tasks * r // R for r in range(1, R)}


def kinds(tasks, i, k):
    """tasks [i, k) that are hot-only, pass-A-only and mixed"""
    t = tasks[i:k]
    return (sum(nh > 0 and na == 0 for _, nh, na in t), sum(nh == 0 and na > 0 for _, nh, na in t),
            sum(nh > 0 and na > 0 for _, nh, na in t))


@pytest.mark.parametrize("case", list(CASES))
def test_cases_reach_consecutive_tasks(case):
    """some block holds at least 2 consecutive tasks of the named kind, and some run of a block's tasks is cut by
    a CTA range boundary"""
    tasks = model(case)
    runs = [(i, k) for i, k in block_runs(tasks) if k - i >= 2]
    want = {"hot_only": 0, "pass_a_only": 1, "mixed": 2, "sell": 0}[case]
    assert any(kinds(tasks, i, k)[want] >= 2 for i, k in runs), (case, runs[:8])
    bounds = range_bounds(len(tasks))
    assert any(any(i < b < k for b in bounds) for i, k in runs), (case, len(tasks))
    if case in ("pass_a_only", "mixed"):  # no more tasks than CTAs: every range holds one task
        assert len(tasks) <= lm.H100_SMS, (case, len(tasks))


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


def device_graph(gb, monkeypatch, case, **env):
    for k in VB_KNOBS:
        monkeypatch.delenv(k, raising=False)
    fx.set_knobs(monkeypatch, case, **CASES[case][1], **env)
    n, out, inc = graph(case)
    return gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])


def run(g):
    return g.page_rank(max_iterations=SWEEPS, tolerance=0.0, mode="jacobi")


def oracle_ranks(case):
    n, out, inc = graph(case)
    return oracle.page_rank_jacobi(inc[0], inc[1], out[0], SWEEPS, 0.0, 0.85, acc64=True)


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_flow_ranks_bits_and_task_sizes(gb, monkeypatch, case):
    g = device_graph(gb, monkeypatch, case)
    stats = g.page_rank_plan_info()
    assert stats["tasks"] == len(model(case)), (case, stats["tasks"], len(model(case)))
    assert (stats["vblock_parts"] > 0) == (CASES[case][3] == "fused"), case
    if CASES[case][3] == "fused":
        assert stats["launches_per_sweep"] == 3, case  # fused k_pr_cb, pass B, k_pr_finish
    pr = run(g)
    want, it, err = oracle_ranks(case)
    assert pr.ran_iterations == it
    rel = np.abs(pr.scores() - want) / want
    assert rel.max() <= PR_RTOL, (case, rel.max(), int(rel.argmax()))
    assert abs(pr.error - err) <= ERR_ATOL, (case, pr.error, err)
    for _ in range(2):
        again = run(g)
        assert again.scores().tobytes() == pr.scores().tobytes() and again.error == pr.error, case
    # the task size regroups the chunks into tasks; with the chunk size fixed the ranks keep their bits
    got = {}
    for t in (32, 128):
        r = run(device_graph(gb, monkeypatch, case, GB_PR_CHUNK=512, GB_PR_TASK_CHUNKS=t))
        rel = np.abs(r.scores() - want) / want
        assert rel.max() <= PR_RTOL, (case, t, rel.max())
        got[t] = (r.scores().tobytes(), r.error)
    assert got[32] == got[128], case


@pytest.mark.gpu
@pytest.mark.parametrize("world", (2, 5))
@pytest.mark.parametrize("case", ("hot_only", "sell"))
def test_flow_virtual_rank_shards(gb, monkeypatch, world, case):
    from virtual_ranks import VirtualRanks
    g = device_graph(gb, monkeypatch, case)
    vr = VirtualRanks(g, world)
    assert all((r.stats["vblock_parts"] > 0) == (CASES[case][3] == "fused") for r in vr.ranks), case
    vr.run(SWEEPS, 0.0)
    got = vr.scores_host()
    want, _, _ = oracle_ranks(case)
    rel = np.abs(got - want) / want
    assert rel.max() <= PR_RTOL, (case, world, rel.max())
    vr.run(SWEEPS, 0.0)
    assert vr.scores_host().tobytes() == got.tobytes(), (case, world)
