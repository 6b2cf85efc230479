"""Pass A of the PageRank virtual blocks inside k_pr_cb's tasks (k_pr_cb<CB_FUSED>): one task list over the union
of the hot blocks and pass A's source blocks, a task holding a source block's hot chunks and its pass-A chunks,
so that the block is loaded once for both walkers; the hot blocks' cut segments are added by pass B's first
warps.  On the CPU the layout model (tools/layout_model.py: hot_chunks, fused_tasks) checks that every hot chunk
and every pass-A chunk lies in exactly one task, that no task mixes blocks, and that the fixtures (GB_PR_VBLOCKS=1)
reach tasks with both kinds of chunks, tasks with pass-A chunks only, and cut segments.  On the GPU, on one device
and on virtual-rank shards, the plan's task and cut-segment counts are the model's, the ranks match the f64
oracle, and repeated runs give the same bits."""
import numpy as np
import pytest

import oracle
import pr_path_fixtures as fx

lm = fx.lm

PR_RTOL = 1e-6
ERR_ATOL = 2e-6
SWEEPS = 10

# (fixture, GB_PR_TAU or None for the default).  rmat18: hot blocks with both kinds of chunks and blocks with
# pass-A chunks only; repeated_source: a segment of 50000 ids cut by chunk boundaries next to pass-A chunks;
# equal_degrees without column blocks: pass-A chunks only, in every task
CASES = [("rmat18", None), ("repeated_source", None), ("equal_degrees", 0)]
WORLDS = (2, 5)

_MODEL: dict = {}


def fused_model(name, tau=None, P=1, p=0):
    """the layout model's fused tasks of a fixture (cached)"""
    key = (name, tau, P, p)
    if key not in _MODEL:
        _, _, n, out, inc = fx.graph(name)
        B = lm.clamp_block(fx.FIXTURES[name][1] or lm.CB_BLOCK_DEFAULT)
        plan = lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)), B,
                            1e30 if tau == 0 else lm.CB_TAU_DEFAULT, P=P, p=p)
        built = lm.build(plan, inc[0], inc[1], np.arange(n))
        vb = lm.vblocks(plan, built)
        assert vb is not None, key
        _MODEL[key] = dict(lm.fused_tasks(plan, built["goff"], vb), plan=plan, vb=vb)
    return _MODEL[key]


def model_cases():
    for name, tau in CASES:
        yield name, tau, 1, 0
    for world in WORLDS:
        for p in range(world):
            yield "rmat18", None, world, p


def test_every_chunk_in_one_task_of_its_block():
    for name, tau, P, p in model_cases():
        m = fused_model(name, tau, P, p)
        blk = m["plan"]["blk"]
        hot_seen = np.zeros(len(m["hot_chunks"]), np.int64)
        bin_seen = np.zeros(len(m["vb"]["bin_chunks"]), np.int64)
        for h0, nh, a0, na, b in m["tasks"]:
            assert nh + na > 0 and nh < 256 and na <= lm.CB_TASK_CHUNKS, (name, P, p)
            hot_seen[h0:h0 + nh] += 1
            bin_seen[a0:a0 + na] += 1
            assert all(blk[m["hot_chunks"][c][2]] == b for c in range(h0, h0 + nh)), "a hot chunk of another block"
            assert (m["bin_blk"][a0:a0 + na] == b).all(), "a pass-A chunk of another block"
        assert (hot_seen == 1).all() and (bin_seen == 1).all(), (name, P, p)
        # a block's tasks are consecutive
        order = [t[4] for t in m["tasks"]]
        firsts = [b for i, b in enumerate(order) if i == 0 or order[i - 1] != b]
        assert len(firsts) == len(set(order)), (name, P, p)


def test_fixtures_reach_the_fused_cases():
    both = lambda m: sum(t[1] > 0 and t[3] > 0 for t in m["tasks"])
    bin_only = lambda m: sum(t[1] == 0 and t[3] > 0 for t in m["tasks"])
    m = fused_model("rmat18")
    assert both(m) > 0 and bin_only(m) > 0, m["tasks"][:8]
    m = fused_model("repeated_source")
    assert m["n_fix"] > 0 and both(m) > 0, m["n_fix"]
    m = fused_model("equal_degrees", 0)
    assert not m["hot_chunks"] and bin_only(m) == len(m["tasks"]) > 0
    for world in WORLDS:
        assert all(both(fused_model("rmat18", None, world, p)) > 0 for p in range(world)), world


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


def knobs(monkeypatch, name, tau):
    env = dict(GB_PR_VBLOCKS=1)
    if tau is not None:
        env["GB_PR_TAU"] = tau
    fx.set_knobs(monkeypatch, name, **env)


def oracle_ranks(name):
    _, _, n, out, inc = fx.graph(name)
    return oracle.page_rank_jacobi(inc[0], inc[1], out[0], SWEEPS, 0.0, 0.85, acc64=True)


def assert_counts(stats, m):
    assert stats["vblock_parts"] > 0
    assert stats["tasks"] == len(m["tasks"]) and stats["cut_segments"] == m["n_fix"], \
        (stats["tasks"], len(m["tasks"]), stats["cut_segments"], m["n_fix"])
    assert stats["launches_per_sweep"] == 3  # fused k_pr_cb, pass B, k_pr_finish


@pytest.mark.gpu
@pytest.mark.parametrize("name,tau", CASES)
def test_fused_ranks_bits_and_counts(gb, monkeypatch, name, tau):
    knobs(monkeypatch, name, tau)
    _, _, n, out, inc = fx.graph(name)
    g = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    m = fused_model(name, tau)
    assert_counts(g.page_rank_plan_info(), m)
    assert g.page_rank_plan_shape()["n_fix"] == m["n_fix"]
    pr = g.page_rank(max_iterations=SWEEPS, tolerance=0.0, mode="jacobi")
    want, it, err = oracle_ranks(name)
    assert pr.ran_iterations == it
    rel = np.abs(pr.scores() - want) / want
    assert rel.max() <= PR_RTOL, (name, rel.max(), int(rel.argmax()))
    assert abs(pr.error - err) <= ERR_ATOL, (name, pr.error, err)
    for _ in range(2):
        again = g.page_rank(max_iterations=SWEEPS, tolerance=0.0, mode="jacobi")
        assert again.scores().tobytes() == pr.scores().tobytes() and again.error == pr.error, name


@pytest.mark.gpu
@pytest.mark.parametrize("world", WORLDS)
def test_fused_virtual_rank_shards(gb, monkeypatch, world):
    from virtual_ranks import VirtualRanks
    name = "rmat18"
    knobs(monkeypatch, name, None)
    _, _, n, out, inc = fx.graph(name)
    g = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    vr = VirtualRanks(g, world)
    for p, r in enumerate(vr.ranks):
        assert_counts(r.stats, fused_model(name, None, world, p))
    vr.run(SWEEPS, 0.0)
    got = vr.scores_host()
    want, _, _ = oracle_ranks(name)
    rel = np.abs(got - want) / want
    assert rel.max() <= PR_RTOL, rel.max()
    vr.run(SWEEPS, 0.0)
    assert vr.scores_host().tobytes() == got.tobytes()
