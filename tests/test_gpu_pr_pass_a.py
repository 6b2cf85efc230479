"""Pass A of the PageRank virtual blocks (k_pr_cb<CB_BIN>): a warp walks its chunk in 256-position steps, lane L
reads the ids of positions L, L + 32, .., L + 224 with one 128-bit load, finds each position's run among the
step's runs by shuffle, and stores the value to V at position + the run's delta; a step with more than 32 runs
takes the slower run-window loop.  The fixtures (GB_PR_VBLOCKS=1, the fixture block sizes of
tests/pr_path_fixtures.py) reach, by the layout model (tools/layout_model.py), steps with more than 32 runs, block
shares shorter than one step, runs that cross a step and a chunk boundary, pad positions, and the virtual-rank
shards.  On the GPU every case checks the ranks against the f64 oracle, that repeated runs give the same bits,
and that the plan counts the model's run-window steps."""
import numpy as np
import pytest

import oracle
import pr_path_fixtures as fx

lm = fx.lm

PR_RTOL = 1e-6
ERR_ATOL = 2e-6
SWEEPS = 10

# (fixture, GB_PR_TAU or None for the default): rmat18 reaches every case on one GPU and on its shards;
# equal_degrees without column blocks has long runs, many of them across chunk boundaries, and no wide step;
# tail_r1's and few_active's block shares are shorter than one step
CASES = [("rmat18", None), ("equal_degrees", 0), ("tail_r1", None), ("few_active", None)]

_MODEL: dict = {}


def pass_a_model(name, tau=None, P=1, p=0):
    """the layout model's pass A cases of a fixture and the run-window steps of its walk (cached)"""
    key = (name, tau, P, p)
    if key not in _MODEL:
        _, _, n, out, inc = fx.graph(name)
        B = lm.clamp_block(fx.FIXTURES[name][1] or lm.CB_BLOCK_DEFAULT)
        plan = lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)), B,
                            1e30 if tau == 0 else lm.CB_TAU_DEFAULT, P=P, p=p)
        built = lm.build(plan, inc[0], inc[1], np.arange(n))
        vb = lm.vblocks(plan, built)
        assert vb is not None, key
        lm.check_vblocks(plan, vb, built)
        _, _, wide = lm.vb_pass_a(plan, vb)
        _MODEL[key] = dict(lm.vb_pass_a_cases(vb), wide=len(wide))
    return _MODEL[key]


def test_fixtures_reach_the_pass_a_cases():
    c = pass_a_model("rmat18")
    assert c["wide"] > 0 and c["short_shares"] > 0 and c["step_runs"] > 0 and c["chunk_runs"] > 0 and c["pads"] > 0, c
    c = pass_a_model("equal_degrees", 0)
    assert c["chunk_runs"] > 100 and c["wide"] == 0, c
    for name in ("tail_r1", "few_active"):
        assert pass_a_model(name)["short_shares"] > 0, name
    for world in (2, 5):
        assert all(pass_a_model("rmat18", None, world, p)["wide"] > 0 for p in range(world)), world


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


def knobs(monkeypatch, name, tau):
    env = dict(GB_PR_VBLOCKS=1)
    if tau is not None:
        env["GB_PR_TAU"] = tau
    fx.set_knobs(monkeypatch, name, **env)


def oracle_ranks(name, sweeps=SWEEPS, tol=0.0):
    _, _, n, out, inc = fx.graph(name)
    return oracle.page_rank_jacobi(inc[0], inc[1], out[0], sweeps, tol, 0.85, acc64=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name,tau", CASES)
def test_pass_a_ranks_bits_and_run_windows(gb, monkeypatch, name, tau):
    knobs(monkeypatch, name, tau)
    _, _, n, out, inc = fx.graph(name)
    g = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    info = g.page_rank_plan_info()
    assert info["vblock_parts"] > 0, (name, info)
    assert info["vblock_wide_steps"] == pass_a_model(name, tau)["wide"], (name, info)
    if name == "rmat18":
        assert info["vblock_wide_steps"] > 0  # every sweep takes the run-window loop on these steps
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
@pytest.mark.parametrize("world", [2, 5])
def test_pass_a_virtual_rank_shards(gb, monkeypatch, world):
    """every rank's pass A walks the steps of its own pairs: the ranks' wide steps are the model's, the scores
    match the oracle, and a second run gives the same bits"""
    from virtual_ranks import VirtualRanks
    name = "rmat18"
    knobs(monkeypatch, name, None)
    _, _, n, out, inc = fx.graph(name)
    g = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    vr = VirtualRanks(g, world)
    for p, r in enumerate(vr.ranks):
        assert r.stats["vblock_parts"] > 0
        assert r.stats["vblock_wide_steps"] == pass_a_model(name, None, world, p)["wide"], p
    vr.run(SWEEPS, 0.0)
    got = vr.scores_host()
    want, _, _ = oracle_ranks(name)
    rel = np.abs(got - want) / want
    assert rel.max() <= PR_RTOL, rel.max()
    vr.run(SWEEPS, 0.0)
    assert vr.scores_host().tobytes() == got.tobytes()
