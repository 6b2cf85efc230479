"""Sector-aligned runs of the PageRank value buffer V: every run (the pairs of one source block inside one
partition) starts on a 32-byte sector, and pass A zeroes its pad slots up to the next sector in the step that
stores its last value, so that no sector of V is left half-written.  Pass B takes the padded virtual blocks in a
window larger than B; when a padded partition would not fit in it, the whole graph keeps the packed slots.

Pass B's window is larger than the shared memory of the other k_pr_cb launches, so a plan built later must not
shrink what an earlier, cached plan launches with.

On the CPU the layout model (tools/layout_model.py) checks the contract (runs on sectors, pads zeroed, pass B ids
below the window and never on a pad, position + delta = slot) on the fixtures, on their virtual-rank shards and
on random graphs, that the fixtures reach every place a run can end, and that a small GB_PR_VB_WINDOW forces the
packed fallback.  On the GPU every case checks the plan's counts against the model, the ranks against the f64
oracle, that repeated runs give the same bits, and, from a value buffer poisoned before one sweep, that pass A
wrote every pair's slot with its source's value, zeroed exactly the pad slots and nothing else.  One case runs
a sector plan again after a packed plan was built on the same device."""
import numpy as np
import pytest

import oracle
import pr_path_fixtures as fx

lm = fx.lm

PR_RTOL = 1e-6
ERR_ATOL = 2e-6
SWEEPS = 10
SMALL_WINDOW = 1024  # GB_PR_VB_WINDOW: below the padded partitions of the fixtures (B = 1024): packed fallback

# (fixture, GB_PR_TAU or None for the default), as in test_gpu_pr_pass_a.py
CASES = [("rmat18", None), ("equal_degrees", 0), ("tail_r1", None), ("few_active", None)]

_MODEL: dict = {}


def model(name, tau=None, P=1, p=0, window=lm.VB_WINDOW):
    """the layout model's virtual blocks of a fixture, checked, with pass A's fills by case (cached)"""
    key = (name, tau, P, p, window)
    if key not in _MODEL:
        _, _, n, out, inc = fx.graph(name)
        B = lm.clamp_block(fx.FIXTURES[name][1] or lm.CB_BLOCK_DEFAULT)
        plan = lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)), B,
                            1e30 if tau == 0 else lm.CB_TAU_DEFAULT, P=P, p=p)
        built = lm.build(plan, inc[0], inc[1], np.arange(n))
        vb = lm.vblocks(plan, built, window)
        assert vb is not None, key
        lm.check_vblocks(plan, vb, built)
        fills: dict = {}
        V, _, wide = lm.vb_pass_a(plan, vb, fills)
        outdeg = np.diff(out[0].astype(np.int64))[plan["order"]]                 # internal order
        with np.errstate(divide="ignore"):                                        # +inf for dangling vertices
            x0 = np.float32(1.0) / np.float32(n) / outdeg.astype(np.float32)     # k_pr_init: init / outdeg
        _MODEL[key] = dict(fills=fills, wide=len(wide), slots=vb["slots"], sectors=int(vb["sectors"]),
                           counts=lm.vb_counts(plan, inc[0], inc[1]), V=V, x0=x0)
    return _MODEL[key]


@pytest.mark.parametrize("name,tau", CASES)
def test_model_holds_and_takes_sectors(name, tau):
    m = model(name, tau)
    assert m["sectors"] == 1 and m["slots"] > 0, (name, m)


def test_fixtures_reach_every_run_end():
    f = model("rmat18")["fills"]
    assert f.get("step_end", 0) > 0 and f.get("chunk_end", 0) > 0 and f.get("share_end", 0) > 0, f
    assert f.get("inside", 0) > 0 and f.get("wide", 0) > 0, f


@pytest.mark.parametrize("world", [2, 5])
def test_model_holds_on_virtual_rank_shards(world):
    for p in range(world):
        assert model("rmat18", None, world, p)["sectors"] == 1, p
        assert model("rmat18", None, world, p, SMALL_WINDOW)["sectors"] == 0, p


def test_small_window_falls_back_to_packed_slots():
    packed = model("rmat18", window=SMALL_WINDOW)
    assert packed["sectors"] == 0 and not packed["fills"]
    assert packed["slots"] < model("rmat18")["slots"]


@pytest.mark.parametrize("seed", range(3))
@pytest.mark.parametrize("P", [1, 2, 5])
def test_model_holds_on_random_graphs(seed, P):
    rng = np.random.default_rng(70 + seed)
    n, m = int(rng.integers(200, 600)), int(rng.integers(2000, 8000))
    in_off, in_tgt, out_deg = lm.random_graph(rng, n, m)
    for p in range(P):
        plan = lm.make_plan(in_off, in_tgt, out_deg, B=64, tau=1.5, P=P, p=p)
        built = lm.build(plan, in_off, in_tgt, np.arange(n))
        for window in (lm.VB_WINDOW, 64):
            vb = lm.vblocks(plan, built, window)
            if vb is None:
                continue
            lm.check_vblocks(plan, vb, built)
            assert vb["sectors"] or window < lm.VB_WINDOW, p


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


def knobs(monkeypatch, name, tau, window=None):
    env = dict(GB_PR_VBLOCKS=1)
    if tau is not None:
        env["GB_PR_TAU"] = tau
    fx.set_knobs(monkeypatch, name, **env)
    if window is None:
        monkeypatch.delenv("GB_PR_VB_WINDOW", raising=False)
    else:
        monkeypatch.setenv("GB_PR_VB_WINDOW", str(window))


def oracle_ranks(name):
    _, _, n, out, inc = fx.graph(name)
    return oracle.page_rank_jacobi(inc[0], inc[1], out[0], SWEEPS, 0.0, 0.85, acc64=True)


def assert_stats(stats, m):
    assert {k: stats[k] for k in m["counts"]} == m["counts"]
    assert stats["vblock_wide_steps"] == m["wide"]
    assert stats["vblock_slots"] == m["slots"] and stats["vblock_sectors"] == m["sectors"]


@pytest.mark.gpu
@pytest.mark.parametrize("window", [None, SMALL_WINDOW])
@pytest.mark.parametrize("name,tau", CASES)
def test_vsectors_ranks_bits_and_plan(gb, monkeypatch, name, tau, window):
    knobs(monkeypatch, name, tau, window)
    _, _, n, out, inc = fx.graph(name)
    g = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    m = model(name, tau, window=window or lm.VB_WINDOW)
    assert_stats(g.page_rank_plan_info(), m)
    pr = g.page_rank(max_iterations=SWEEPS, tolerance=0.0, mode="jacobi")
    want, it, err = oracle_ranks(name)
    assert pr.ran_iterations == it
    rel = np.abs(pr.scores() - want) / want
    assert rel.max() <= PR_RTOL, (name, rel.max(), int(rel.argmax()))
    assert abs(pr.error - err) <= ERR_ATOL, (name, pr.error, err)
    again = g.page_rank(max_iterations=SWEEPS, tolerance=0.0, mode="jacobi")
    assert again.scores().tobytes() == pr.scores().tobytes() and again.error == pr.error, name


@pytest.mark.gpu
@pytest.mark.parametrize("window", [None, SMALL_WINDOW])
@pytest.mark.parametrize("world", [2, 5])
def test_vsectors_virtual_rank_shards(gb, monkeypatch, world, window):
    from virtual_ranks import VirtualRanks
    name = "rmat18"
    knobs(monkeypatch, name, None, window)
    _, _, n, out, inc = fx.graph(name)
    g = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    vr = VirtualRanks(g, world)
    for p, r in enumerate(vr.ranks):
        assert_stats(r.stats, model(name, None, world, p, window or lm.VB_WINDOW))
    vr.run(SWEEPS, 0.0)
    got = vr.scores_host()
    want, _, _ = oracle_ranks(name)
    rel = np.abs(got - want) / want
    assert rel.max() <= PR_RTOL, rel.max()
    vr.run(SWEEPS, 0.0)
    assert vr.scores_host().tobytes() == got.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("window", [None, SMALL_WINDOW])
@pytest.mark.parametrize("name,tau", [("rmat18", None), ("equal_degrees", 0)])
def test_vsectors_pass_a_writes_slots_and_zeroes_pads(gb, monkeypatch, name, tau, window):
    """V poisoned with NaN bits, then one sweep: every pair's slot holds its source's x0, every pad slot of a run
    is +0.0 (sector slots only), and every other slot (between the virtual blocks) is still poisoned"""
    import ctypes as C
    from graph_b200._capi import check, lib
    knobs(monkeypatch, name, tau, window)
    _, _, n, out, inc = fx.graph(name)
    g = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    m = model(name, tau, window=window or lm.VB_WINDOW)
    assert_stats(g.page_rank_plan_info(), m)
    V = np.empty(m["slots"], np.float32)
    check(lib.gb_page_rank_plan_values(g._g, 1, None, m["slots"]))
    g.page_rank(max_iterations=1, tolerance=0.0, mode="jacobi")
    check(lib.gb_page_rank_plan_values(g._g, 0, V.ctypes.data_as(C.c_void_p), m["slots"]))
    bits = V.view(np.uint32)
    pair, pad = m["V"] >= 0, m["V"] == -2
    assert (V[pair] == m["x0"][m["V"][pair]]).all(), "a pair's slot holds its source's value"
    assert (bits[pad] == 0).all(), "pad slots are +0.0"
    assert (bits[~pair & ~pad] == 0xFFFFFFFF).all(), "pass A writes nothing outside the runs and their pads"
    assert pad.any() == (window is None), name


@pytest.mark.gpu
def test_vsectors_plan_runs_after_a_packed_plan_on_the_device(gb, monkeypatch):
    """the shared-memory limit of k_pr_cb is the kernel's, not the plan's: a sector plan (pass B's window of
    about 58 k slots) still runs after a packed plan (window B) and a SELL plan were built on the same device"""
    name = "rmat18"
    _, _, n, out, inc = fx.graph(name)
    knobs(monkeypatch, name, None)
    g = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    assert g.page_rank_plan_info()["vblock_sectors"] == 1
    first = g.page_rank(max_iterations=SWEEPS, tolerance=0.0, mode="jacobi")
    knobs(monkeypatch, name, None, SMALL_WINDOW)
    packed = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    assert packed.page_rank_plan_info()["vblock_sectors"] == 0
    packed.page_rank(max_iterations=SWEEPS, tolerance=0.0, mode="jacobi")
    fx.set_knobs(monkeypatch, name, GB_PR_VBLOCKS=2)
    sell = gb.DiGraph.from_csr(out[0], out[1], inc[0], inc[1])
    assert sell.page_rank_plan_info()["vblock_parts"] == 0
    sell.page_rank(max_iterations=SWEEPS, tolerance=0.0, mode="jacobi")
    again = g.page_rank(max_iterations=SWEEPS, tolerance=0.0, mode="jacobi")
    assert again.scores().tobytes() == first.scores().tobytes() and again.error == first.error
