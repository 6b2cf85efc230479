"""CPU check that every fixture graph of test_gpu_pr_paths.py reaches the sweep path it was built for,
by the layout model (tools/layout_model.py: the layout_order, layout_hot_blocks and plan_sweep_shape
stages of build_pr_plan) on an H100's 132 SMs.
If a retuned default moves a graph off its path, this fails here, without a GPU."""
import pytest

import pr_path_fixtures as fx


@pytest.mark.parametrize("name", list(fx.FIXTURES))
def test_fixture_reaches_its_path(name):
    plan, shape, counts = fx.model(name)
    print(f"{name}: {fx.check_path(name, plan, shape)}")
    assert counts["segments"] == plan["S"] and counts["block_edges"] > 0


def test_fixtures_reach_every_walker_instantiation():
    """k_pr_cb walks a chunk with G = 2 or 4 groups per lane (cb_step_groups), with or without the side-buffer
    logic of a segment cut at a chunk end: the fixtures reach all four instantiations"""
    kinds = set()
    for name in fx.FIXTURES:
        kinds |= {(fx.bm.cb_model.step_groups(g0, g1), cut) for g0, g1, cut in fx.chunks(name) if g0 < g1}
    assert kinds == {(2, False), (2, True), (4, False), (4, True)}


def test_finish_knobs_on_rmat18():
    plan, auto, _ = fx.model("rmat18")
    assert (auto["hot_blocks"], auto["n_cb"], auto["n_fin"], auto["n_fin_warp"]) == (148, 69628, 12640, 192)
    u4 = fx.lm.launch_shape(plan, fin_u=4)
    assert u4["fin_u"] == 4 and u4["fin_hub_ctas"] == 0 and u4["grid_fin"] < auto["grid_fin"]
    split = fx.lm.launch_shape(plan, fin_split=1)          # KB = 148 <= 256: automatic would not split
    assert split["fin_hub_ctas"] == 6 and split["grid_fin"] == auto["grid_fin"]
    both = fx.lm.launch_shape(plan, fin_u=4, fin_split=1)
    assert both["fin_u"] == 4 and both["fin_hub_ctas"] == 6
    assert fx.lm.launch_shape(plan, fin_split=2)["fin_hub_ctas"] == 0


def test_finish_knobs_on_the_capped_grid():
    plan, auto, _ = fx.model("capped_finish")
    u2 = fx.lm.launch_shape(plan, fin_u=2)
    assert u2["grid_capped"] and u2["grid_fin"] == 8 * fx.lm.H100_SMS and u2["fin_hub_ctas"] == 0
    split = fx.lm.launch_shape(plan, fin_u=2, fin_split=1)   # forced: the grid is capped
    assert split["fin_hub_ctas"] == 1
    # the tail CTAs of the split grid need more than one pass: a wrong stride would skip row groups
    tail_warps = (split["n_fin"] - split["n_fin_warp"] + 63) // 64
    assert tail_warps > (split["grid_fin"] - 1) * fx.lm.PR_FIN_WARPS


def test_split_keeps_its_structural_conditions():
    plan, shape, _ = fx.model("few_active")                 # hub group only, nothing left for the tail
    assert fx.lm.launch_shape(plan, fin_split=1)["fin_hub_ctas"] == 0
    plan, shape, _ = fx.model("equal_degrees")              # no hub group at all
    assert shape["n_fin_warp"] == 0 and fx.lm.launch_shape(plan, fin_split=1)["fin_hub_ctas"] == 0


@pytest.mark.parametrize("world", [2, 3])
def test_split_on_virtual_rank_shards(world):
    for p in range(world):
        plan, _, _ = fx.model("rmat18", P=world, p=p)
        sh = fx.lm.launch_shape(plan, fin_split=1)
        assert sh["fin_hub_ctas"] > 0, (world, p)


def test_block_clamp_and_mega_threshold():
    assert [fx.lm.clamp_block(b) for b in (0, 1000, 1024, 3000, 49152, 1 << 20)] == [1024, 1024, 1024, 2048,
                                                                                     49152, 56 * 1024]
    plan, shape, _ = fx.model("star_in")
    assert shape["n_mega"] == 1
    _, _, n, out, inc = fx.graph("star_in")
    import numpy as np
    plan = fx.lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)), 49152, 1.5,
                           mega=n)                         # GB_PR_MEGA above the hub's in-degree
    assert plan["n_mega"] == 0
