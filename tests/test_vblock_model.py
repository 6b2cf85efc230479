"""The contract of the PageRank layout's virtual blocks, checked on the layout model (tools/layout_model.py,
which restates layout_vblocks of graph_b200/csrc/pr_layout.cu): pass A writes every slot of V exactly once,
every cold edge appears exactly once in pass B and its id resolves to the slot of its source, the streamed
and resident classifications give the same virtual blocks, and the graphs the GPU tests use reach (or keep
off) the path."""
import numpy as np
import pytest

import vblock_fixtures as vf

lm = vf.lm


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("P", [1, 3])
def test_vblock_contract_on_random_graphs(seed, P):
    rng = np.random.default_rng(50 + seed)
    n, m = int(rng.integers(200, 600)), int(rng.integers(2000, 8000))
    in_off, in_tgt, out_deg = lm.random_graph(rng, n, m)
    parts = []
    for p in range(P):
        plan = lm.make_plan(in_off, in_tgt, out_deg, B=64, tau=1.5, P=P, p=p)
        streamed = lm.build(plan, in_off, in_tgt, np.arange(n))
        resident = lm.build(plan, in_off, in_tgt, plan["order"])
        a, b = lm.vblocks(plan, streamed), lm.vblocks(plan, resident)
        assert a is not None
        parts.append(a["parts"])
        lm.check_vblocks(plan, a, streamed)
        assert all(np.array_equal(a[k], b[k]) for k in a)
        assert lm.vb_counts(plan, in_off, in_tgt) == dict(vblock_parts=a["parts"], vblock_pairs=a["pairs"],
                                                          vblock_edges=a["edges"])
    assert max(parts) > 1


def test_vblock_partitions_and_fallback():
    lens = np.array([3, 0, 5, 2, 4, 0, 1])
    row0, mseg = lm.vb_partitions(lens, 8)
    assert row0.tolist() == [0, 3, 7] and mseg.tolist() == [2, 1]
    assert lm.vb_partitions(np.array([3, 9, 1]), 8) is None          # a row with more than B cold edges
    assert lm.vb_partitions(np.zeros(5, np.int64), 8) is None        # no cold edge


@pytest.mark.parametrize("name", vf.VB_FIXTURES)
def test_gpu_fixtures_reach_vblocks(name):
    c = vf.model_counts(name)
    assert c["vblock_parts"] > 0 and 0 < c["vblock_pairs"] <= c["vblock_edges"], (name, c)


def test_gpu_fixtures_no_hot_block_and_fallback():
    name, knobs = vf.NO_HOT
    assert vf.model_counts(name, tau=knobs["GB_PR_TAU"])["vblock_parts"] > 0
    name, knobs = vf.FALLBACK
    assert vf.model_counts(name, tau=knobs["GB_PR_TAU"])["vblock_parts"] == 0
