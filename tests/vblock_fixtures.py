"""Which graphs of tests/pr_path_fixtures.py reach the virtual blocks of the PageRank layout under
GB_PR_VBLOCKS=1, and which keep SELL.  Shared by the CPU check against the layout model (test_vblock_model.py)
and the GPU tests (test_gpu_pr_vblocks.py), so that a graph that drifts off the path fails on the CPU first."""
from __future__ import annotations

import numpy as np

import pr_path_fixtures as fx

lm = fx.lm

# graphs with cold edges, none of whose rows has more than B of them
VB_FIXTURES = [f"tail_r{r}" for r in fx.TAIL_R] + ["equal_degrees", "repeated_source", "few_active", "rmat18"]
# (graph, knobs): GB_PR_TAU=0 switches the column blocks off, so every edge is cold.  equal_degrees then takes
# the virtual blocks with no hot block at all; star_in's hub row has 2e5 cold edges > B, so it keeps SELL.
NO_HOT = ("equal_degrees", {"GB_PR_TAU": 0})
FALLBACK = ("star_in", {"GB_PR_TAU": 0})


def model_counts(name, tau=lm.CB_TAU_DEFAULT, P=1, p=0):
    """the model's vblock_parts / vblock_pairs / vblock_edges of a fixture (tau 0: no column blocks)"""
    _, _, n, out, inc = fx.graph(name)
    B = lm.clamp_block(fx.FIXTURES[name][1] or lm.CB_BLOCK_DEFAULT)
    plan = lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)), B,
                        tau if tau > 0 else 1e30, P=P, p=p)
    return lm.vb_counts(plan, inc[0], inc[1])
