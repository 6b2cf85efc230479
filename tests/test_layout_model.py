"""CPU check of the PageRank layout build's contract (tools/layout_model.py): the numpy restatement of
cb_classify_row / k_cb_count[_rows] / k_cb_groups / k_cb_fill in graph_b200/csrc/pr_layout.cu — one record per
edge, positions in CSR order — must reproduce the layout stated directly, for every rank of a cyclic deal,
and must not depend on the order in which rows are classified (streamed upload vs resident graph)."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import layout_model as lm  # noqa: E402


@pytest.mark.parametrize("seed,world", [(1, 1), (2, 2), (3, 3)])
def test_records_reproduce_the_direct_layout(seed, world):
    rng = np.random.default_rng(seed)
    n, m = 300, 4000
    in_off, in_tgt, out_deg = lm.random_graph(rng, n, m)
    segments = 0
    for p in range(world):
        plan = lm.make_plan(in_off, in_tgt, out_deg, B=64, tau=1.5, P=world, p=p)
        streamed = lm.build(plan, in_off, in_tgt, rng.permutation(n))     # any classification order
        resident = lm.build(plan, in_off, in_tgt, plan["order"])
        lm.check(plan, streamed, in_off, in_tgt)
        assert (streamed["ids"] == resident["ids"]).all() and (streamed["goff"] == resident["goff"]).all()
        assert all((streamed["sell"][l] == resident["sell"][l]).all() for l in range(plan["n_loc"]))
        segments += int((streamed["cnt"] > 0).sum())
    assert segments > 0


def test_deal_count_matches_the_row_owners_on_tiny_graphs():
    """deal_count (what every shard's local_rows must be) against the owner of each row as the multi-GPU
    driver assigns it, for every world and every active-row count up to a bit more than one slice per rank:
    ranks that own nothing, a partial last slice, a partial slice on a later rank"""
    from graph_b200.multigpu import owner_of_rows
    for P in range(1, 9):
        for n_active in range(0, 32 * P + 41):
            owner = owner_of_rows(range(n_active), P)
            for p in range(P):
                assert lm.deal_count(n_active, P, p) == int((owner == p).sum()), (P, n_active, p)


def test_cyclic_deal_is_a_partition():
    for P in (1, 2, 3, 8):
        for R in (0, 1, 31, 32, 33, 1000, 1024):
            counts = [lm.deal_count(R, P, p) for p in range(P)]
            assert sum(counts) == R
            seen = sorted(lm.deal_global(l, P, p) for p in range(P) for l in range(counts[p]))
            assert seen == list(range(R))
            for p in range(P):
                for l in range(counts[p]):
                    assert lm.deal_local(lm.deal_global(l, P, p), P, p) == l
