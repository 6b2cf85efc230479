"""Weighted graphs for the one-shot SSSP call (graph_b200.sssp_csr, gb_sssp_csr_u32), whose rows land chunk by
chunk from the start's chunk on: shapes where relax passes meet rows that have not landed yet.  Each comes with
the chunk budget (entries per chunk) that cuts it as its docstring says.  Shared by the CPU replay
(test_sssp_csr_cpu.py) and the GPU tests (test_gpu_sssp_csr.py); the queue fixtures of sssp_fixtures.py run
there too."""
from __future__ import annotations

import numpy as np

from sssp_fixtures import Fixture, _fx


def backward_chain(n=64):
    """edges i -> i - 1 (weights 1 + i / n), start n - 1: at one entry per chunk every row is a chunk, the start's
    is sent first and the next row the chain needs is the one sent last, so every pass but the first parks"""
    i = np.arange(1, n)
    return _fx(i, i - 1, 1.0 + i / n, n, n - 1, 1.0)


BACKWARD_CHAIN_ENTRIES = 1


def late_improver(k=8, fill=24):
    """the start 0 reaches x = 1 directly at weight 5 and through p = n - 1, the last row, at 0.1 + 0.1.  x's
    descendants d_1 .. d_k (ids 2 .. k + 1, weight 0.1 each) and `fill` rows of self-loops lie between them, one
    row per chunk.  p is parked in the first bucket; x and its chain are settled in bucket [5, 6) while p's row
    is still on its way; p's late relax then improves x to 0.2, below that drained bucket's lower bound, and the
    chain must be relaxed again.  A pass that still drops entries below `lower` keeps x's chain at 5.x."""
    n = k + 2 + fill + 1
    p = n - 1
    src = [0, 0, p] + list(range(1, k + 1)) + list(range(k + 2, k + 2 + fill))
    dst = [1, p, 1] + list(range(2, k + 2)) + list(range(k + 2, k + 2 + fill))
    w = [5.0, 0.1, 0.1] + [0.1] * k + [1.0] * fill
    return _fx(src, dst, w, n, 0, 1.0)


LATE_IMPROVER_ENTRIES = 1


def hub_row(leaves=5000, n=1001, hub=500):
    """the start 0 -> hub (weight 0.5); the hub's row of `leaves` edges is 20 chunk budgets long and stands alone;
    3000 random edges around it"""
    rng = np.random.default_rng(9)
    others = np.array([x for x in range(n) if x != hub])
    src = np.concatenate([[0], np.full(leaves, hub), rng.integers(0, n, 3000)])
    dst = np.concatenate([[hub], rng.choice(others, leaves), rng.integers(0, n, 3000)])
    w = np.concatenate([[0.5], rng.random(leaves + 3000, dtype=np.float32) * np.float32(2.0)])
    return _fx(src, dst, w, n, 0, 0.5)


HUB_ROW_ENTRIES = 250

FIXTURES = {"backward_chain": (backward_chain, BACKWARD_CHAIN_ENTRIES),
            "late_improver": (late_improver, LATE_IMPROVER_ENTRIES),
            "hub_row": (hub_row, HUB_ROW_ENTRIES)}

__all__ = ["Fixture", "FIXTURES", "backward_chain", "late_improver", "hub_row"]
