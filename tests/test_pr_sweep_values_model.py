"""What the single-sweep check of test_gpu_pr_sweep_values.py can see, on the CPU.  Two wrong gathers are stated
on every path fixture's in-CSR (tests/pr_path_fixtures.py, which holds the graphs of tests/vblock_fixtures.py too):
every entry moved to its source's neighbour in the internal order with the same degree key (what an off-by-one
source index reads when the keys tie), and one source block's ids shifted by one (a wrong block base).  From
each of the test's integer vectors the expected bytes of at least one row change; from the start vector
init / outdeg the first sweep cannot tell the tie neighbours apart at all."""
import numpy as np
import pytest

import pr_path_fixtures as fx
import pr_sweep_values as sv

lm = fx.lm
SEEDS = (1, 2, 3)   # one vector per sweep_no of the GPU test


def setup(name):
    _, _, n, out, inc = fx.graph(name)
    B = lm.clamp_block(fx.FIXTURES[name][1] or lm.CB_BLOCK_DEFAULT)
    plan = lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)), B, lm.CB_TAU_DEFAULT)
    ic = sv.internal(plan, out, inc)
    return ic, B, sv.owned(n, ic["n_active"])


def changed(ic, mine, x, src):
    """rows whose score or x_next bytes differ (x_next alone is +inf on every row without out-edges)"""
    want, got = sv.expected(ic, x), sv.expected(ic, x, src)
    diff = [w[mine].view(np.uint32) != g[mine].view(np.uint32) for w, g in zip(want, got)]
    return int((diff[0] | diff[1]).sum())


@pytest.mark.parametrize("name", list(fx.FIXTURES))
def test_wrong_gathers_change_the_expected_bytes(name):
    ic, B, mine = setup(name)
    used = sv.gathered(ic, mine)
    assert not np.isnan(sv.expected(ic, sv.vector(ic, used, 1))[0][mine]).any(), "no row reads a NaN"
    ties = sv.tie_neighbours(ic)
    assert (ties != ic["src"]).mean() > 0.3, "the fixture has tied sources"
    shifted = sv.shift_block(ic, B, sv.busiest_block(ic, B))
    for seed in SEEDS:
        x = sv.vector(ic, used, seed)
        assert changed(ic, mine, x, ties) > 0, (name, seed, "tie neighbours")
        assert changed(ic, mine, x, shifted) > 0, (name, seed, "shifted block")


@pytest.mark.parametrize("name", list(fx.FIXTURES))
def test_start_vector_hides_tie_neighbours(name):
    """from x0 = init / outdeg a tie neighbour holds the same value: the first sweep's sums are the same bits"""
    ic, _, mine = setup(name)
    init, _ = sv.start(ic["n"])
    with np.errstate(divide="ignore"):
        x0 = init / ic["outdeg_int"].astype(np.float32)
    rows = np.repeat(ic["new_id"], ic["indeg"])
    sums = lambda src: np.bincount(rows, weights=x0[src].astype(np.float64), minlength=ic["n"])
    assert sums(sv.tie_neighbours(ic))[mine].tobytes() == sums(ic["src"])[mine].tobytes(), name


def test_expected_values_restate_the_update():
    """a hand-sized graph: 0 -> 2, 1 -> 2, 2 -> 0 (internal order 2, 0, 1), x = (5, 7, 9) by internal id"""
    src, dst, n = np.array([0, 1, 2], np.uint32), np.array([2, 2, 0], np.uint32), 3
    import oracle
    out = oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED)
    inc = oracle.csr_build(src, dst, n, oracle.INCOMING, oracle.SORTED)
    plan = lm.make_plan(inc[0].astype(np.int64), inc[1], np.diff(out[0].astype(np.int64)), 1024, lm.CB_TAU_DEFAULT)
    assert list(plan["order"]) == [2, 0, 1] and plan["n_active"] == 2
    ic = sv.internal(plan, out, inc)
    x = np.array([5, 7, 9], np.float32)
    S, bad = sv.row_sums(ic, x)
    assert list(S) == [7 + 9, 5, 0] and not bad.any()
    score, xn = sv.expected(ic, x)
    base = (np.float32(1) - np.float32(0.85)) / np.float32(3)
    assert score[0] == np.float32(base + np.float32(np.float32(0.85) * np.float32(16)))
    assert xn[1] == score[1] / np.float32(1)
    x[1] = sv.nan_of([1])[0]
    assert sv.row_sums(ic, x)[1].tolist() == [True, False, False]
