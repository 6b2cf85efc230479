"""The CPU replay of gb_wcc (tools/wcc_model.py) on the fixtures of test_gpu_wcc.py: its labels are the
oracle's on every one, every fixture still reaches the k_cc_link_remaining classes, work lengths and skip
label it claims, and the bridge fixtures need the link they are named for: without it the labels are
wrong, and where the bridge is the last entry of its list, without that one entry.  A change of the
lane/warp threshold that moves a fixture off its path fails here, without a GPU."""
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
import wcc_fixtures as fx

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import wcc_model as wm  # noqa: E402


@pytest.fixture(scope="module", params=sorted(fx.FIXTURES))
def case(request):
    f = fx.get(request.param)
    return request.param, f, wm.replay(*f.out, *f.inc, f.rounds, f.samples)


def test_model_labels_are_the_oracle_labels(case):
    name, f, r = case
    want = oracle.wcc_min_label(*f.out)
    assert r.labels.tobytes() == want.tobytes(), name
    if not f.heavy:
        got = oracle.wcc_afforest(*f.out, *f.inc, neighbor_rounds=f.rounds, sampling_size=f.samples)
        assert got.tobytes() == want.tobytes(), name


def test_fixture_reaches_its_classes(case):
    name, f, r = case
    c = r.classes
    for v, want in f.expect.items():
        assert (c.cls[v], c.out_len[v], c.in_len[v]) == want, (name, v)
    if f.label is not None:
        assert r.found and r.label == f.label, (name, r.label)
    assert r.launches == 4 + (f.rounds > 0) + r.found


def test_bridges_need_the_link_they_are_named_for(case):
    name, f, r = case
    if f.bridge is None:
        return
    side, v = f.bridge
    assert r.labels[v] == r.labels[f.giant], name
    if side == "sample":        # the sample itself joins v to the giant, and v has nothing to link
        assert r.forest[v] == r.forest[f.giant] == r.label, name
        assert r.classes.cls[v] in (wm.SKIP, wm.DEAD), name
        return
    assert r.forest[v] != r.forest[f.giant] and r.forest[f.giant] == r.label, name
    assert r.classes.cls[v] in (wm.LANE, wm.WARP), name
    mine, other = ("keep_out", "keep_in") if side == "out" else ("keep_in", "keep_out")
    length = int((r.classes.out_len if side == "out" else r.classes.in_len)[v])

    def labels(**keep):
        return wm.replay(*f.out, *f.inc, f.rounds, f.samples, **keep).labels

    cut = labels(**{mine: {v: 0}})
    assert cut[v] != cut[f.giant], name
    if f.bridge_last:           # the last entry alone: a lane or warp that stops one short misses it
        cut = labels(**{mine: {v: length - 1}})
        assert cut[v] != cut[f.giant], name
    assert labels(**{other: {v: 0}}).tobytes() == r.labels.tobytes(), name   # the other list does not matter


def test_work_matrix_names():
    for k in fx.OUT_ONLY:
        f = fx.get(f"work_out_{k}")
        assert f.expect == {f.n - 1: ("dead" if k == 0 else "lane" if k <= 8 else "warp", k, 0)}
    assert wm.LANE_WORK == 8
    seen = set()
    for name in fx.FIXTURES:
        if name.startswith("work_"):
            f = fx.get(name)
            (v, (cls, o, i)), = f.expect.items()
            seen.add((cls, o + i))
            assert v == f.n - 1 and f.bridge[1] == v and (f.n % 32 != 0) == ("last_warp" in name), name
            assert f.bridge_last == (o + i > 0) and f.bridge[0] == ("sample" if o + i == 0 else
                                                                    "out" if o > i else "in"), name
    # the threshold and both sides of the 32-entry stride
    assert {("lane", 8), ("warp", 9), ("warp", 31), ("warp", 32), ("warp", 33), ("warp", 64),
            ("warp", 65), ("dead", 0), ("lane", 1)} <= seen


def test_deg_rounds_and_rounds_plus_one():
    f = fx.get("work_out_0")
    assert np.diff(f.out[0].astype(np.int64))[-1] == fx.WORK_ROUNDS
    f = fx.get("work_out_1")
    assert np.diff(f.out[0].astype(np.int64))[-1] == fx.WORK_ROUNDS + 1


def test_tied_samples_pick_the_smallest_label():
    f = fx.get("tied_samples")
    forest = wm.sampled_forest(*f.out, f.rounds)
    labels, counts = wm.sample_counts(forest, f.samples)
    assert len(labels) == 2 and counts[0] == counts[1] == f.samples // 2
    assert wm.sample_label(forest, f.samples) == (int(labels[0]), True) and labels[0] == f.label
    # any other tie rule would skip the other component
    assert labels[1] != f.label


def test_unsorted_first_rounds_follow_edge_list_order():
    f = fx.get("unsorted_first_rounds")
    s = oracle.csr_build(f.src, f.dst, f.n, oracle.OUTGOING, oracle.SORTED)
    assert f.out[1][f.out[0][10]:f.out[0][11]].tolist() == [1500, 11, 12]
    assert s[1][s[0][10]:s[0][11]].tolist() == [11, 12, 1500]
    r = wm.replay(*s, *f.inc, f.rounds, f.samples)        # sorted, the same edge is a late out-edge
    assert r.classes.cls[10] == wm.LANE and r.forest[10] == 10


def test_hub_is_served_by_the_warp():
    f = fx.get("hub")
    (h, (cls, o, i)), _ = f.expect.items()
    assert cls == "warp" and o > 10 ** 5 - 1 and i == 10 ** 5


def test_sample_label_clamps_and_edges():
    forest = np.arange(100, dtype=np.uint32)
    assert wm.sample_label(forest, 0) == (0, False)
    assert wm.sample_label(np.zeros(0, np.uint32), 5) == (0, False)
    one = int(wm.sample_draws(100, 1)[0])
    assert wm.sample_label(forest, 1) == (one, True)
    assert len(wm.sample_draws(100, 2 ** 40)) == 1 << 20
    assert (wm.sample_draws(100, (1 << 20) + 1) == wm.sample_draws(100, 2 ** 64 - 1)).all()


def test_rounds_clamp():
    f = fx.get("work_split_32_32")
    full = wm.sampled_forest(*f.out, 2 ** 64 - 1)
    assert (full == wm.sampled_forest(*f.out, 2 ** 32)).all()
    assert (full == oracle.wcc_min_label(*f.out)).all()
    c = wm.classify(f.out[0], f.inc[0], full, 2 ** 64 - 1, 0, False)
    assert (c.out_len == 0).all()
    assert wm.kernel_launches(2 ** 64 - 1, True) == 6 and wm.kernel_launches(0, False) == 4


@pytest.mark.parametrize("vb,ve", [(0, 13), (13, 50), (50, 1000), (0, 4100), (4099, 4100), (7, 7)])
def test_range_forest_is_a_subgraph(vb, ve):
    f = fx.get("bridge_out_late")
    part = wm.sampled_forest(*f.out, f.rounds, vb, ve)
    u, v = wm.first_round_edges(*f.out, f.rounds, vb, ve)
    assert ((u >= vb) & (u < ve)).all()
    assert (part[u] == part[v]).all() and (part <= np.arange(f.n)).all()
