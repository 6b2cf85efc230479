"""gb_wcc (the Afforest WCC of graph_b200/csrc/wcc.cu) on the H100 against the oracle and the CPU replay of
tools/wcc_model.py, on every fixture of wcc_fixtures.py: the labels over a grid of neighbor_rounds and
sampling_size values (both at and past their clamps) are the bytes of oracle.wcc_min_label on the CSR read
back from the device, each call reports the model's launches, the forest after INIT / SAMPLE / COMPRESS is
the model's sampled forest and gb_wcc_sample_label picks the model's label, gb_wcc_device agrees with
gb_wcc, and virtual ranks on 32-aligned and unaligned vertex ranges end with the oracle's labels after
sampling exactly the model's per-range forests.  Forests after LINK_REMAINING are not compared: which
vertices are hooked under the label before their own turn depends on the schedule.  Every fixture, the
2^24-id one, the 2^20 path and the hub included, runs the whole grid: the file takes about a minute on
one H100, most of it in those three."""
import ctypes as C
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
import wcc_fixtures as fx

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import wcc_model as wm  # noqa: E402

pytestmark = pytest.mark.gpu

ROUNDS = (0, 1, 2, 2 ** 32, 2 ** 64 - 1)                       # and each fixture's own
SAMPLES = (0, 1, 16, 1024, 2 ** 20 + 1, 2 ** 40)
WORLDS = (2, 3, 5, 8)
RANKED = fx.BRIDGES + ["n_31", "n_33", "work_out_33", "work_in_65", "work_last_warp_40_40", "work_split_32_32",
                       "tied_samples"]


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


_graphs = {}


def device(gb, name):
    """(fixture, its device twin, the oracle's labels on the CSR read back from the device)"""
    if name not in _graphs:
        _graphs.clear()                          # one twin at a time: the 2^24-id fixture is large
        f = fx.get(name)
        g = gb.DiGraph.from_csr(*f.out, *f.inc)
        out, inc = g.csr("out"), g.csr("in")
        for got, want in zip(out + inc, f.out + f.inc):
            assert got.tobytes() == want.tobytes(), name
        _graphs[name] = (f, g, oracle.wcc_min_label(*out))
    return _graphs[name]


def host(p):
    return p.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("name", sorted(fx.FIXTURES))
def test_labels_and_launches_over_the_config_grid(gb, name):
    f, g, want = device(gb, name)
    for rounds in sorted({*ROUNDS, f.rounds}):
        for samples in SAMPLES:
            comp = g.wcc(neighbor_rounds=rounds, sampling_size=samples).components()
            assert comp.tobytes() == want.tobytes(), (name, rounds, samples)
            assert g.last_timing()["kernel_launches"] == wm.kernel_launches(rounds, samples > 0), \
                (name, rounds, samples)


def test_unsorted_build_keeps_edge_list_order(gb):
    f = fx.get("unsorted_first_rounds")
    g = gb.DiGraph.from_numpy(np.stack([f.src, f.dst], 1), layout=gb.Layout.Unsorted, node_count=f.n)
    off, tgt = g.csr("out")
    assert off.tobytes() == f.out[0].tobytes() and tgt.tobytes() == f.out[1].tobytes()
    want = oracle.wcc_min_label(off, tgt)
    for rounds in (1, 2, 3):
        assert g.wcc(neighbor_rounds=rounds).components().tobytes() == want.tobytes(), rounds


@pytest.mark.parametrize("name", sorted(fx.FIXTURES))
def test_shard_phases_on_one_rank(gb, name):
    """the phases over [0, n): the sampled forest and the label are the model's, the end is the oracle's"""
    from graph_b200 import _capi
    from graph_b200.multigpu import CudaWccBackend
    f, g, want = device(gb, name)
    for rounds in sorted({0, 1, f.rounds, 2 ** 64 - 1}):
        forest = wm.sampled_forest(*f.out, rounds)
        for samples in sorted({0, 1, 16, f.samples, 2 ** 40}):
            b = CudaWccBackend(g, neighbor_rounds=rounds, sampling_size=samples)
            p = b.new_parent()
            b.phase(_capi.WCC_INIT, p)
            b.phase(_capi.WCC_SAMPLE, p, 0, f.n)
            b.phase(_capi.WCC_COMPRESS, p)
            if samples == 0:
                assert host(p).tobytes() == forest.tobytes(), (name, rounds)
            label = b.sample_label(p)
            assert label == wm.sample_label(forest, samples), (name, rounds, samples)
            if rounds == f.rounds and samples == f.samples and f.label is not None:
                assert label == (f.label, True), name
            b.phase(_capi.WCC_LINK_REMAINING, p, 0, f.n, *label)
            b.phase(_capi.WCC_COMPRESS, p)
            assert host(p).tobytes() == want.tobytes(), (name, rounds, samples)


@pytest.mark.parametrize("name", sorted(fx.FIXTURES))
def test_wcc_device_into_a_tensor(gb, name):
    import torch
    from graph_b200 import _capi
    f, g, want = device(gb, name)
    cfg = _capi.WccConfig(16384, f.rounds, f.samples)
    got = []
    for _ in range(2):
        t = torch.full((f.n,), -1, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()                 # the fill runs on torch's stream, the call on the graph's
        _capi.check(_capi.lib.gb_wcc_device(g._g, C.byref(cfg), C.c_void_p(t.data_ptr())))
        got.append(host(t))
    assert got[0].tobytes() == got[1].tobytes() == want.tobytes(), name
    assert g.wcc(neighbor_rounds=f.rounds, sampling_size=f.samples).components().tobytes() == want.tobytes()


def unaligned_ranges(n, world):
    """world contiguous ranges over [0, n) cut at ids that are not multiples of 32 (where n allows)"""
    rng = np.random.default_rng(n * 31 + world)
    cuts = np.sort(rng.choice(np.arange(1, n), min(world - 1, n - 1), replace=False)) if n > 1 else []
    cuts = [c + 1 if c % 32 == 0 and c + 1 < n else c for c in cuts]
    cuts = [0] + sorted(set(int(c) for c in cuts)) + [n]
    cuts += [n] * (world + 1 - len(cuts))
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


@pytest.mark.parametrize("aligned", [True, False], ids=["aligned", "unaligned"])
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("name", RANKED)
def test_virtual_ranks(gb, name, world, aligned):
    from graph_b200.multigpu import vertex_ranges
    from virtual_ranks import wcc_virtual_ranks
    f, g, want = device(gb, name)
    ranges = vertex_ranges(f.n, world) if aligned else unaligned_ranges(f.n, world)
    assert ranges[0][0] == 0 and ranges[-1][1] == f.n
    assert all(a[1] == b[0] for a, b in zip(ranges, ranges[1:]))
    if not aligned and f.n > 64 * world:
        assert all(vb % 32 for vb, _ in ranges[1:]), ranges
    forest = wm.sampled_forest(*f.out, f.rounds)
    forests = []
    parents, labels = wcc_virtual_ranks(g, world, ranges=ranges, forests=forests, neighbor_rounds=f.rounds,
                                        sampling_size=f.samples)
    for r, (vb, ve) in enumerate(ranges):
        own, merged = forests[r]
        assert own.tobytes() == wm.sampled_forest(*f.out, f.rounds, vb, ve).tobytes(), (name, r)
        assert merged.tobytes() == forest.tobytes(), (name, r)
        assert labels[r] == wm.sample_label(forest, f.samples), (name, r)
        assert host(parents[r]).tobytes() == want.tobytes(), (name, r)
