"""Delta-stepping SSSP (graph_b200/csrc/sssp.cu) on graphs that target its queue bookkeeping: a far pile that
vertices re-enter in every bucket (it outgrew its capacity while a vertex could have one entry per bucket),
lists around the lane/warp split of k_sssp_relax, hub edges racing on one target, warps appending to the
near queue and the far pile at once, distances exactly on a bucket bound, a pile left with nothing live, f32
extremes, tiny graphs, the device entry point, repeated calls, one bucket per distance and RMAT-20.

Every result is checked twice: bit for bit against oracle.sssp_bellman_ford on the CSR read back from the
device (so the order the build gives parallel edges cannot matter), and by an O(m) certificate that does not
use the oracle: the start is at 0, no edge improves a distance in f32, and every reached vertex is reached
from the start over tight edges.  Graphs are in sssp_fixtures.py; test_sssp_model.py replays them on the
CPU."""
import ctypes as C

import numpy as np
import pytest

import oracle
import sssp_fixtures as fx

pytestmark = pytest.mark.gpu

FLT_MAX = fx.FLT_MAX


@pytest.fixture(scope="module")
def gb():
    import graph_b200
    return graph_b200


def certify(off, tgt, w, start, d):
    """the certificate of the f32 shortest-path distances d; returns the number of reached vertices"""
    from scipy.sparse import csr_matrix
    from scipy.sparse.csgraph import breadth_first_order
    n = len(off) - 1
    assert d.dtype == np.float32 and len(d) == n
    assert d[start] == 0.0 and not np.signbit(d[start])
    assert np.isfinite(d).all() and (d >= 0).all()
    src = np.repeat(np.arange(n, dtype=np.int64), np.diff(off.astype(np.int64)))
    tgt = tgt.astype(np.int64)
    live = d[src] < FLT_MAX
    with np.errstate(over="ignore"):
        via = d[src] + w                                  # f32 + f32: rounded to f32
    bad = live & ~(d[tgt] <= via)
    assert not bad.any(), f"{int(bad.sum())} edges improve a distance, first {np.flatnonzero(bad)[:5]}"
    tight = live & (d[tgt] == via) & (d[tgt] < FLT_MAX)
    adj = csr_matrix((np.ones(int(tight.sum()), np.int8), (src[tight], tgt[tight])), shape=(n, n))
    order = breadth_first_order(adj, start, directed=True, return_predecessors=False)
    on_tight = np.zeros(n, bool)
    on_tight[order] = True
    reached = d < FLT_MAX
    assert (on_tight == reached).all(), f"{int((on_tight != reached).sum())} vertices not reached over tight edges"
    return int(reached.sum())


def check_run(g, start, delta):
    """g.delta_stepping == Bellman-Ford on g's own CSR, bit for bit, and the certificate holds"""
    off, tgt = g.csr("out")
    w = g.out_weights()
    got = g.delta_stepping(start_node=start, delta=delta).distances()
    want = oracle.sssp_bellman_ford(off, tgt, w, start)
    assert got.tobytes() == want.tobytes(), int((got.view(np.uint32) != want.view(np.uint32)).sum())
    certify(off, tgt, w, start, got)
    return got


def build(gb, f, layout=None):
    return gb.DiGraph.from_numpy(np.stack([f.src, f.dst], 1), layout=layout or gb.Layout.Sorted, weights=f.w,
                                 node_count=f.n)


# ---- the far pile: one entry per vertex, whatever the number of buckets ------------------------------------
@pytest.mark.parametrize("k", [64, 200])
def test_comb(gb, k):
    """chain vertex i improves every target in bucket i; the pile held k * s entries while a vertex could have
    one per bucket (4096 for 64 x 64 against a capacity of 2n + 1024 = 1280)"""
    f = fx.comb(k, k)
    d = check_run(build(gb, f), f.start, f.delta)
    assert (d[:k] == np.arange(k)).all() and (d[k:] == 3 * k + 1).all()


@pytest.mark.parametrize("k", [64, 200])
def test_star(gb, k):
    """the start queues every a_i in its first pass; each a_i is then settled in a bucket of its own"""
    f = fx.star(k, k)
    d = check_run(build(gb, f), f.start, f.delta)
    assert (d[:k + 1] == np.arange(k + 1)).all() and (d[k + 1:] == 3 * k).all()


@pytest.mark.parametrize("name", ["dense128", "dense256"])
def test_dense_random(gb, name):
    """128 / 256 uniform random out-edges per vertex at delta 1e-3 / 1e-30: under the old pile rule the pile
    grows with the log of the in-degree times n, past 2n + 1024 here"""
    f = fx.FIXTURES[name]()
    d = check_run(build(gb, f), f.start, f.delta)
    assert (d < FLT_MAX).sum() > 0.99 * f.n


# ---- k_sssp_relax: lane and warp walks, reservations -----------------------------------------------------
@pytest.mark.parametrize("layout", ["Unsorted", "Sorted"])
def test_degrees_around_the_lane_warp_split(gb, layout):
    """out-degrees 0, 1, 7, 8, 9, 31, 32, 33, 1000 and a hub of 1e5 edges relaxed in one pass; every edge but
    the hub's parallel ones leads to a private leaf, so a skipped edge leaves a vertex unreached"""
    f = fx.degrees()
    d = check_run(build(gb, f, getattr(gb.Layout, layout)), f.start, f.delta)
    assert (d < FLT_MAX).all()
    hub = len(fx.DEGREES) * 4 + 1
    assert d[f.n - 1] == np.float32(d[hub] + np.float32(0.25))       # the lightest of the parallel edges


def test_warp_appends_to_near_and_far_together(gb):
    f = fx.mixed_hub()
    d = check_run(build(gb, f), f.start, f.delta)
    t = np.arange(1, f.n)
    assert (d[t[t % 2 == 0]] < 1.0).all() and (d < FLT_MAX).all()


# ---- bucket bounds ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["int_half", "int_one", "int_two", "tenths"])
def test_distances_on_bucket_bounds(gb, name):
    """integer weights with delta 0.5 / 1 / 2, and multiples of f32(0.1) with delta f32(0.1): a distance equal
    to a bucket's upper bound goes to the pile and is settled in the next bucket"""
    f = fx.FIXTURES[name]()
    d = check_run(build(gb, f), f.start, f.delta)
    reached = d[d < FLT_MAX]
    assert len(reached) > 0.9 * f.n
    if name.startswith("int"):
        assert (reached == np.floor(reached)).all() and len(np.unique(reached)) >= 4


def test_pile_with_nothing_live(gb):
    """x enters the pile at 5 and is improved to 0.2 in the first bucket: the loop ends on an empty minimum"""
    f = fx.far_into_near()
    d = check_run(build(gb, f), f.start, f.delta)
    assert d.tolist() == [0.0, np.float32(0.1), np.float32(np.float32(0.1) + np.float32(0.1))]


# ---- f32 extremes and tiny graphs -----------------------------------------------------------------------
def test_f32_extremes(gb):
    f = fx.extremes()
    d = check_run(build(gb, f), f.start, f.delta)
    half = np.float32(FLT_MAX) / np.float32(2)
    assert [bool(d[i] == FLT_MAX) for i in (1, 2, 5, 6, 8)] == [True] * 5   # FLT_MAX is "unreached"
    assert d[3] == 0.0 and not np.signbit(d[3]) and d[11] == 0.0
    assert d[4] == half and d[7] == half and d[10] == half and d[12] == 2.0


@pytest.mark.parametrize("name,want", [("single_self_loop", [0.0]),
                                       ("isolated_start", [FLT_MAX, FLT_MAX, 0.0, FLT_MAX, FLT_MAX]),
                                       ("self_loop_start", [0.0, FLT_MAX, FLT_MAX])])
def test_tiny_graphs(gb, name, want):
    f = fx.FIXTURES[name]()
    d = check_run(build(gb, f), f.start, f.delta)
    assert d.tobytes() == np.array(want, np.float32).tobytes()


# ---- the device entry point and repeated calls ----------------------------------------------------------
def test_device_entry_and_repeated_calls(gb):
    import torch
    from graph_b200 import _capi
    from graph_b200._capi import check, lib
    f = fx.dense_random(3000, 128, 0.001, 21)
    g = build(gb, f)
    starts = (f.start, 1234)
    first = {s: check_run(g, s, f.delta) for s in starts}

    def on_device(s):
        buf = torch.full((f.n,), float("nan"), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()          # the fill runs on torch's stream, the graph has its own
        cfg = _capi.SsspConfig(s, f.delta)
        check(lib.gb_sssp_device(g._g, C.byref(cfg), C.c_void_p(buf.data_ptr())))
        return buf.cpu().numpy()

    for rnd in range(3):                  # alternating starts and entry points: nothing carries over
        for s in starts:
            assert on_device(s).tobytes() == first[s].tobytes(), (rnd, s)
            assert g.delta_stepping(start_node=s, delta=f.delta).distances().tobytes() == first[s].tobytes()


# ---- many buckets, and size -----------------------------------------------------------------------------
def rmat_start(g):
    off, _ = g.csr("out")
    return int(np.argmax(np.diff(off.astype(np.int64))))


def test_rmat16_one_bucket_per_distance(gb):
    """delta 1e-30: every bucket is [dmin, next f32 above dmin), so there is one bucket per distinct distance"""
    g = gb.DiGraph.rmat(16, seed=42, layout=gb.Layout.Sorted, weights=True)
    d = check_run(g, rmat_start(g), 1e-30)
    distinct = len(np.unique(d[(d > 0) & (d < FLT_MAX)]))
    assert distinct > 10000
    # each bucket after the first takes a minimum, a split and at least one relax pass (3 launches); below
    # 2^22 delta a bucket can hold a few distances
    assert g.last_timing()["kernel_launches"] >= 2 * distinct


def test_rmat20_certificate(gb):
    g = gb.DiGraph.rmat(20, seed=42, layout=gb.Layout.Sorted, weights=True)
    off, tgt = g.csr("out")
    w = g.out_weights()
    start = rmat_start(g)
    d = g.delta_stepping(start_node=start, delta=0.01).distances()
    assert certify(off, tgt, w, start, d) > (1 << 19)
