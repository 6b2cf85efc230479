"""Weighted graphs that drive the delta-stepping queues of graph_b200/csrc/sssp.cu onto their edges: a far pile
that a vertex re-enters in many buckets, adjacency lists around the lane/warp split of k_sssp_relax, warps
that append to the near queue and the far pile at once, distances that land exactly on a bucket bound, f32
extremes and tiny graphs.  Shared by the CPU replay of the queue rules (test_sssp_model.py) and the GPU
tests (test_gpu_sssp.py)."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

F32 = np.float32
FLT_MAX = np.finfo(np.float32).max


@dataclass
class Fixture:
    src: np.ndarray
    dst: np.ndarray
    w: np.ndarray
    n: int
    start: int
    delta: float          # an f32 value


def _fx(src, dst, w, n, start, delta):
    return Fixture(np.asarray(src, np.uint32), np.asarray(dst, np.uint32), np.asarray(w, np.float32), int(n),
                   int(start), float(F32(delta)))


def comb(k, s):
    """a chain 0 -> 1 -> ... -> k-1 of weight 1, and chain vertex i -> each of s targets with weight 4k - 2i.
    Chain vertex i is alone in bucket i (delta 1) and improves every target to 4k - i, still far: every
    target re-enters the pile in each of the k buckets."""
    i = np.arange(k)
    tg = np.arange(k, k + s)
    src = np.concatenate([i[:-1], np.repeat(i, s)])
    dst = np.concatenate([i[1:], np.tile(tg, k)])
    w = np.concatenate([np.ones(k - 1), np.repeat(4 * k - 2 * i, s)])
    return _fx(src, dst, w, k + s, 0, 1.0)


def star(k, s):
    """start 0 -> a_i (i = 1..k) with weight i, a_i -> each of s targets with weight 4k - 2i: the start's
    first pass puts every a_i into the pile, and each a_i is then settled in a bucket of its own"""
    a = np.arange(1, k + 1)
    tg = np.arange(k + 1, k + 1 + s)
    src = np.concatenate([np.zeros(k, np.int64), np.repeat(a, s)])
    dst = np.concatenate([a, np.tile(tg, k)])
    w = np.concatenate([a, np.repeat(4 * k - 2 * a, s)])
    return _fx(src, dst, w, k + 1 + s, 0, 1.0)


def dense_random(n, deg, delta, seed):
    """deg out-edges per vertex to uniform random targets, weights U[0, 1)"""
    rng = np.random.default_rng(seed)
    src = np.repeat(np.arange(n), deg)
    dst = rng.integers(0, n, n * deg)
    return _fx(src, dst, rng.random(n * deg, dtype=np.float32), n, 0, delta)


DEGREES = (0, 1, 7, 8, 9, 31, 32, 33, 1000)
HUB_EDGES = 100_000
HUB_PARALLEL = 1000


def degrees():
    """start 0 -> 4 probes of each out-degree in DEGREES and one hub of HUB_EDGES edges, all in the first
    bucket, so one near pass relaxes lists on both sides of the lane/warp split in the same warps.  Every
    probe and hub edge leads to a private leaf (a dropped or skipped edge leaves its leaf unreached),
    except the hub's last HUB_PARALLEL edges: parallel edges to one target with distinct weights, shuffled,
    whose lanes race on one atomicMin and one stamp."""
    rng = np.random.default_rng(11)
    probe_degs = [d for d in DEGREES for _ in range(4)]
    nprobe = len(probe_degs) + 1                      # + the hub
    nxt = 1 + nprobe
    src, dst, w = [np.zeros(nprobe, np.int64)], [np.arange(1, 1 + nprobe)], \
        [(rng.permutation(nprobe) + 1) * F32(1e-3)]
    for p, d in enumerate(probe_degs):
        src.append(np.full(d, 1 + p))
        dst.append(np.arange(nxt, nxt + d))
        w.append(rng.random(d, dtype=np.float32) * F32(2.0))
        nxt += d
    hub = nprobe
    leaves = HUB_EDGES - HUB_PARALLEL
    src.append(np.full(HUB_EDGES, hub))
    dst.append(np.concatenate([np.arange(nxt, nxt + leaves), np.full(HUB_PARALLEL, nxt + leaves)]))
    w.append(np.concatenate([rng.random(leaves, dtype=np.float32) * F32(2.0),
                             F32(0.25) + rng.permutation(HUB_PARALLEL).astype(np.float32) * F32(1e-3)]))
    nxt += leaves + 1
    return _fx(np.concatenate(src), np.concatenate(dst), np.concatenate(w), nxt, 0, 1.0)


def mixed_hub(n=4096):
    """a hub (the start) whose even edges weigh below delta and odd edges far above it: the lanes of one warp
    step append to the near queue and the far pile in the same window; each target has two onward edges"""
    rng = np.random.default_rng(12)
    t = np.arange(1, n)
    hw = np.where(t % 2 == 0, rng.random(n - 1, dtype=np.float32) * F32(0.5), F32(100.0) + rng.random(n - 1))
    src = np.concatenate([np.zeros(n - 1, np.int64), np.repeat(t, 2)])
    dst = np.concatenate([t, rng.integers(1, n, 2 * (n - 1))])
    w = np.concatenate([hw, rng.random(2 * (n - 1), dtype=np.float32) * F32(3.0)])
    return _fx(src, dst, w, n, 0, 1.0)


def on_bounds(kind, delta, n=3000):
    """8 random out-edges per vertex with weights 0..5 (kind "int") or 0..5 times f32(0.1) ("tenths"): most
    distances are sums that land exactly on a bucket bound, which belongs to the next bucket"""
    rng = np.random.default_rng(13)
    src = np.repeat(np.arange(n), 8)
    dst = rng.integers(0, n, 8 * n)
    k = rng.integers(0, 6, 8 * n).astype(np.float32)
    w = k if kind == "int" else k * F32(0.1)
    return _fx(src, dst, w, n, 0, delta)


def far_into_near():
    """start -> x (weight 5) files x in the pile; start -> y -> x (0.1 + 0.1) improves it into the first
    bucket before that bucket drains, so the pile holds nothing live and the loop ends on h_min == inf"""
    return _fx([0, 0, 1], [2, 1, 2], [5.0, 0.1, 0.1], 3, 0, 1.0)


def extremes():
    """weights FLT_MAX, +inf and -0.0; a path whose f32 sum is exactly FLT_MAX (the unreached distance, so its
    end stays unreached); sums that overflow to inf"""
    half = F32(FLT_MAX) / F32(2)
    e = [(0, 1, FLT_MAX),      # 0 + FLT_MAX is not below FLT_MAX: 1 stays unreached
         (0, 2, np.inf),       # unreached
         (0, 3, -0.0),         # reached at +0
         (3, 4, half),         # FLT_MAX / 2
         (4, 5, half),         # FLT_MAX / 2 + FLT_MAX / 2 == FLT_MAX: unreached
         (4, 6, FLT_MAX),      # overflows to inf: unreached
         (4, 7, 1.0),          # rounds back to FLT_MAX / 2
         (7, 8, np.inf),
         (3, 9, 3.0e38),       # 3e38 + (FLT_MAX / 2) overflows: 10 only through 4
         (9, 10, half),
         (4, 10, 1.0e30),
         (3, 11, -0.0),
         (11, 12, 2.0), (12, 12, -0.0), (12, 3, 0.0)]
    src, dst, w = zip(*e)
    return _fx(src, dst, np.array(w, np.float32), 13, 0, 1.0)


def single_self_loop():
    return _fx([0], [0], [1.0], 1, 0, 1.0)


def isolated_start():
    """the start has no edges at all; the rest of the graph has some"""
    return _fx([0, 1, 3, 4], [1, 2, 4, 0], [1.0, 2.0, 0.5, 0.0], 5, 2, 1.0)


def self_loop_start():
    """the start's only edge is a self-loop"""
    return _fx([0, 1, 2], [0, 2, 0], [0.0, 1.0, 1.0], 3, 0, 0.5)


FIXTURES = {
    "comb64": lambda: comb(64, 64),
    "comb200": lambda: comb(200, 200),
    "star64": lambda: star(64, 64),
    "star200": lambda: star(200, 200),
    "dense128": lambda: dense_random(3000, 128, 0.001, 21),
    "dense256": lambda: dense_random(2000, 256, 1e-30, 22),
    "degrees": degrees,
    "mixed_hub": mixed_hub,
    "int_half": lambda: on_bounds("int", 0.5),
    "int_one": lambda: on_bounds("int", 1.0),
    "int_two": lambda: on_bounds("int", 2.0),
    "tenths": lambda: on_bounds("tenths", 0.1),
    "far_into_near": far_into_near,
    "extremes": extremes,
    "single_self_loop": single_self_loop,
    "isolated_start": isolated_start,
    "self_loop_start": self_loop_start,
}
# the fixtures the CPU replay runs (all of them: the large cases of test_gpu_sssp.py are RMAT graphs)
REPLAYED = tuple(FIXTURES)
# the fixtures whose far pile overflowed 2n + 1024 entries while a vertex could have one entry per bucket
LEGACY_OVERFLOW = ("comb64", "comb200", "star64", "star200", "dense128", "dense256")
