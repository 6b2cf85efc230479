"""Directed graphs that drive gb_wcc (graph_b200/csrc/wcc.cu) onto each Afforest phase and kernel path: edges
into and out of the sampled giant that only one endpoint can link, a giant hooked under a component
holding id 0, tied sample counts, the lane/warp split of k_cc_link_remaining around its 8-entry threshold
and the 32-entry warp stride on the out side, the in side and both, a 10^5-edge hub, small n around a
warp, self loops and parallel edges inside and past the first rounds, stars, a 2^20 reverse-id path,
ids past 2^16 and 2^24, and an Unsorted build whose first rounds follow edge-list order.
Shared by the CPU replay of the kernels (test_wcc_model.py) and the GPU tests (test_gpu_wcc.py).

Most fixtures hold a giant: a path through a block of ids, every vertex also linked to the one two
further on, so that each of its out-lists starts with two edges inside the giant and the sampled forest
(neighbor_rounds >= 1) joins it whole.  The sample then skips it, and an edge that leaves it late in a
list is linked by its other endpoint only."""
from __future__ import annotations

import functools
import sys
from dataclasses import dataclass, field
from pathlib import Path

import numpy as np

import oracle

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import wcc_model as wm  # noqa: E402

ROUNDS = 2          # the default neighbor_rounds, which most claims are made for
SAMPLES = 1024      # the default sampling_size
_LAYOUT = {"Sorted": oracle.SORTED, "Unsorted": oracle.UNSORTED}


@dataclass
class Fixture:
    n: int
    src: np.ndarray
    dst: np.ndarray
    layout: str = "Sorted"
    rounds: int = ROUNDS                          # the neighbor_rounds the claims below hold for
    samples: int = SAMPLES                        # the sampling_size they hold for
    expect: dict = field(default_factory=dict)    # vertex -> (class, out-remainder, in-list length)
    label: int | None = None                      # the skip label the sample must pick
    bridge: tuple | None = None                   # ("out" | "in" | "sample", v): who alone links v to the giant
    giant: int | None = None                      # some vertex of the giant the bridge joins
    bridge_last: bool = False                     # the bridge is the last entry of v's list on its side
    tied: bool = False                            # the two most drawn labels are drawn equally often
    heavy: bool = False                           # checked against oracle.wcc_min_label only

    @functools.cached_property
    def out(self):
        return oracle.csr_build(self.src, self.dst, self.n, oracle.OUTGOING, _LAYOUT[self.layout])

    @functools.cached_property
    def inc(self):
        return oracle.csr_build(self.src, self.dst, self.n, oracle.INCOMING, _LAYOUT[self.layout])


class Edges:
    def __init__(self):
        self.s, self.d = [], []

    def add(self, s, d):
        s, d = np.atleast_1d(np.asarray(s, np.int64)), np.atleast_1d(np.asarray(d, np.int64))
        s, d = np.broadcast_arrays(s, d)
        self.s.append(s.ravel())
        self.d.append(d.ravel())
        return self

    def giant(self, lo: int, hi: int):
        """a path lo -> lo+1 -> ... -> hi-1 and the chords v -> v+2"""
        v = np.arange(lo, hi - 1)
        self.add(v, v + 1)
        return self.add(v[:-1], v[:-1] + 2)

    def fixture(self, n, **kw) -> Fixture:
        s = np.concatenate(self.s) if self.s else np.zeros(0, np.int64)
        d = np.concatenate(self.d) if self.d else np.zeros(0, np.int64)
        assert len(s) == 0 or max(s.max(), d.max()) < n
        return Fixture(n, s.astype(np.uint32), d.astype(np.uint32), **kw)


# ---- edges between the giant and the rest --------------------------------------------------------------
G_LO, G_HI, N_BRIDGE = 1000, 4000, 4100      # the giant [1000, 4000) holds 3/4 of n and every sample run


def bridge_out_late() -> Fixture:
    """v = 10 -> [11, 12, 1500]: the edge into the giant is at out-position 2 = rounds, and 1500, which
    has v in its in-list, is skipped; only v's out-remainder links {10, 11, 12} to the giant"""
    e = Edges().giant(G_LO, G_HI).add(10, [11, 12, 1500])
    return e.fixture(N_BRIDGE, expect={10: ("lane", 1, 0), 1500: ("skip", 0, 3)}, label=G_LO,
                     bridge=("out", 10), giant=1500, bridge_last=True)


def bridge_in_only() -> Fixture:
    """2000 -> [2001, 2002, 4050]: the edge out of the giant is late in a skipped list; only the in-list
    of v = 4050 links it"""
    e = Edges().giant(G_LO, G_HI).add(2000, 4050)
    return e.fixture(N_BRIDGE, expect={4050: ("lane", 0, 1), 2000: ("skip", 1, 2)}, label=G_LO,
                     bridge=("in", 4050), giant=2000, bridge_last=True)


def bridge_out_early() -> Fixture:
    """v = 20 -> [1500, 1501, 4060]: the edge into the giant is inside the first rounds, so the sample
    puts v in the giant, whose root it becomes, and v is skipped; 4060 links v's late edge from its in-list"""
    e = Edges().giant(G_LO, G_HI).add(20, [1500, 1501, 4060])
    return e.fixture(N_BRIDGE, expect={20: ("skip", 1, 0), 4060: ("lane", 0, 1)}, label=20,
                     bridge=("sample", 20), giant=1500)


def giant_hooked_under_0() -> Fixture:
    """the giant's root is 1000; {0, 1, 2} reaches it through 0 -> 1500 at out-position 2 only, so while
    the kernel runs the skipped root 1000 is hooked under 0"""
    e = Edges().giant(G_LO, G_HI).add(0, [1, 2, 1500])
    return e.fixture(N_BRIDGE, expect={0: ("lane", 1, 0)}, label=G_LO, bridge=("out", 0), giant=1500,
                     bridge_last=True)


def hooked_mid_kernel(k: int = 2000) -> Fixture:
    """y_i = 4000 + i is the root of {y_i, w_i = 6000 + i} (w_i -> y_i), and the giant vertex 1000 + i
    -> w_i late: w_i's in-list hooks y_i straight under the label 1000, and a y_i that is looked at
    afterwards drops out of its own lists"""
    i = np.arange(k)
    e = Edges().giant(G_LO, G_HI).add(6000 + i, 4000 + i).add(G_LO + i, 6000 + i)
    return e.fixture(8000, expect={6000: ("lane", 0, 1), 4000: ("lane", 0, 1)}, label=G_LO,
                     bridge=("in", 6000 + k - 1), giant=G_LO + k - 1, bridge_last=True)


def giant_at_top() -> Fixture:
    """the giant is [1001, 4001), the highest ids, and 5 -> [6, 7, 4000] reaches it late"""
    e = Edges().giant(1001, 4001).add(5, [6, 7, 4000])
    return e.fixture(4001, expect={5: ("lane", 1, 0), 4000: ("skip", 0, 3)}, label=1001, bridge=("out", 5),
                     giant=4000, bridge_last=True)


def tied_samples() -> Fixture:
    """two paths A and B over all of n = 4001 that the 1024 draws hit exactly 512 times each: the label
    is the smaller of their roots"""
    n = 4001
    hits = np.bincount(wm.sample_draws(n, SAMPLES), minlength=n)
    order = np.argsort(-hits, kind="stable")
    side = np.zeros(n, bool)
    tot = [0, 0]
    for v in order:                               # largest first, each onto the lighter side
        b = int(tot[1] < tot[0])
        side[v] = bool(b)
        tot[b] += hits[v]
    assert tot[0] == tot[1]
    a, b = np.flatnonzero(~side), np.flatnonzero(side)
    rng = np.random.default_rng(5)
    a, b = rng.permutation(a), rng.permutation(b)
    e = Edges().add(a[:-1], a[1:]).add(b[:-1], b[1:])
    return e.fixture(n, label=int(min(a.min(), b.min())), tied=True)


# ---- the lane/warp split ---------------------------------------------------------------------------------
WORK_ROUNDS = 3


def work(out_rem: int, in_len: int, at_end: bool = False) -> Fixture:
    """u = n - 1 has rounds + out_rem out-edges and in_len in-edges.  The last entry of its longer remaining
    list (the in-list on a tie) is its only link to a 1000-vertex giant whose ids lie above its other
    neighbours: the out-edge u -> g, or the in-edge g -> u, which comes after three giant edges in the
    skipped g's list.  A lane that stops one entry short, or a warp that stops after a 32-entry stride,
    leaves u's component apart.  With nothing remaining, g is the last of u's first rounds instead, and the
sample joins u's targets 0 and 1 to the giant.  The
    other neighbours are u's own: out-targets only u reaches, in-sources whose only edge is u.  n is a
    multiple of 32, or (at_end) 13 past one: u is the last lane of a full warp or of a partial last warp"""
    k = WORK_ROUNDS + out_rem + in_len
    glo = k
    n0 = glo + 1000 + 1
    n = n0 + ((13 if at_end else 0) - n0) % 32
    u, g = n - 1, glo + 500
    tg = np.arange(WORK_ROUNDS + out_rem)
    sr = WORK_ROUNDS + out_rem + np.arange(in_len)
    rem = out_rem + in_len
    side = "sample" if rem == 0 else "out" if out_rem > in_len else "in"
    if side == "in":
        sr[-1] = g
    else:
        tg[-1] = g
    e = Edges().giant(glo, glo + 1000).add(u, tg).add(sr, u).add(g, g + 3)
    cls = "dead" if rem == 0 else "lane" if rem <= 8 else "warp"
    return e.fixture(n, rounds=WORK_ROUNDS, expect={u: (cls, out_rem, in_len)},
                     label=0 if side == "sample" else glo, bridge=(side, u),
                     giant=g, bridge_last=side != "sample")


OUT_ONLY = (0, 1, 8, 9, 31, 32, 33, 64, 65)
IN_ONLY = (8, 9, 31, 32, 33, 64, 65)
SPLIT = ((4, 4), (5, 4), (4, 5), (16, 16), (17, 16), (31, 1), (1, 31), (32, 32), (33, 32), (64, 1), (1, 64))
AT_END = ((9, 0), (0, 33), (40, 40))


def hub() -> Fixture:
    """hub H = 2 * 10^5 with 10^5 + 100 out-edges (T = [10^5, 2 * 10^5), the first 100 twice) and 10^5
    in-edges from S = [0, 10^5), a path whose edges come first in every list of S: S is the skipped giant
    and the hub links both of its long lists with the whole warp at neighbor_rounds 1"""
    m = 100_000
    s = np.arange(m)
    h = 2 * m
    e = Edges().add(s[:-1], s[1:]).add(m - 1, m - 2).add(s, h)
    e.add(h, np.arange(m, 2 * m)).add(h, np.arange(m, m + 100))
    return e.fixture(h + 1, rounds=1, expect={h: ("warp", m + 99, m), m - 1: ("skip", 1, 1)}, label=0,
                     bridge=("in", h), giant=5, heavy=True)


def path_into_hub_unsampled(m: int = 100_000) -> Fixture:
    """regression: at neighbor_rounds 0 nothing is sampled, the lanes of k_cc_link_remaining hook the path
    0 -> 1 -> ... -> m-1 into a parent chain about as deep as the path, and the warp of the hub m, which
    every path vertex points at, walked that chain once per in-edge: some 30 s a call at m = 10^5 while
    the links did not shorten the paths they walked"""
    s = np.arange(m)
    e = Edges().add(s[:-1], s[1:]).add(s, m)
    return e.fixture(m + 1, rounds=0, expect={m: ("warp", 0, m), m - 1: ("lane", 1, 1)})


# ---- small n, loops and parallel edges, stars, deep chains -------------------------------------------------
def small(n: int) -> Fixture:
    """n // 2 random edges and a self loop on n - 1 (n = 1: the self loop alone)"""
    rng = np.random.default_rng(n)
    e = Edges().add(rng.integers(0, n, n // 2), rng.integers(0, n, n // 2)).add(n - 1, n - 1)
    return e.fixture(n)


def loops_and_parallel() -> Fixture:
    """50 -> [3, 3, 50, 50, 1500, 1500]: a parallel pair inside the first rounds, a loop pair past them
    and, last, a parallel pair into the giant, {3, 50}'s only link to it; 70 -> [70, 70, 80, 80, 80]:
    loops inside, parallel edges past; 90 -> 90 nine times"""
    e = Edges().giant(G_LO, G_HI).add(50, [3, 3, 50, 50, 1500, 1500]).add(70, [70, 70, 80, 80, 80])
    e.add(90, np.full(9, 90))
    return e.fixture(N_BRIDGE, expect={50: ("lane", 4, 2), 70: ("lane", 3, 2), 90: ("warp", 7, 9)}, label=G_LO,
                     bridge=("out", 50), giant=1500)


def star(hub_last: bool, inward: bool = False) -> Fixture:
    """a star over 4001 vertices: the hub's out-edges to every leaf, or (inward) every leaf's edge to it"""
    n = 4001
    h = n - 1 if hub_last else 0
    leaves = np.delete(np.arange(n), h)
    e = Edges().add(leaves, h) if inward else Edges().add(h, leaves)
    return e.fixture(n)


def reverse_path(n: int = 1 << 20) -> Fixture:
    """v -> v - 1 for every v > 0: k_cc_sample hooks every root under the next lower one in one launch,
    a parent chain n deep for k_cc_compress"""
    v = np.arange(1, n)
    return Edges().add(v, v - 1).fixture(n, expect={n - 1: ("dead", 0, 0), 0: ("skip", 0, 1)}, label=0,
                                         heavy=True)


def comb(k: int = 4096, tooth: int = 3) -> Fixture:
    """a spine 0 <- 1 <- ... <- k-1 and under every spine vertex a tooth of `tooth` vertices hanging off
    it by edges pointing up to it"""
    e = Edges()
    spine = np.arange(k)
    e.add(spine[1:], spine[:-1])
    prev = spine
    for t in range(tooth):
        cur = k * (t + 1) + spine
        e.add(cur, prev)
        prev = cur
    return e.fixture(k * (tooth + 1))


def high_ids(bits: int) -> Fixture:
    """ids around t = 2^bits: a path t-2 -> t-1 -> t -> t+1 -> t+2 whose edge out of t-1 comes after
    t-1 -> [t-100, t-99], a late edge t+5 -> [t-50, t-49, t+2] into it, and n-1 -> t+10"""
    t = 1 << bits
    n = t + 40
    e = Edges().giant(100, 400).add(np.arange(t - 2, t + 2), np.arange(t - 1, t + 3))
    e.add(t + 5, [t - 50, t - 49, t + 2]).add(t - 1, [t - 100, t - 99]).add(n - 1, t + 10)
    return e.fixture(n, expect={t + 5: ("lane", 1, 0), t - 1: ("lane", 1, 1), t + 2: ("lane", 0, 2)},
                     heavy=bits >= 24)


def unsorted_first_rounds() -> Fixture:
    """v = 10 -> 1500 -> ... listed first, then 10 -> 11 and 10 -> 12: in edge-list order the edge into
    the giant is one of the first rounds (a Sorted build would put it last, past them)"""
    e = Edges().giant(G_LO, G_HI).add(10, [1500, 11, 12])
    return e.fixture(N_BRIDGE, layout="Unsorted", expect={10: ("skip", 1, 0), 12: ("lane", 0, 1)}, label=10,
                     bridge=("sample", 10), giant=1500)


FIXTURES = {
    "bridge_out_late": bridge_out_late,
    "bridge_in_only": bridge_in_only,
    "bridge_out_early": bridge_out_early,
    "giant_hooked_under_0": giant_hooked_under_0,
    "hooked_mid_kernel": hooked_mid_kernel,
    "giant_at_top": giant_at_top,
    "tied_samples": tied_samples,
    **{f"work_out_{k}": (lambda k=k: work(k, 0)) for k in OUT_ONLY},
    **{f"work_in_{k}": (lambda k=k: work(0, k)) for k in IN_ONLY},
    **{f"work_split_{a}_{b}": (lambda a=a, b=b: work(a, b)) for a, b in SPLIT},
    **{f"work_last_warp_{a}_{b}": (lambda a=a, b=b: work(a, b, at_end=True)) for a, b in AT_END},
    "hub": hub,
    "path_into_hub_unsampled": path_into_hub_unsampled,
    **{f"n_{n}": (lambda n=n: small(n)) for n in (1, 31, 32, 33, 4001)},
    "loops_and_parallel": loops_and_parallel,
    "star_hub_first": lambda: star(False),
    "star_hub_last": lambda: star(True),
    "star_inward_hub_last": lambda: star(True, inward=True),
    "reverse_path_2_20": reverse_path,
    "comb": comb,
    "ids_past_2_16": lambda: high_ids(16),
    "ids_past_2_24": lambda: high_ids(24),
    "unsorted_first_rounds": unsorted_first_rounds,
}
BRIDGES = sorted(k for k, f in FIXTURES.items() if k.startswith(("bridge_", "giant_", "hooked_")) or k == "hub")


@functools.lru_cache(maxsize=None)
def get(name: str) -> Fixture:
    return FIXTURES[name]()
