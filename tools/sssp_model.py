"""sssp_model.py — a one-thread replay of the delta-stepping host loop of sssp.cu and its queue rules.

The replay follows sssp_impl pass by pass: the near queue of a bucket is relaxed in queue order, a target is
appended to the near queue once per pass (near stamps) and to the far pile only while it has no entry there
(in_pile), a near entry below the bucket's lower bound is stale, k_sssp_min_far takes the smallest pile
distance >= the old upper bound, sssp_next_bucket (ported below) gives the next bucket, and the split moves
pile entries below the new upper bound to the near queue (clearing in_pile) and carries the rest.
Arithmetic is f32 throughout.  It returns the distances, the number of buckets and the largest near queue
and far pile, so that the bound the device's queue capacity relies on can be checked on the CPU.

`legacy_carry=True` replays the rule sssp.cu had before in_pile: a target entered the pile once per bucket
epoch, and the split carried every entry still far, so a vertex improved in k buckets while it stayed far
had k entries.
Run: python tools/sssp_model.py   (also exercised by tests/test_sssp_model.py)."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

F32 = np.float32
FLT_MAX = np.finfo(np.float32).max
INF = F32(np.inf)


def sssp_next_bucket(dmin, delta, old_upper):
    """sssp_bucket.h: (lower, upper, steps) of the bucket after one whose upper bound was old_upper"""
    dmin, delta, old_upper = F32(dmin), F32(delta), F32(old_upper)
    with np.errstate(over="ignore", invalid="ignore"):
        lower, upper, steps = dmin, np.nextafter(dmin, INF), 0
        q = dmin / delta
        if not (q < F32(4194304.0)):
            return lower, upper, steps
        k = np.floor(q)
        lo, up = delta * k, delta * (k + F32(1.0))
        if not (dmin < up):
            k += F32(1.0)
            lo = up
            up = delta * (k + F32(1.0))
            steps = 1
        elif dmin < lo:
            k -= F32(1.0)
            up = lo
            lo = delta * k
            steps = 1
        if old_upper <= lo and lo <= dmin and dmin < up:
            lower, upper = lo, up
    return lower, upper, steps


@dataclass
class Replay:
    dist: np.ndarray
    buckets: int
    max_near: int
    max_far: int


def replay(off, tgt, w, start: int, delta: float, legacy_carry: bool = False) -> Replay:
    off = np.asarray(off, np.int64)
    tgt = np.asarray(tgt, np.int64)
    w = np.asarray(w, np.float32)
    n = len(off) - 1
    delta = F32(delta)
    dist = np.full(n, FLT_MAX, np.float32)
    dist[start] = 0.0
    near_stamp = np.zeros(n, np.int64)
    far_stamp = np.zeros(n, np.int64)                     # legacy_carry: the last epoch t entered the pile
    in_pile = np.zeros(n, bool)
    pass_, epoch = 0, 1
    near, far = [start], []
    lower, upper = F32(0.0), delta
    buckets, max_near, max_far = 1, 1, 0
    while True:
        while near:                                       # drain the near queue of this bucket
            pass_ += 1
            out = []
            for u in near:
                du = dist[u]
                if du < lower:                            # stale: settled in an earlier bucket
                    continue
                b, e = off[u], off[u + 1]
                if e == b:
                    continue
                with np.errstate(over="ignore"):
                    nd = du + w[b:e]
                ts = tgt[b:e]
                # an edge can only improve its target if it beats the distance before this list
                for i in np.flatnonzero(nd < dist[ts]):
                    t, d = ts[i], nd[i]
                    if not (d < dist[t]):
                        continue
                    dist[t] = d
                    if d < upper:
                        if near_stamp[t] < pass_:
                            near_stamp[t] = pass_
                            out.append(t)
                    elif legacy_carry:
                        if far_stamp[t] < epoch:
                            far_stamp[t] = epoch
                            far.append(t)
                    elif not in_pile[t]:
                        in_pile[t] = True
                        far.append(t)
            near = out
            max_near, max_far = max(max_near, len(near)), max(max_far, len(far))
        if not far:
            break
        pile = np.asarray(far, np.int64)
        dp = dist[pile]
        live = dp[dp >= upper]                            # k_sssp_min_far
        if len(live) == 0:
            break
        lower, upper, _ = sssp_next_bucket(live.min(), delta, upper)
        epoch += 1
        buckets += 1
        near = pile[dp < upper]                           # the split (its lower bound is 0)
        in_pile[near] = False
        near = near.tolist()
        far = pile[dp >= upper].tolist()
        max_near, max_far = max(max_near, len(near)), max(max_far, len(far))
    return Replay(dist, buckets, max_near, max_far)


if __name__ == "__main__":
    import sys
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    sys.path.insert(0, str(root))
    sys.path.insert(0, str(root / "tests"))
    import oracle
    import sssp_fixtures as fx
    for name in fx.REPLAYED:
        f = fx.FIXTURES[name]()
        off, tgt, w = oracle.csr_build(f.src, f.dst, f.n, oracle.OUTGOING, oracle.SORTED, f.w)
        for legacy in (True, False):
            r = replay(off, tgt, w, f.start, f.delta, legacy_carry=legacy)
            print(f"{name:>16} n {f.n:>7} m {len(f.src):>7} delta {f.delta:<8.3g} legacy {legacy!s:>5}: "
                  f"buckets {r.buckets:>6} near {r.max_near:>6} far {r.max_far:>6} (2n + 1024 = {2 * f.n + 1024})")
