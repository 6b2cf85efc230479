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

`landing=Landing(...)` replays the one-shot call gb_sssp_csr_u32, whose rows land chunk by chunk: the chunks of
tc_split (chunk_rows below) go out from the start's chunk on, wrapping round, and the available rows are one
cyclic interval from the start's chunk.  A near entry whose row is not available is parked (once per vertex)
instead of relaxed; after each pass the landed bound is raised by the schedule and the parked vertices now
covered go to the near queue (k_sssp_unpark); when only parked vertices are left one more chunk lands.  The
schedule is the call's GB_SSSP_FEED_STEP: `step=p` lands the j-th chunk of the order after j * p passes, and
`step=None` lands nothing but the start's chunk until the loop has to wait.  From the first park on the stale
filter is off (lower = 0); `stale_filter=True` keeps it, the rule that gives wrong distances once a parked
vertex relaxed late improves a vertex below the current bucket.
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
    parked: int = 0                      # with a landing schedule: distinct vertices parked
    passes_before_last_landed: int = 0


@dataclass
class Landing:
    rows: list                           # chunk row bounds [0, ..., n] (chunk_rows)
    step: int | None = None              # None: the start's chunk only, until the loop waits
    stale_filter: bool = False           # keep `du < lower` after a park (wrong)


def chunk_rows(off, c):
    """tc_split (csr_split.h) restated: greedy row-aligned chunks of at most c entries; a longer row stands alone
    with the empty rows next to it"""
    off = [int(x) for x in off]
    n, rows, r = len(off) - 1, [0], 0
    while r < n:
        p = max(int(np.searchsorted(off, off[r] + c, side="right")) - 1, r)   # the last boundary within budget
        if p < n and off[p] == off[r]:          # a hub
            p += 1
            while p < n and off[p + 1] == off[p]:
                p += 1
        rows.append(p)
        r = p
    return rows


def start_chunk(rows, start: int) -> int:
    """the chunk that holds row `start`, sent first (sssp_send_order)"""
    return int(np.searchsorted(rows, start, side="right")) - 1


def replay(off, tgt, w, start: int, delta: float, legacy_carry: bool = False, landing: Landing | None = None) -> Replay:
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
    if landing is not None:
        rows = landing.rows
        K = len(rows) - 1
        ks = start_chunk(rows, start)
        first = rows[ks]
    avail = 1                                             # chunks of the send order available
    parked, parked_flag, any_parked = [], np.zeros(n, bool), False
    total_parked = before_last = 0

    def present(u):
        if landing is None or avail == K:
            return True
        stop = rows[(ks + avail) % K]
        span = stop - first if stop > first else stop + n - first
        return (u - first if u >= first else u + n - first) < span

    def unpark():
        nonlocal parked, near
        keep = []
        for u in parked:
            if present(u):
                parked_flag[u] = False
                if near_stamp[u] < pass_:
                    near_stamp[u] = pass_
                    near.append(u)
            else:
                keep.append(u)
        parked = keep

    while True:
        while near:                                       # drain the near queue of this bucket
            pass_ += 1
            if landing is not None and avail < K:
                before_last += 1
            filt = lower if landing is None or landing.stale_filter or not any_parked else F32(0.0)
            out = []
            for u in near:
                du = dist[u]
                if du < filt:                             # stale: settled in an earlier bucket
                    continue
                if not present(u):                        # k_sssp_relax<true>: park once
                    if not parked_flag[u]:
                        parked_flag[u] = True
                        parked.append(u)
                        total_parked += 1
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
            if landing is not None:
                any_parked = any_parked or bool(parked)
                if landing.step is not None and avail < min(K, pass_ // landing.step + 1):
                    avail = min(K, pass_ // landing.step + 1)
                    unpark()
            max_near, max_far = max(max_near, len(near)), max(max_far, len(far))
        if far:
            pile = np.asarray(far, np.int64)
            dp = dist[pile]
            live = dp[dp >= upper]                        # k_sssp_min_far
            if len(live):
                lower, upper, _ = sssp_next_bucket(live.min(), delta, upper)
                epoch += 1
                buckets += 1
                near = pile[dp < upper]                   # the split (its lower bound is 0)
                in_pile[near] = False
                near = near.tolist()
                far = pile[dp >= upper].tolist()
                max_near, max_far = max(max_near, len(near)), max(max_far, len(far))
                continue
            far = []                                      # everything left is stale
        if landing is None or not parked:
            break
        avail += 1                                        # only parked vertices are left: wait for a chunk
        unpark()
        max_near = max(max_near, len(near))
    return Replay(dist, buckets, max_near, max_far, total_parked, before_last)


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
