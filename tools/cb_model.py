"""cb_model.py — lane-level numpy model of the column-block kernel's chunk logic (pr_layout.cu:
cb_cut / k_cb_chunks; pagerank.cu: cb_walk / cb_fix_segment).

There is no GPU in the build container, so the trickiest index logic (chunk cuts inside long
segments, start-bit row counting, the carried run, side buffers and their fixed-order fixup) is
restated here lane by lane and checked against a direct per-segment sum on random segment lengths.
Run: python tools/cb_model.py   (also exercised by tests/test_cb_model.py)."""
from __future__ import annotations

import numpy as np

HEAD, TAIL, INTERIOR = 1, 2, 4


def cb_cut(goff_j, nr, gend, q, C):
    if q >= gend:
        return gend, nr, False
    lo, hi = 0, nr
    while hi - lo > 1:
        mid = lo + (hi - lo) // 2
        if goff_j[mid] <= q:
            lo = mid
        else:
            hi = mid
    s0 = goff_j[lo]
    s1 = goff_j[lo + 1] if lo + 1 < nr else gend
    if s0 == q:
        return q, lo, False
    if s1 - s0 > C:
        return q, lo, True
    return s1, lo + 1, False


def build_chunks(goff, poff, nrows, gbeg, C):
    """k_cb_chunks on the host: returns chunks [(g0, g1, row_before, j, flags)], tail_slot, fix_list."""
    chunks, tail_slot, fix = [], [], []
    for j in range(len(nrows)):
        g0, g1, nr = gbeg[j], gbeg[j + 1], nrows[j]
        goff_j = goff[poff[j]:poff[j] + nr]
        nc = (g1 - g0 + C - 1) // C
        for k in range(nc):
            a = cb_cut(goff_j, nr, g1, g0 + k * C, C)
            b = (g1, nr, False) if k + 1 == nc else cb_cut(goff_j, nr, g1, g0 + (k + 1) * C, C)
            fl = 0
            if a[2]:
                fl |= HEAD
            if b[2]:
                fl |= TAIL
            last_row = b[1] if b[2] else b[1] - 1
            if a[2] and last_row == a[1]:
                fl |= INTERIOR
            row_before = a[1] if a[2] else a[1] - 1
            c = len(chunks)
            chunks.append((a[0], b[0], row_before, j, fl))
            tail_slot.append(poff[j] + b[1] if b[2] else -1)
            if b[2] and not (fl & INTERIOR):
                fix.append(c)
    return chunks, tail_slot, fix


WIDE_MIN = 128   # CB_WIDE_MIN


def step_groups(g0, g1):
    """cb_step_groups: groups per lane in the steps of chunk [g0, g1), 4 from WIDE_MIN groups on, else 2"""
    return 4 if g1 - g0 >= WIDE_MIN else 2


def seg_scan(T, F, carry):
    """the segmented inclusive warp scan of cb_walk: T = each lane's share of the run open at its end
    (f32), F = the lane holds a segment start.  Returns (inclD, XD): the run open at the end of each lane
    and at the end of the lane before it, in f64 with the carried run added."""
    lanes = np.arange(32)
    seg_start = np.full(32, -1)
    cur = -1
    for l in range(32):
        if F[l]:
            cur = l
        seg_start[l] = cur
    lo = np.maximum(seg_start, 0)
    incl = T.astype(np.float32).copy()
    d = 1
    while d < 32:
        t = np.zeros(32, np.float32)
        t[d:] = incl[:-d]
        incl = np.where((lanes - d) >= lo, (incl + t).astype(np.float32), incl)
        d <<= 1
    inclD = incl.astype(np.float64) + np.where(seg_start < 0, carry, 0.0)
    XD = np.empty(32)
    XD[0] = carry
    XD[1:] = inclD[:-1]
    return inclD, XD


def run_chunk(c, chunks, vals, bits, poff, partial, side):
    """cb_walk: vals[g] = f32 sum of group g's four gathers; bits[g] = group g starts a segment.
    A step covers 32 G groups (G = step_groups) from g0 & ~1; lane L owns groups G L .. G L + G - 1 of the
    window, adds the runs inside the lane in f32, and takes part in ONE segmented scan per step.
    Returns G (None for an empty chunk)."""
    g0, g1, row_before, j, fl = chunks[c]
    if g0 >= g1:
        return None
    G = step_groups(g0, g1)
    S = 32 * G
    head_cont, tail_cont = bool(fl & HEAD), bool(fl & TAIL)
    in_head = head_cont
    carry = 0.0
    for gs in range(g0 & ~1, g1, S):
        pos = np.arange(S)
        valid = (gs + pos >= g0) & (gs + pos < g1)
        W = np.zeros(S, bool)
        W[valid] = bits[gs + pos[valid]]
        v = np.zeros(S, np.float32)
        v[valid] = vals[gs + pos[valid]]
        last = int(np.nonzero(valid)[0][-1])
        last_step = gs + S >= g1
        run_continues = tail_cont if last_step else (not bits[gs + S])
        F, V = W.reshape(32, G), v.reshape(32, G)
        r = np.zeros((32, G), np.float32)        # run sums inside the lane, restarted at each start
        for i in range(G):
            prev = r[:, i - 1] if i else np.zeros(32, np.float32)
            r[:, i] = np.where(F[:, i], V[:, i], (prev + V[:, i]).astype(np.float32))
        inclD, XD = seg_scan(r[:, G - 1], F.any(axis=1), carry)
        cum = np.cumsum(W)                 # starts at positions <= q
        for l in range(32):
            for i in range(G):
                q = G * l + i
                nxt = W[q + 1] if q + 1 < S else False
                if not (valid[q] and (q == last or nxt)):
                    continue
                if q == last and run_continues and not last_step:
                    continue
                if i == G - 1:
                    tot = inclD[l]
                else:
                    tot = float(r[l, i]) + (0.0 if F[l, :i + 1].any() else XD[l])
                if in_head and cum[q] == 0:
                    side[2 * c] = tot
                elif q == last and last_step and tail_cont:
                    side[2 * c + 1] = tot
                else:
                    partial[poff[j] + row_before + cum[q]] = np.float32(tot)
        carry = inclD[31] if (run_continues and not last_step) else 0.0
        if W.any():
            in_head = False
        row_before += int(W.sum())
    return G


def fixup(fix, chunks, tail_slot, side, partial):
    n = len(chunks)
    for c0 in fix:
        t = side[2 * c0 + 1]
        k = c0 + 1
        while True:
            fl = chunks[k][4] if k < n else 0
            t += side[2 * k]
            if not ((fl & INTERIOR) and (fl & TAIL)):
                break
            k += 1
        partial[tail_slot[c0]] = np.float32(t)


def simulate(nrows, groups_per_pair, C, rng, kinds=None):
    """nrows[j] non-increasing; groups_per_pair: list of arrays (>= 1 group each).  kinds: a set that
    receives (G, a segment is cut at either end) of every chunk that ran."""
    poff = np.concatenate([[0], np.cumsum(nrows)]).astype(np.int64)
    gpp = np.concatenate(groups_per_pair).astype(np.int64)
    goff = np.concatenate([[0], np.cumsum(gpp)]).astype(np.int64)
    NG = int(goff[-1])
    gbeg = goff[poff]
    bits = np.zeros(NG + 64, bool)
    bits[goff[:-1]] = True
    vals = rng.random(NG + 64).astype(np.float32)
    vals[NG:] = 0
    chunks, tail_slot, fix = build_chunks(goff, poff, nrows, gbeg, C)
    partial = np.full(int(poff[-1]), np.nan, np.float32)
    side = np.zeros(2 * len(chunks) + 2)
    for c in range(len(chunks)):
        G = run_chunk(c, chunks, vals, bits, poff, partial, side)
        if G and kinds is not None:
            kinds.add((G, bool(chunks[c][4] & (HEAD | TAIL))))
    fixup(fix, chunks, tail_slot, side, partial)
    want = np.array([vals[goff[e]:goff[e + 1]].astype(np.float64).sum() for e in range(len(gpp))])
    # coverage: every chunk boundary is consistent and every group belongs to exactly one chunk
    covered = np.zeros(NG, int)
    for (g0, g1, _, _, _) in chunks:
        covered[g0:g1] += 1
    assert (covered == 1).all(), "chunks do not tile the streams"
    assert not np.isnan(partial).any(), "a pair never got its partial"
    err = np.abs(partial - want) / np.maximum(want, 1e-30)
    return float(err.max()), len(chunks), len(fix)


def random_case(rng, kb, max_rows, long_frac, C):
    nrows = np.sort(rng.integers(1, max_rows + 1, kb))[::-1].copy()
    gpp = []
    for nr in nrows:
        g = rng.geometric(0.5, nr)
        big = rng.random(nr) < long_frac
        g[big] = rng.integers(C // 2, 6 * C, int(big.sum()))
        gpp.append(g)
    return nrows, gpp


def main():
    rng = np.random.default_rng(1)
    worst = 0.0
    for it in range(60):
        C = int(rng.choice([32, 64, 96, 256]))
        nrows, gpp = random_case(rng, int(rng.integers(1, 6)), int(rng.integers(1, 400)), float(rng.choice([0, 0.02, 0.2])), C)
        e, nc, nf = simulate(nrows, gpp, C, rng)
        worst = max(worst, e)
    print("cb model ok; worst relative error", worst)


if __name__ == "__main__":
    main()
