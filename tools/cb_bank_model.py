"""cb_bank_model.py — CPU count of the shared-memory bank conflicts of k_pr_cb's gathers, before and
after the bank-aware order of the ids inside each group (pr_layout.cu: k_cb_bank_order).

A warp step of k_pr_cb covers a WINDOW of 32 G groups (G = cb_step_groups: 4 in chunks of at least
CB_WIDE_MIN groups, else 2): lane L reads groups G L .. G L + G - 1 and then issues 4 shared-memory reads
xs[id] per group, one per SLOT.  The reads of group G L + i of all lanes form the SET i of the window.  One read instruction
takes as many wavefronts as the most crowded bank holds distinct words (bank = id & 31); all lanes that
read the padding id B hit the same word, which is a broadcast.  The 4 ids of a group belong to one
(row, block) pair, so their order is free: k_cb_bank_order lets lane 0, 1, ... in turn put the 4 ids of
its group of a set into the 4 slots (24 possible orders) so that each lands where its bank is least loaded
by the lanes before it.  A set keeps its old order unless the new one lowers its conflict bound (sum over
the slots of the largest per-bank count of non-pad ids), so no set gets worse by that bound.

Windows follow the kernel's steps: chunk c covers groups [g0, g1) and steps from g0 & ~1 by 32 G; a group
of a step outside [g0, g1) is read as padding and is ordered by the chunk that owns it.

Run: python tools/cb_bank_model.py [scale ...]   (default 20 22; tests/test_cb_bank_order.py checks it)."""
from __future__ import annotations

import itertools
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parent))
import cb_model  # noqa: E402
import layout_model as lm  # noqa: E402

PERMS = np.array(list(itertools.permutations(range(4))), np.int64)   # [24, slot] -> id index; identity first
CB_TASK_CHUNKS = 32


def build_streams(in_off, in_tgt, out_deg, B=lm.CB_BLOCK_DEFAULT, tau=lm.CB_TAU_DEFAULT):
    """The column-block streams of the layout build (one GPU), vectorised: the same ids, groups and pad
    positions as layout_model.build (k_cb_count + k_cb_groups + scan + k_cb_fill)."""
    plan = lm.make_plan(in_off, in_tgt, out_deg, B, tau)
    in_off = np.asarray(in_off, np.int64)
    n = len(in_off) - 1
    row = np.repeat(np.arange(n, dtype=np.int64), np.diff(in_off))   # original row of every in-edge (CSR order)
    l = plan["new_id"][row]
    src = plan["new_id"][np.asarray(in_tgt, np.int64)]
    j = plan["hot_of_blk"][src // B]
    nrows = plan["nrows"] if len(plan["nrows"]) else np.zeros(1, np.int64)
    seg = (l < plan["n_active"]) & (j >= 0)
    seg &= l < nrows[np.maximum(j, 0)]
    e = plan["poff"][j[seg]] + l[seg]                                  # staircase pair of every segment id
    local = src[seg] - plan["blk"][j[seg]] * B
    order = np.argsort(e, kind="stable")                               # CSR order inside a pair
    e_s = e[order]
    first = np.searchsorted(e_s, e_s, side="left")
    pos = np.arange(len(e_s)) - first
    cnt = np.bincount(e, minlength=plan["S"])[:plan["S"]]
    groups = np.where(cnt > 0, (cnt + lm.CB_G - 1) // lm.CB_G, 1)
    goff = np.concatenate([[0], np.cumsum(groups)]).astype(np.int64)
    NG = int(goff[-1])
    ids = np.full(NG * lm.CB_G, B, np.int64)
    ids[goff[e_s] * lm.CB_G + pos] = local[order]
    return plan, goff, ids.reshape(NG, lm.CB_G)


def chunk_table(plan, goff, sms=lm.H100_SMS, T=CB_TASK_CHUNKS):
    """The layout_chunks stage of build_pr_plan: per-block chunk sizes, then k_cb_chunks (cb_model.cb_cut).
    Returns (g0, g1, a segment is cut at either end) per chunk."""
    NG = int(goff[-1])
    gbeg = goff[plan["poff"]]
    C = min(max(NG // (sms * 8 * T), 16384 // T), 65536 // T)
    C = max(32, (C + 31) // 32 * 32)
    chunks = []
    for j in range(plan["KB"]):
        g0, g1, nr = int(gbeg[j]), int(gbeg[j + 1]), int(plan["nrows"][j])
        G = g1 - g0
        Cj = min(C, max(min(64, C), (G // 64 + 63) // 64 * 64))
        nc = (G + Cj - 1) // Cj
        goff_j = goff[plan["poff"][j]:plan["poff"][j] + nr]
        for k in range(nc):
            a = cb_model.cb_cut(goff_j, nr, g1, g0 + k * Cj, Cj)
            b = (g1, nr, False) if k + 1 == nc else cb_model.cb_cut(goff_j, nr, g1, g0 + (k + 1) * Cj, Cj)
            chunks.append((int(a[0]), int(b[0]), bool(a[2] or b[2])))
    return chunks


def windows(chunks):
    """(first group of the step, lowest and highest+1 group the step may read, groups per lane) for every
    kernel step"""
    out = []
    for g0, g1, *_ in chunks:
        G = cb_model.step_groups(g0, g1)
        for gs in range(g0 & ~1, g1, 32 * G):
            out.append((gs, g0, g1, G))
    return np.array(out, np.int64).reshape(-1, 4)


def gather_sets(ids, win, B):
    """[S, 32 lanes, 4] ids of every SET of a step (set i of a step with G groups per lane = group G L + i
    of every lane L; padding where the step reads padding) and the group index of each (or -1).  Sets come
    in window order, the G sets of a window one after another."""
    grps, gis, order = [], [], []
    for G in (2, 4):
        sel = np.nonzero(win[:, 3] == G)[0]
        w = win[sel]
        gs, g0, g1 = w[:, 0:1], w[:, 1:2], w[:, 2:3]
        g = gs + np.arange(32 * G)[None, :]
        valid = (g >= g0) & (g < g1)
        gi = np.where(valid, g, -1)
        grp = np.full(gi.shape + (4,), B, np.int64)
        grp[valid] = ids[gi[valid]]
        # position G L + i -> set i, lane L
        grps.append(grp.reshape(-1, 32, G, 4).transpose(0, 2, 1, 3).reshape(-1, 32, 4))
        gis.append(gi.reshape(-1, 32, G).transpose(0, 2, 1).reshape(-1, 32))
        order.append(np.repeat(sel * 4, G) + np.tile(np.arange(G), len(sel)))
    o = np.argsort(np.concatenate(order), kind="stable")
    return np.concatenate(grps)[o], np.concatenate(gis)[o]


def conflict_bound(grp, B):
    """[..., 32, 4] -> sum over the 4 slots of max(1, largest per-bank count of non-pad ids): the order's
    cost as k_cb_bank_order counts it (an upper bound of the wavefronts of the real ids)."""
    real = grp != B
    bank = np.where(real, grp & 31, 32)
    flat = bank.reshape(-1, 32, 4)
    tot = np.zeros(flat.shape[0], np.int64)
    for s in range(4):
        h = np.zeros((flat.shape[0], 33), np.int64)
        np.add.at(h, (np.arange(flat.shape[0])[:, None], flat[:, :, s]), 1)
        tot += np.maximum(h[:, :32].max(axis=1), 1)
    return tot.reshape(grp.shape[:-2])


def wavefronts(grp, active):
    """[..., 32, 4] ids and [..., 32] active lanes -> wavefronts of each of the 4 read instructions:
    per bank, the number of distinct words read (the padding id is one word like any other)."""
    shp = grp.shape[:-2]
    flat = grp.reshape(-1, 32, 4)
    act = np.broadcast_to(active[..., None], grp.shape).reshape(-1, 32, 4)
    out = np.zeros((flat.shape[0], 4), np.int64)
    for s in range(4):
        v = flat[:, :, s]
        a = act[:, :, s]
        key = np.where(a, v, -1)
        srt = np.sort(key, axis=1)
        new = np.ones_like(srt, bool)
        new[:, 1:] = srt[:, 1:] != srt[:, :-1]
        new &= srt >= 0
        h = np.zeros((flat.shape[0], 32), np.int64)
        rows = np.broadcast_to(np.arange(flat.shape[0])[:, None], srt.shape)
        np.add.at(h, (rows[new], srt[new] & 31), 1)
        out[:, s] = h.max(axis=1)
    return out.reshape(shp + (4,))


def bank_order(grp, B):
    """k_cb_bank_order on every set at once: grp [..., 32, 4] -> reordered copy."""
    shp = grp.shape
    flat = grp.reshape(-1, 32, 4)
    H = flat.shape[0]
    hist = np.zeros((H, 4, 33), np.int64)       # bin 32: padding (free, never counted)
    out = flat.copy()
    r = np.arange(H)
    for L in range(32):
        g = flat[:, L, :]
        bank = np.where(g != B, g & 31, 32)                       # [H, 4]
        # cost[h, s, k] = load of id k's bank in slot s so far
        cost = hist[r[:, None, None], np.arange(4)[None, :, None], bank[:, None, :]]
        cost[:, :, :][np.broadcast_to((bank == 32)[:, None, :], cost.shape)] = 0
        pc = cost[:, np.arange(4)[None, :], PERMS].sum(axis=2)     # [H, 24]
        best = pc.argmin(axis=1)                                   # first minimum: identity on ties
        sel = PERMS[best]                                          # [H, slot] -> id index
        newg = np.take_along_axis(g, sel, axis=1)
        out[:, L, :] = newg
        nb = np.take_along_axis(bank, sel, axis=1)
        for s in range(4):
            hist[r, s, nb[:, s]] += 1
    before = conflict_bound(flat, B)
    after = conflict_bound(out, B)
    keep = after >= before
    out[keep] = flat[keep]
    return out.reshape(shp)


def apply(ids, win, B):
    """Reorder the groups as the kernel does; returns the new ids and the sets before and after."""
    grp, gi = gather_sets(ids, win, B)
    new = bank_order(grp, B)
    m = gi >= 0
    out = ids.copy()
    out[gi[m]] = new[m]
    return out, grp, new, gi


def report(scale, seed=42):
    import oracle  # built by __graft_entry__.build()
    n = 1 << scale
    src, dst = oracle.rmat_edges(scale, seed)
    out_off, _ = oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED)
    in_off, in_tgt = oracle.csr_build(src, dst, n, oracle.INCOMING, oracle.SORTED)
    plan, goff, ids = build_streams(in_off, in_tgt, np.diff(out_off.astype(np.int64)))
    B = plan["B"]
    win = windows(chunk_table(plan, goff))
    new_ids, grp, new, gi = apply(ids, win, B)
    active = np.ones(gi.shape, bool)   # every lane issues all 8 reads (padding included)
    wf0, wf1 = wavefronts(grp, active), wavefronts(new, active)
    reads = wf0.size
    print(f"RMAT-{scale}: {ids.shape[0]} groups, {len(win)} warp steps, {reads} read instructions")
    print(f"  wavefronts per read: before {wf0.sum() / reads:.3f}  after {wf1.sum() / reads:.3f}"
          f"  ({100.0 * (1 - wf1.sum() / wf0.sum()):.1f} % fewer)")
    print(f"  conflict bound per read: before {conflict_bound(grp, B).sum() / reads:.3f}"
          f"  after {conflict_bound(new, B).sum() / reads:.3f}")
    return wf0.sum() / reads, wf1.sum() / reads


def main():
    scales = [int(a) for a in sys.argv[1:]] or [20, 22]
    sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
    for s in scales:
        report(s)


if __name__ == "__main__":
    main()
