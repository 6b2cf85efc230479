"""layout_model.py — numpy restatement of the PageRank layout build's edge classification and fill
(pagerank.cu: cb_classify_row / k_cb_count[_rows] -> k_cb_groups + scan -> k_cb_fill, and the cyclic deal).

There is no GPU in the build container; this model pins down the CONTRACT of the two passes so that it
can be checked on the CPU: one 8-byte record per edge, positions in CSR order, every (row, block) pair of
the staircase keeps at least one 4-id group, the remainder of a row fills its SELL lane in CSR order, and
the result does not depend on the order in which rows are classified (the streamed upload classifies them
in original-id chunks, the resident path in internal order).
Run: python tools/layout_model.py   (also exercised by tests/test_layout_model.py)."""
from __future__ import annotations

import numpy as np

CB_G = 4
REC_SEG = 0x80000000
NONE = 0xFFFFFFFF
CB_BLOCK_DEFAULT = 49152
CB_BLOCK_MAX = 56 * 1024
CB_TAU_DEFAULT = 1.5
CB_MAX_BLOCKS = 8192
CB_MEGA_DEG = 32768
CB_MEGA_JBITS = 14
SELL_FEW = 4
FIN_CTA_BLOCKS = 64
PR_FIN_WARPS = 8          # PR_FIN_THREADS / 32
PR_SELL_WARPS = 16        # PR_SELL_THREADS / 32
H100_SMS = 132


def deal_global(l, P, p):
    return (((l >> 5) * P + p) << 5) | (l & 31)


def deal_local(g, P, p):
    """inverse of deal_global; None when global row g is not rank p's"""
    sl = g >> 5
    if sl % P != p:
        return None
    return ((sl // P) << 5) | (g & 31)


def deal_count(R, P, p):
    F, rem = R >> 5, R & 31
    full = (F - p + P - 1) // P if F > p else 0
    c = full * 32
    if rem and F % P == p:
        c += rem
    return c


def clamp_block(B):
    """GB_PR_BLOCK as build_pr_plan applies it: a multiple of 1024 in [1024, CB_BLOCK_MAX]"""
    return min(max(B & ~1023, 1024), CB_BLOCK_MAX)


def make_plan(in_off, in_tgt, out_deg, B, tau, P=1, p=0, mega=CB_MEGA_DEG):
    """Renumbering + staircase, like steps 1-3 of build_pr_plan (host side, no edge data needed).
    B is used as given (see clamp_block); `mega` is GB_PR_MEGA, the in-degree above which a row takes the
    sort path of the layout build."""
    n = len(in_off) - 1
    indeg = np.diff(in_off).astype(np.int64)
    # in-degree descending, then out-degree descending, then id
    order = np.lexsort((np.arange(n), -out_deg.astype(np.int64), -indeg))
    new_id = np.empty(n, np.int64)
    new_id[order] = np.arange(n)
    n_active = int((indeg > 0).sum())
    m = int(in_off[-1])
    nblk = (n + B - 1) // B
    outdeg_int = out_deg[order]
    blk_edges = np.array([int(outdeg_int[b * B:(b + 1) * B].sum()) for b in range(nblk)])
    indeg_int = indeg[order]
    rows_ge = []
    for b in range(nblk):
        if blk_edges[b] == 0:
            rows_ge.append(0)
            continue
        dmin = max(1, int(np.ceil(tau * m / blk_edges[b])))
        rows_ge.append(int((indeg_int[:n_active] >= dmin).sum()))
    hot = [b for b in range(nblk) if deal_count(rows_ge[b], P, p) > 0]
    hot.sort(key=lambda b: (-rows_ge[b], b))
    hot = hot[:CB_MAX_BLOCKS]
    hot_of_blk = np.full(nblk, -1, np.int64)
    nrows, poff, S = [], [0], 0
    for j, b in enumerate(hot):
        hot_of_blk[b] = j
        nrows.append(deal_count(rows_ge[b], P, p))
        S += nrows[-1]
        poff.append(S)
    n_loc = deal_count(n_active, P, p)
    n_cb = nrows[0] if nrows else 0
    # rows on the sort path: in-degree > mega, a prefix of the rows with segments (the 32-bit prefix trim of
    # the sort index needs graphs beyond any test)
    n_mega = deal_count(int((indeg_int[:n_active] >= mega + 1).sum()), P, p) if m else 0
    n_mega = min(n_mega, n_cb, (1 << (32 - CB_MEGA_JBITS)) - 1)
    if len(hot) >= (1 << CB_MEGA_JBITS) - 1:
        n_mega = 0
    return dict(n=n, order=order, new_id=new_id, n_active=n_active, n_loc=n_loc, blk=np.array(hot, np.int64),
                hot_of_blk=hot_of_blk, nrows=np.array(nrows, np.int64), poff=np.array(poff, np.int64), S=S,
                n_cb=n_cb, KB=len(hot), n_mega=n_mega, last_hot_block=max(hot) if hot else NONE, nblk=nblk,
                B=B, P=P, p=p)


def launch_shape(plan, sms=H100_SMS, fin_u=0, fin_split=0, dual=False):
    """Step 8 of build_pr_plan: the SELL grid (one warp per 32-row slice, no launch for a shard without
    rows) and which rows k_pr_finish completes and how (fin_u, grid, role split).
    fin_u / fin_split are GB_PR_FIN_U / GB_PR_FIN_SPLIT; dual is GB_PR_DUAL=1 (taken when there are hot
    blocks and active rows)."""
    KB, n_cb, nr = plan["KB"], plan["n_cb"], plan["nrows"]
    dual = bool(dual) and KB > 0 and plan["n_loc"] > 0
    ceil32 = lambda x: (int(x) + 31) // 32 * 32
    num_slices = (plan["n_loc"] + 31) // 32
    grid_sell = min((num_slices + PR_SELL_WARPS - 1) // PR_SELL_WARPS, sms * 2)
    n_fin = n_cb if dual else (min(n_cb, ceil32(nr[SELL_FEW])) if KB > SELL_FEW else 0)
    n_fin_warp = min(n_fin, ceil32(nr[FIN_CTA_BLOCKS])) if KB > FIN_CTA_BLOCKS else 0
    warps2 = n_fin_warp // 32 * PR_FIN_WARPS + (n_fin - n_fin_warp + 63) // 64
    warps4 = n_fin_warp // 32 * PR_FIN_WARPS + (n_fin - n_fin_warp + 127) // 128
    u = 2 if (warps2 + PR_FIN_WARPS - 1) // PR_FIN_WARPS <= sms * 8 else 4
    if fin_u in (2, 4):
        u = fin_u
    want_fin = ((warps2 if u == 2 else warps4) + PR_FIN_WARPS - 1) // PR_FIN_WARPS
    grid_fin = max(1, min(want_fin, sms * 8))
    pays = want_fin <= sms * 8 and KB > 4 * FIN_CTA_BLOCKS
    structural = n_fin_warp > 0 and n_fin > n_fin_warp and grid_fin > n_fin_warp // 32
    split = structural and (fin_split == 1 or (fin_split == 0 and pays))
    return dict(hot_blocks=KB, n_cb=n_cb, n_fin=n_fin, n_fin_warp=n_fin_warp, fin_u=u, grid_sell=grid_sell,
                grid_fin=grid_fin,
                fin_hub_ctas=n_fin_warp // 32 if split else 0, grid_capped=want_fin > sms * 8,
                n_mega=plan["n_mega"], dual=int(dual), last_hot_block=plan["last_hot_block"])


def layout_counts(plan, in_off, in_tgt):
    """Staircase pairs, 4-id groups and edges served from column blocks (k_cb_count + k_cb_groups),
    vectorised: the statistics gb_pr_shard_stats reports as segments / groups / block_edges."""
    n, B, P, p = plan["n"], plan["B"], plan["P"], plan["p"]
    in_off = np.asarray(in_off, np.int64)
    row = np.repeat(np.arange(n, dtype=np.int64), np.diff(in_off))   # original row of every in-edge
    g = plan["new_id"][row]
    sl = g >> 5
    l = ((sl // P) << 5) | (g & 31)
    j = plan["hot_of_blk"][plan["new_id"][np.asarray(in_tgt, np.int64)] // B]
    nrows = plan["nrows"] if len(plan["nrows"]) else np.zeros(1, np.int64)
    seg = (sl % P == p) & (g < plan["n_active"]) & (j >= 0)
    seg &= l < nrows[np.maximum(j, 0)]
    cnt = np.bincount(plan["poff"][j[seg]] + l[seg], minlength=plan["S"])[:plan["S"]]
    groups = int(np.where(cnt > 0, (cnt + CB_G - 1) // CB_G, 1).sum())
    return dict(segments=int(plan["S"]), groups=groups, block_edges=int(seg.sum()))


def classify_row(plan, l, tgt_row, cnt, rec_out):
    """cb_classify_row: records of one local row, 32 edges (one batch) at a time in CSR order."""
    B, rem = plan["B"], 0
    for i in range(0, len(tgt_row), 32):
        batch = tgt_row[i:i + 32]
        src = plan["new_id"][batch]
        j = plan["hot_of_blk"][src // B]
        j = np.where((j >= 0) & (l < plan["nrows"][np.maximum(j, 0)]), j, -1)
        for lane in range(len(batch)):
            if j[lane] >= 0:
                e = plan["poff"][j[lane]] + l
                pos = cnt[e]              # the per-pair counter: batches in order, lanes in order
                cnt[e] += 1
                local = src[lane] - plan["blk"][j[lane]] * B
                rec_out[i + lane] = (int(local) | (int(j[lane]) << 16), REC_SEG | int(pos))
            else:
                rec_out[i + lane] = (int(src[lane]), rem)
                rem += 1
    return rem


def build(plan, in_off, in_tgt, row_order):
    """Classification in the given order of ORIGINAL row ids, then the scans and the fill."""
    cnt = np.zeros(plan["S"] + 1, np.int64)
    lens = np.zeros(max(plan["n_loc"], 1), np.int64)
    rec = [None] * int(in_off[-1])
    for v in row_order:
        g = int(plan["new_id"][v])
        if g >= plan["n_active"]:
            continue
        l = deal_local(g, plan["P"], plan["p"])
        if l is None:
            continue
        b0, b1 = int(in_off[v]), int(in_off[v + 1])
        if l < plan["n_cb"]:
            out = [None] * (b1 - b0)
            lens[l] = classify_row(plan, l, in_tgt[b0:b1], cnt, out)
            rec[b0:b1] = out
        else:
            lens[l] = b1 - b0
    groups = np.where(cnt[:plan["S"]] > 0, (cnt[:plan["S"]] + CB_G - 1) // CB_G, 1)   # k_cb_groups
    goff = np.concatenate([[0], np.cumsum(groups)])
    NG = int(goff[-1])
    ids = np.full(NG * CB_G, plan["B"], np.int64)                                       # pad id = B
    sell = {l: np.full(int(lens[l]), NONE, np.int64) for l in range(plan["n_loc"])}
    for l in range(plan["n_loc"]):                                                      # k_cb_fill / k_sell_fill_tail
        v = int(plan["order"][deal_global(l, plan["P"], plan["p"])])
        b0, b1 = int(in_off[v]), int(in_off[v + 1])
        if l < plan["n_cb"]:
            for x, y in rec[b0:b1]:
                if y & REC_SEG:
                    j = x >> 16
                    ids[goff[plan["poff"][j] + l] * CB_G + (y & ~REC_SEG)] = x & 0xFFFF
                else:
                    sell[l][y] = x
        else:
            sell[l][:] = plan["new_id"][in_tgt[b0:b1]]
    return dict(cnt=cnt[:plan["S"]], goff=goff, ids=ids, sell=sell, lens=lens)


def direct(plan, in_off, in_tgt):
    """The layout stated directly: per local row, edges grouped by hot block in CSR order."""
    seg, rest = {}, {}
    for l in range(plan["n_loc"]):
        v = int(plan["order"][deal_global(l, plan["P"], plan["p"])])
        src = plan["new_id"][in_tgt[int(in_off[v]):int(in_off[v + 1])]]
        r = []
        for s in src:
            j = plan["hot_of_blk"][s // plan["B"]]
            if j >= 0 and l < plan["nrows"][j]:
                seg.setdefault((int(j), l), []).append(int(s - plan["blk"][j] * plan["B"]))
            else:
                r.append(int(s))
        rest[l] = r
    return seg, rest


def check(plan, got, in_off, in_tgt):
    seg, rest = direct(plan, in_off, in_tgt)
    for j in range(len(plan["nrows"])):
        for l in range(int(plan["nrows"][j])):
            e = int(plan["poff"][j]) + l
            want = seg.get((j, l), [])
            g0, g1 = int(got["goff"][e]), int(got["goff"][e + 1])
            assert g1 - g0 == max(1, (len(want) + CB_G - 1) // CB_G), "a pair keeps ceil(edges / 4) groups, at least one"
            have = got["ids"][g0 * CB_G:g1 * CB_G]
            assert have[:len(want)].tolist() == want, "segment ids in CSR order"
            assert (have[len(want):] == plan["B"]).all(), "padding = the zero slot"
    for l in range(plan["n_loc"]):
        assert got["sell"][l].tolist() == rest[l], "SELL lane = the row's other sources, CSR order"
    assert sum(len(v) for v in seg.values()) + sum(len(v) for v in rest.values()) == sum(
        int(in_off[int(plan["order"][deal_global(l, plan["P"], plan["p"])]) + 1]) -
        int(in_off[int(plan["order"][deal_global(l, plan["P"], plan["p"])])]) for l in range(plan["n_loc"]))


def random_graph(rng, n, m, skew=1.5):
    w = (np.arange(1, n + 1) ** -skew)
    w /= w.sum()
    src = rng.choice(n, m, p=w)
    dst = rng.choice(n, m, p=rng.permutation(w))
    order = np.lexsort((src, dst))
    dst, src = dst[order], src[order]
    in_off = np.concatenate([[0], np.cumsum(np.bincount(dst, minlength=n))]).astype(np.int64)
    out_deg = np.bincount(src, minlength=n).astype(np.int64)
    return in_off, src.astype(np.int64), out_deg


def main():
    rng = np.random.default_rng(3)
    for it in range(6):
        n, m = int(rng.integers(200, 600)), int(rng.integers(2000, 8000))
        in_off, in_tgt, out_deg = random_graph(rng, n, m)
        for P in (1, 3):
            for p in range(P):
                plan = make_plan(in_off, in_tgt, out_deg, B=64, tau=1.5, P=P, p=p)
                a = build(plan, in_off, in_tgt, np.arange(n))                 # streamed upload: original order
                b = build(plan, in_off, in_tgt, plan["order"])                # resident path: internal order
                check(plan, a, in_off, in_tgt)
                assert (a["ids"] == b["ids"]).all() and (a["goff"] == b["goff"]).all()
    print("layout model ok")


if __name__ == "__main__":
    main()
