"""layout_model.py — numpy restatement of the PageRank layout build's edge classification and fill
(pr_layout.cu: cb_classify_row / k_cb_count[_rows] -> k_cb_groups + scan -> k_cb_fill, and the cyclic deal).

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
    """Renumbering + staircase, like the layout_order and layout_hot_blocks stages of build_pr_plan
    (pr_layout.cu; host side, no edge data needed).
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


def launch_shape(plan, sms=H100_SMS, fin_u=0, fin_split=0):
    """plan_sweep_shape (pagerank.cu), the last stage of build_pr_plan: the SELL grid (one warp per 32-row
    slice, no launch for a shard without rows) and which rows k_pr_finish completes and how (fin_u, grid,
    role split).  fin_u / fin_split are GB_PR_FIN_U / GB_PR_FIN_SPLIT."""
    KB, n_cb, nr = plan["KB"], plan["n_cb"], plan["nrows"]
    ceil32 = lambda x: (int(x) + 31) // 32 * 32
    num_slices = (plan["n_loc"] + 31) // 32
    grid_sell = min((num_slices + PR_SELL_WARPS - 1) // PR_SELL_WARPS, sms * 2)
    n_fin = min(n_cb, ceil32(nr[SELL_FEW])) if KB > SELL_FEW else 0
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
                n_mega=plan["n_mega"], dual=0, last_hot_block=plan["last_hot_block"])  # gb_pr_plan_shape.dual is 0


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
    """The layout_classify stage of build_pr_plan (pr_layout.cu) in the given order of ORIGINAL row ids,
    then the group scan and the layout_fill stage."""
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


# ---- virtual blocks (layout_vblocks in pr_layout.cu, PrVBlocks in pr_plan.cuh) ----------------------------------
VB_ALIGN = 32
VB_RUN_ALIGN = 8     # with sectors, runs of V start at multiples of 8 slots (32-byte sectors) and fill them
VB_WINDOW = 58048    # pr_vb_window on an H100: (227 KB opt-in - 128 B static) / 4 - the zero slot, to 32 slots
VB_BLK_SHIFT = 43
BIN_PAD = 0xFFFF
BIN_STEP = 256   # pass A positions per warp step: 8 groups of 32
BIN_CHUNK = 8    # pass A steps per chunk


def bin_id_index(pos):
    """where pass A stores the id of position pos: 32 k + L of a step at 8 L + k"""
    pos = np.asarray(pos, np.int64)
    return (pos & ~(BIN_STEP - 1)) | (pos & 31) << 3 | (pos >> 5 & 7)


def cold_lens(plan, in_off, in_tgt):
    """cold edges (those outside every segment: the SELL lane lengths) of every local row, vectorised"""
    n, B, P, p = plan["n"], plan["B"], plan["P"], plan["p"]
    in_off = np.asarray(in_off, np.int64)
    row = np.repeat(np.arange(n, dtype=np.int64), np.diff(in_off))
    g = plan["new_id"][row]
    sl = g >> 5
    l = ((sl // P) << 5) | (g & 31)
    j = plan["hot_of_blk"][plan["new_id"][np.asarray(in_tgt, np.int64)] // B]
    nrows = plan["nrows"] if len(plan["nrows"]) else np.zeros(1, np.int64)
    mine = (sl % P == p) & (g < plan["n_active"])
    seg = (j >= 0) & (l < nrows[np.maximum(j, 0)])
    return np.bincount(l[mine & ~seg], minlength=plan["n_loc"])[:plan["n_loc"]]


def vb_counts(plan, in_off, in_tgt):
    """gb_pr_shard_stats' vblock_parts / vblock_pairs / vblock_edges (all 0 when the graph keeps SELL), vectorised"""
    n, B, P, p = plan["n"], plan["B"], plan["P"], plan["p"]
    lens = cold_lens(plan, in_off, in_tgt)
    cut = vb_partitions(lens, B)
    if cut is None:
        return dict(vblock_parts=0, vblock_pairs=0, vblock_edges=0)
    in_off = np.asarray(in_off, np.int64)
    row = np.repeat(np.arange(n, dtype=np.int64), np.diff(in_off))
    g = plan["new_id"][row]
    sl = g >> 5
    l = ((sl // P) << 5) | (g & 31)
    s = plan["new_id"][np.asarray(in_tgt, np.int64)]
    j = plan["hot_of_blk"][s // B]
    nrows = plan["nrows"] if len(plan["nrows"]) else np.zeros(1, np.int64)
    cold = (sl % P == p) & (g < plan["n_active"]) & ~((j >= 0) & (l < nrows[np.maximum(j, 0)]))
    part = np.searchsorted(cut[0], l[cold], side="right") - 1
    pairs = np.unique((part << 32) | s[cold]).size
    return dict(vblock_parts=len(cut[1]), vblock_pairs=int(pairs), vblock_edges=int(cold.sum()))


def vb_partitions(lens, B):
    """the greedy cut of the local rows into partitions of at most B cold edges: (first rows + n_loc, longest
    segment of each partition in groups), or None when the graph keeps SELL (no cold edge, or a row with more
    than B of them)"""
    row0, mseg, acc, ms = [0], [], 0, 0
    for l, d in enumerate(int(x) for x in lens):
        if d > B:
            return None
        if acc + d > B and l > row0[-1]:
            row0.append(l)
            mseg.append(ms)
            acc, ms = 0, 0
        acc += d
        ms = max(ms, (d + CB_G - 1) // CB_G if d else 1)
    if not len(lens) or int(np.sum(lens)) == 0:
        return None
    mseg.append(ms)
    row0.append(len(lens))
    return np.array(row0, np.int64), np.array(mseg, np.int64)


def vblocks(plan, built, window=VB_WINDOW):
    """layout_vblocks from the SELL lanes of `built` (build()): partitions, the pairs and V's slots, pass B's
    segments (k_vb_place) and pass A's positions, run bits, first runs and run table (k_bin_place).  `window` is
    pass B's largest window (pr_vb_window; GB_PR_VB_WINDOW lowers it).  Every run (the pairs of one source block
    inside one partition) starts at a multiple of VB_RUN_ALIGN slots and is padded to one (sectors), unless a
    padded partition would exceed the window: then the whole graph keeps the packed slots and a window of B."""
    B, n_loc = plan["B"], plan["n_loc"]
    lens = np.asarray(built["lens"][:n_loc], np.int64)
    cut = vb_partitions(lens, B)
    if cut is None:
        return None
    row0, mseg = cut
    parts = len(mseg)
    rows = np.repeat(np.arange(n_loc, dtype=np.int64), lens)                  # cold edges by row, CSR order
    src = np.concatenate([built["sell"][l] for l in range(n_loc)]).astype(np.int64)
    part = np.searchsorted(row0, rows, side="right") - 1
    key = (part << 32) | src
    order = np.argsort(key, kind="stable")                                    # the radix sort of (partition, source)
    sk = key[order]
    start = np.r_[True, sk[1:] != sk[:-1]]
    rank = np.cumsum(start) - 1                                               # pair of every sorted edge
    NP = int(rank[-1]) + 1
    pfirst = np.array([rank[i] if i < len(sk) else NP for i in np.searchsorted(sk >> 32, np.arange(parts + 1))])
    psrc, ppart = sk[start] & 0xFFFFFFFF, sk[start] >> 32
    # sector slots (k_vb_run_flags .. k_vb_run_pos): a run starts where the partition or source / B changes
    vrun = np.r_[True, (ppart[1:] != ppart[:-1]) | (psrc[1:] // B != psrc[:-1] // B)]
    rfirst = np.flatnonzero(vrun)
    rlen = np.diff(np.r_[rfirst, NP])
    roff = np.concatenate([[0], np.cumsum((rlen + VB_RUN_ALIGN - 1) // VB_RUN_ALIGN * VB_RUN_ALIGN)])
    rid = np.cumsum(vrun) - 1
    gpos = np.r_[roff[rid] + np.arange(NP) - rfirst[rid], roff[-1]]
    gfirst = gpos[pfirst]
    sectors = bool((np.diff(gfirst) <= window).all()) and NP + (VB_RUN_ALIGN - 1) * len(rfirst) < 0x7FFFFFFF
    slot_of = gpos[:NP] if sectors else np.arange(NP)
    first = gfirst if sectors else pfirst
    win = window if sectors else B
    vbase = np.concatenate([[0], np.cumsum((np.diff(first) + VB_ALIGN - 1) // VB_ALIGN * VB_ALIGN)])
    # pass B: one segment per local row, V-local slot ids in CSR order, pad id = its window
    groups = np.where(lens > 0, (lens + CB_G - 1) // CB_G, 1)
    goffv = np.concatenate([[0], np.cumsum(groups)])
    coff = np.concatenate([[0], np.cumsum(lens)])
    ids = np.full(int(goffv[-1]) * CB_G, win, np.int64)
    e = order
    ids[goffv[rows[e]] * CB_G + (e - coff[rows[e]])] = slot_of[rank] - first[sk >> 32]
    # pass A: the pairs by (source block, partition, source), each block's share starting at a step
    pslot = vbase[ppart] + slot_of - first[ppart]
    akey = ((psrc // B) << VB_BLK_SHIFT) | (ppart << 16) | (psrc % B)
    ao = np.argsort(akey, kind="stable")
    akey, aslot = akey[ao], pslot[ao]
    blk = akey >> VB_BLK_SHIFT
    bcnt = np.bincount(blk, minlength=plan["nblk"])
    bsteps = (bcnt + BIN_STEP - 1) // BIN_STEP
    bpos = np.concatenate([[0], np.cumsum(bsteps * BIN_STEP)])
    bfirst = np.concatenate([[0], np.cumsum(bcnt)])
    pos = bpos[blk] + np.arange(NP) - bfirst[blk]
    npos = int(bpos[-1])
    bin_ids = np.full(npos, BIN_PAD, np.int64)
    bin_ids[bin_id_index(pos)] = akey & 0xFFFF
    rstart = np.r_[True, (akey[1:] >> 16) != (akey[:-1] >> 16)]
    bin_bits = np.zeros(npos // 32, np.int64)
    np.bitwise_or.at(bin_bits, pos[rstart] // 32, 1 << (pos[rstart] % 32))
    # the last run that starts at or before each group's first position
    bin_grun = np.searchsorted(pos[rstart], np.arange(0, npos, 32), side="right") - 1
    bin_runs = (aslot[rstart] - pos[rstart]) & 0xFFFFFFFF                     # first slot - first position
    pos_blk = np.repeat(np.arange(plan["nblk"]), np.diff(bpos))              # source block of every position
    s0 = bpos[:-1] // BIN_STEP
    bin_chunks = np.array([(t, min(t + BIN_CHUNK, s0[b] + bsteps[b])) for b in np.flatnonzero(bcnt)
                           for t in range(s0[b], s0[b] + bsteps[b], BIN_CHUNK)], np.int64).reshape(-1, 2)
    return dict(parts=parts, row0=row0, mseg=mseg, vbase=vbase, pairs=NP, edges=int(lens.sum()), lens=lens,
                goffv=goffv, ids=ids, bin_ids=bin_ids, bin_bits=bin_bits, bin_grun=bin_grun, bin_runs=bin_runs,
                bin_chunks=bin_chunks, pos_blk=pos_blk, bcnt=bcnt, run_pos=pos[rstart], pos=pos, aslot=aslot,
                run_of=np.cumsum(rstart) - 1, slots=int(vbase[-1]), sectors=sectors, window=win,
                vrun_slot=vbase[ppart[rfirst]] + roff[:-1] - gfirst[ppart[rfirst]] if sectors else None,
                vrun_len=rlen)


def vb_pass_a(plan, vb, fills=None):
    """pass A (bin_chunk in k_pr_cb<CB_FUSED>), chunk by chunk, step by step, lane by lane: the source of every slot
    of V it writes, how often it writes it, and the steps that take the run-window loop (more than 32 runs).  With
    sectors the lane of a run's last position also zeroes the run's pad slots (bin_fill_pad): each is counted in
    `writes` and marked -2 in V, and `fills` (a dict, when given) counts the fills by where the run ends: at a
    step's last position (step_end; chunk_end when that is also its chunk's), before pads (share_end), in a wide
    step (wide)."""
    B = plan["B"]
    V = np.full(int(vb["vbase"][-1]), -1, np.int64)
    writes = np.zeros(len(V), np.int64)
    wide = []
    bits_all = np.r_[vb["bin_bits"], 1, np.zeros(BIN_STEP // 32 - 1, np.int64)]   # the step after the last: a start
    gs = BIN_STEP // 32
    lanes = np.arange(32)
    upto = (2 << lanes) - 1                                                   # positions 0 .. lane of a group
    popc = lambda x: np.array([bin(int(v)).count("1") for v in np.atleast_1d(x)])
    for s0, s1 in vb["bin_chunks"]:
        for s in range(int(s0), int(s1)):
            bits = vb["bin_bits"][gs * s:gs * s + gs]
            r0 = int(vb["bin_grun"][gs * s])
            ids = vb["bin_ids"][s * BIN_STEP:(s + 1) * BIN_STEP].reshape(32, 8)  # lane L's 128-bit load
            runs = int(popc(bits).sum()) - int(bits[0] & 1)                   # run starts after the first position
            if runs >= 32:
                wide.append(s)
            before = -int(bits[0] & 1)
            for k in range(gs):
                r = r0 + before + popc(bits[k] & upto)                        # every lane's run
                before += int(popc(bits[k])[0])
                p = s * BIN_STEP + 32 * k + lanes
                slot = (p + vb["bin_runs"][r]) & 0xFFFFFFFF
                sid = ids[:, k]
                ok = sid != BIN_PAD
                V[slot[ok]] = vb["pos_blk"][p[ok]] * B + sid[ok]
                np.add.at(writes, slot[ok], 1)
                if not vb["sectors"]:
                    continue
                nvalid = int((ids != BIN_PAD).sum())
                nxt = bits_all[gs * s + k + 1]                                # bits[k + 1], or the next step's
                q = 32 * k + lanes
                nstart = np.where(lanes < 31, (int(bits[k]) >> np.minimum(lanes + 1, 31)) & 1, int(nxt) & 1)
                last = ok & ((nstart == 1) | ((q + 1 == nvalid) & (nvalid < BIN_STEP)))
                for L in np.flatnonzero(last):
                    e = int(slot[L]) + 1
                    pad = np.arange(e, (e + VB_RUN_ALIGN - 1) // VB_RUN_ALIGN * VB_RUN_ALIGN)
                    V[pad] = -2
                    np.add.at(writes, pad, 1)
                    if fills is not None:
                        end = q[L] == BIN_STEP - 1
                        key = "share_end" if nstart[L] == 0 else "chunk_end" if end and s + 1 == s1 else \
                            "step_end" if end else "inside"
                        fills[key] = fills.get(key, 0) + 1
                        if runs >= 32:
                            fills["wide"] = fills.get("wide", 0) + 1
    return V, writes, wide


def vb_pass_a_cases(vb):
    """what a fixture's pass A layout reaches: steps with more than 32 runs, block shares shorter than a step,
    runs that cross a step boundary and a chunk boundary, and pad positions"""
    # a run's positions: from its first one to the next run's first or to its block's last pair
    bcnt = vb["bcnt"][vb["bcnt"] > 0]
    share = (bcnt + BIN_STEP - 1) // BIN_STEP * BIN_STEP
    share_end = np.cumsum(share) - share + bcnt                               # one past each block's last pair
    first = vb["run_pos"]
    nxt = np.r_[first[1:], np.iinfo(np.int64).max]
    last = np.minimum(nxt, share_end[np.searchsorted(share_end, first, side="right")]) - 1
    chunk_start = vb["bin_chunks"][:, 0] * BIN_STEP
    cross_chunk = np.searchsorted(chunk_start, last, side="right") > np.searchsorted(chunk_start, first, side="right")
    return dict(short_shares=int((bcnt < BIN_STEP).sum()),
                step_runs=int((first // BIN_STEP != last // BIN_STEP).sum()),
                chunk_runs=int(cross_chunk.sum()),
                pads=int((vb["bin_ids"] == BIN_PAD).sum()))


def check_vblocks(plan, vb, built):
    """the contract of the two passes: pass A writes every slot of V exactly once (and nothing between the
    virtual blocks), every cold edge appears exactly once in pass B, and every pass B id resolves to the slot
    of its edge's source; position + delta is every pair's slot.  Packed: a virtual block's slots are a prefix of
    at most B.  Sectors: every run starts at a multiple of VB_RUN_ALIGN slots, its pad slots up to the next one
    are zeroed (so every sector a run touches is written whole), and no virtual block exceeds the window."""
    B = plan["B"]
    V, writes, _ = vb_pass_a(plan, vb)
    W = vb["window"]
    slot = (vb["pos"] + vb["bin_runs"][vb["run_of"]]) % (1 << 32)
    assert (slot == vb["aslot"]).all(), "position + delta = the pair's slot"
    if vb["sectors"]:
        rs, rl = vb["vrun_slot"], vb["vrun_len"]
        assert (rs % VB_RUN_ALIGN == 0).all(), "runs start on a sector"
        pad = np.zeros(len(V) + 1, np.int64)
        np.add.at(pad, rs + rl, 1)
        np.add.at(pad, (rs + rl + VB_RUN_ALIGN - 1) // VB_RUN_ALIGN * VB_RUN_ALIGN, -1)
        want_pad = np.cumsum(pad)[:-1] > 0
        assert ((V == -2) == want_pad).all(), "pass A zeroes exactly the runs' pad slots"
    else:
        assert W == B
    for k in range(vb["parts"]):
        lo, hi = int(vb["vbase"][k]), int(vb["vbase"][k + 1])
        assert hi - lo <= max(W, (B + VB_ALIGN - 1) // VB_ALIGN * VB_ALIGN), "a virtual block fits in pass B's window"
        used = writes[lo:hi] > 0
        assert (writes[lo:hi][used] == 1).all(), "pass A writes a slot once"
        cnt = int(used.sum())
        assert used[:cnt].all(), "a virtual block's slots are a prefix"
        assert vb["sectors"] or cnt <= B, "a packed virtual block holds at most B slots"
    for l in range(plan["n_loc"]):
        k = int(np.searchsorted(vb["row0"], l, side="right") - 1)
        g0, g1 = int(vb["goffv"][l]), int(vb["goffv"][l + 1])
        d = int(vb["lens"][l])
        assert g1 - g0 == max(1, (d + CB_G - 1) // CB_G), "one segment per row, ceil(cold / 4) groups, at least one"
        seg = vb["ids"][g0 * CB_G:g1 * CB_G]
        assert (seg[d:] == W).all(), "padding = the zero slot"
        assert (seg[:d] < W).all()
        assert (V[int(vb["vbase"][k]) + seg[:d]] >= 0).all(), "pass B never names a pad slot"
        assert V[int(vb["vbase"][k]) + seg[:d]].tolist() == built["sell"][l].tolist(), \
            "pass B's ids resolve to the sources of the row's cold edges, in CSR order"
    assert vb["edges"] == sum(len(built["sell"][l]) for l in range(plan["n_loc"]))


# ---- k_pr_cb's chunks and tasks (cb_chunk_table, layout_fused_tasks in pr_layout.cu) ----------------------------
CB_TASK_CHUNKS = 32


def _cb_cut(goff_j, nr, gend, q, C):
    """cb_cut of k_cb_chunks: where a chunk boundary aimed at group q of a block lands -> (group, row, the boundary
    lies inside a segment longer than C)"""
    if q >= gend:
        return gend, nr, False
    lo = int(np.searchsorted(goff_j, q, side="right")) - 1
    s0 = int(goff_j[lo])
    s1 = int(goff_j[lo + 1]) if lo + 1 < nr else gend
    if s0 == q:
        return q, lo, False
    if s1 - s0 > C:
        return q, lo, True
    return s1, lo + 1, False


def hot_chunks(plan, goff, sms=H100_SMS, T=CB_TASK_CHUNKS):
    """cb_chunk_table of the hot blocks' stream: the chunks (g0, g1, hot rank j) in block order, the tasks (first
    chunk, chunks, j) of up to T consecutive chunks of one block, and n_fix, the chunks whose end cuts a segment
    that goes on past the next chunk's start (the fix list of k_pr_fixup / pass B)"""
    NG = int(goff[-1])
    if NG == 0:
        return [], [], 0
    gbeg = goff[plan["poff"]]
    C = min(max(NG // (sms * 8 * T), 16384 // T), 65536 // T)
    C = max(32, (C + 31) // 32 * 32)
    chunks, tasks, n_fix = [], [], 0
    for j in range(plan["KB"]):
        g0, g1, nr = int(gbeg[j]), int(gbeg[j + 1]), int(plan["nrows"][j])
        Cj = min(C, max(min(64, C), ((g1 - g0) // 64 + 63) // 64 * 64))
        nc = (g1 - g0 + Cj - 1) // Cj
        goff_j = goff[plan["poff"][j]:plan["poff"][j] + nr]
        c0 = len(chunks)
        for k in range(nc):
            a = _cb_cut(goff_j, nr, g1, g0 + k * Cj, Cj)
            b = (g1, nr, False) if k + 1 == nc else _cb_cut(goff_j, nr, g1, g0 + (k + 1) * Cj, Cj)
            interior = a[2] and (b[1] if b[2] else b[1] - 1) == a[1]
            n_fix += b[2] and not interior
            chunks.append((a[0], b[0], j))
        tasks += [(c0 + c, min(nc, c + T) - c, j) for c in range(0, nc, T)]
    return chunks, tasks, n_fix


def fused_tasks(plan, goff, vb, sms=H100_SMS):
    """layout_fused_tasks: k_pr_cb<CB_FUSED>'s tasks (first hot chunk, hot chunks, first pass-A chunk, pass-A
    chunks, source block).  Source blocks with hot or pass-A chunks, fattest first by the bytes their chunks stream
    (8 per hot group, 6 per pass-A position: a 2-byte id and a 4-byte value), ties by block; task i of a block
    takes the block's i-th hot task and its i-th run of CB_TASK_CHUNKS pass-A chunks.  Also returns the hot
    chunks and tasks and n_fix (hot_chunks)."""
    chunks, htasks, n_fix = hot_chunks(plan, goff, sms)
    nblk = plan["nblk"]
    nbytes = np.zeros(nblk, np.int64)
    hot_of = [[] for _ in range(nblk)]
    for t in htasks:
        b = int(plan["blk"][t[2]])
        hot_of[b].append(t)
        nbytes[b] += sum(8 * (chunks[c][1] - chunks[c][0]) for c in range(t[0], t[0] + t[1]))
    bin_blk = vb["pos_blk"][vb["bin_chunks"][:, 0] * BIN_STEP]
    a_first = np.searchsorted(bin_blk, np.arange(nblk))
    a_count = np.bincount(bin_blk, minlength=nblk)
    nbytes += 6 * BIN_STEP * ((vb["bcnt"] + BIN_STEP - 1) // BIN_STEP)
    tasks = []
    for b in sorted(np.flatnonzero(nbytes), key=lambda b: -nbytes[b]):
        na_all = int(a_count[b])
        for i in range(max(len(hot_of[b]), (na_all + CB_TASK_CHUNKS - 1) // CB_TASK_CHUNKS)):
            h0, nh = hot_of[b][i][:2] if i < len(hot_of[b]) else (0, 0)
            a0 = min(na_all, i * CB_TASK_CHUNKS)
            tasks.append((h0, nh, int(a_first[b]) + a0, min(na_all - a0, CB_TASK_CHUNKS), int(b)))
    return dict(tasks=tasks, hot_chunks=chunks, hot_tasks=htasks, n_fix=n_fix, bin_blk=bin_blk)


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
                va, vr = vblocks(plan, a), vblocks(plan, b)
                check_vblocks(plan, va, a)
                assert all(np.array_equal(va[k], vr[k]) for k in va), "streamed and resident virtual blocks agree"
    print("layout model ok")


if __name__ == "__main__":
    main()
