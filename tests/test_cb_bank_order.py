"""CPU check of the bank-aware order of the ids inside each column-block group (tools/cb_bank_model.py,
the restatement of k_cb_bank_order in graph_b200/csrc/pr_layout.cu): the pass only permutes the ids of a
group, follows the kernel's steps chunk by chunk, and never raises a window's modelled conflict count."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import cb_bank_model as bm  # noqa: E402
import layout_model as lm  # noqa: E402


def _streams(seed, n=3000, m=60000, B=1024):
    rng = np.random.default_rng(seed)
    in_off, in_tgt, out_deg = lm.random_graph(rng, n, m, skew=1.1)
    plan, goff, ids = bm.build_streams(in_off, in_tgt, out_deg, B=B)
    return plan, goff, ids, (in_off, in_tgt, out_deg)


def test_vectorised_streams_match_the_layout_model():
    rng = np.random.default_rng(5)
    in_off, in_tgt, out_deg = lm.random_graph(rng, 400, 5000)
    plan, goff, ids = bm.build_streams(in_off, in_tgt, out_deg, B=64)
    want = lm.build(plan, in_off, in_tgt, plan["order"])
    assert (goff == want["goff"]).all()
    assert (ids.reshape(-1) == want["ids"]).all()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_order_is_a_permutation_inside_each_group(seed):
    plan, goff, ids, _ = _streams(seed)
    B = plan["B"]
    chunks = bm.chunk_table(plan, goff, sms=4)
    win = bm.windows(chunks)
    new_ids, grp, new, gi = bm.apply(ids, win, B)
    # every group is read by exactly one step of its chunk
    seen = np.bincount(gi[gi >= 0], minlength=ids.shape[0])
    assert (seen == 1).all()
    # the same ids in every group, none moved to another group
    assert (np.sort(new_ids, axis=1) == np.sort(ids, axis=1)).all()
    assert (new_ids != ids).any(), "the pass reordered nothing"
    # no set is worse by the kernel's bound, and the real wavefronts go down overall
    assert (bm.conflict_bound(new, B) <= bm.conflict_bound(grp, B)).all()
    active = np.ones(gi.shape, bool)
    assert bm.wavefronts(new, active).sum() < bm.wavefronts(grp, active).sum()
    # deterministic
    again, _, _, _ = bm.apply(ids, win, B)
    assert (again == new_ids).all()


def test_windows_follow_the_chunk_steps():
    # a chunk that starts on an odd group reads its first step from the even group before it (as padding);
    # chunks of at least CB_WIDE_MIN groups step by 128 groups (4 per lane), shorter ones by 64
    win = bm.windows([(0, 7), (7, 200), (200, 200), (200, 300)])
    assert win.tolist() == [[0, 0, 7, 2], [6, 7, 200, 4], [134, 7, 200, 4], [200, 200, 300, 2], [264, 200, 300, 2]]
    ids = np.arange(4 * 512, dtype=np.int64).reshape(512, 4) + 5
    grp, gi = bm.gather_sets(ids, win, B=1 << 15)
    assert grp.shape == (2 + 4 + 4 + 2 + 2, 32, 4)
    assert (gi[0, :4] == [0, 2, 4, 6]).all() and gi[0, 4] == -1     # set 0 of chunk 0: groups 0, 2, 4, 6
    assert gi[2, 0] == -1 and (grp[2, 0] == 1 << 15).all()          # group 6 belongs to chunk 0
    assert gi[3, 0] == 7 and (grp[3, 0] == ids[7]).all()            # set 1 of the wide step: groups 4L + 1
    assert (gi[4, :3] == [8, 12, 16]).all()                         # set 2: groups 4L + 2
    assert gi[6 + 3, 16] == -1                                      # group 200: past the chunk's end
    assert (gi[10, :2] == [200, 202]).all()


def test_full_conflict_is_spread_over_the_banks():
    # every lane's group holds banks 0, 1, 2, 3 in that order: 32-way conflicts in each of the 4 reads
    B = 4096
    grp = (np.arange(32)[:, None] * 32 + np.arange(4)[None, :]).astype(np.int64)[None]
    assert bm.conflict_bound(grp, B)[0] == 4 * 32
    new = bm.bank_order(grp, B)
    assert (np.sort(new, axis=-1) == grp).all()
    assert bm.conflict_bound(new, B)[0] == 4 * 8          # 8 lanes per bank and read: the least possible


def test_padding_is_free_and_a_good_order_is_kept():
    B = 4096
    # lane L reads bank L in every slot: no conflict anywhere, nothing to improve
    grp = (np.arange(32)[:, None] * 33 + np.arange(4)[None, :] * 1024).astype(np.int64)[None]
    assert bm.conflict_bound(grp, B)[0] == 4
    assert (bm.bank_order(grp, B) == grp).all()
    # padding only: left alone
    pad = np.full((1, 32, 4), B, np.int64)
    assert (bm.bank_order(pad, B) == pad).all()
