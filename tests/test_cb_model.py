"""CPU check of the column-block chunk logic (tools/cb_model.py): the lane-level numpy restatement of
cb_cut / k_cb_chunks (graph_b200/csrc/pr_layout.cu) and cb_walk / cb_fix_segment (pagerank.cu) must reproduce a direct
per-segment sum for random segment lengths, including segments cut by chunk and step boundaries."""
import sys
from pathlib import Path

import numpy as np
import pytest

sys.path.insert(0, str(Path(__file__).resolve().parent.parent / "tools"))
import cb_model  # noqa: E402


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_chunk_model_matches_direct_sums(seed):
    rng = np.random.default_rng(seed)
    cuts = 0
    kinds = set()
    for _ in range(16):
        C = int(rng.choice([32, 64, 96, 256]))
        nrows, gpp = cb_model.random_case(rng, int(rng.integers(1, 6)), int(rng.integers(1, 300)),
                                          float(rng.choice([0, 0.02, 0.2])), C)
        err, n_chunks, n_fix = cb_model.simulate(nrows, gpp, C, rng, kinds)
        assert err <= 2.5e-7          # one f32 rounding of the partial
        cuts += n_fix
    assert cuts > 0                   # the cut-segment path was exercised
    # both step widths ran, each on chunks with and without a cut segment at an end
    assert kinds == {(2, False), (2, True), (4, False), (4, True)}


def test_chunk_cut_rules():
    # a segment longer than C is cut at the nominal position; a shorter one moves the cut to its end
    goff = np.array([0, 10, 200, 205])       # three segments: 10, 190, 5 groups
    assert cb_model.cb_cut(goff, 3, 205, 0, 64) == (0, 0, False)
    assert cb_model.cb_cut(goff, 3, 205, 5, 64) == (10, 1, False)      # inside the 10-group segment: snap forward
    assert cb_model.cb_cut(goff, 3, 205, 64, 64) == (64, 1, True)      # inside the 190-group segment: cut stays
    assert cb_model.cb_cut(goff, 3, 205, 202, 64) == (205, 3, False)   # inside the last short segment
    assert cb_model.cb_cut(goff, 3, 205, 300, 64) == (205, 3, False)
