"""CPU-side checks of graph_b200.sssp_csr (one-shot SSSP of a host weighted out-CSR): the send order of its chunks
(sssp_send_order, graph_b200/csrc/csr_split.h) compiled with g++; the CPU replay of its bucket loop
(tools/sssp_model.py with a landing schedule: parking, unparking, lower = 0 from the first park) on every
sssp_fixtures.py graph and the sssp_csr_fixtures.py graphs, bit for bit against oracle.sssp_bellman_ford; the
late-improver graph, on which the replay goes wrong when the stale filter is kept after a park; the C symbols with
their ctypes declarations and header lines; and the Python argument checks."""
import ctypes
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
import sssp_csr_fixtures as cfx
import sssp_fixtures as fx

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import sssp_model as sm  # noqa: E402


def test_send_order_starts_at_the_start_and_wraps(tmp_path):
    exe = tmp_path / "sssp_split_check"
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'graph_b200' / 'csrc'}",
           str(ROOT / "tests" / "cpp" / "sssp_split_check.cpp"), "-o", str(exe)]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0 and "sssp_send_order ok" in r.stdout, r.stdout + r.stderr


# ---- the bucket loop with rows that land chunk by chunk, replayed -----------------------------------------------
def csr(f):
    return oracle.csr_build(f.src, f.dst, f.n, oracle.OUTGOING, oracle.SORTED, f.w)


def graphs():
    """(name, fixture, chunk budget): the queue fixtures cut into about 24 chunks, and the one-shot fixtures"""
    out = []
    for name in fx.REPLAYED:
        f = fx.FIXTURES[name]()
        out.append((name, f, max(1, -(-len(f.src) // 24))))
    for name, (make, entries) in cfx.FIXTURES.items():
        out.append((name, make(), entries))
    return out


GRAPHS = {name: (f, c) for name, f, c in graphs()}
SCHEDULES = {"start chunk only": None, "one chunk per pass": 1, "one chunk every 3 passes": 3}


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_replay_with_landing_is_the_fixed_point(name, schedule):
    f, c = GRAPHS[name]
    off, tgt, w = csr(f)
    rows = sm.chunk_rows(off, c)
    r = sm.replay(off, tgt, w, f.start, f.delta, landing=sm.Landing(rows, SCHEDULES[schedule]))
    want = oracle.sssp_bellman_ford(off, tgt, w, f.start)
    assert r.dist.tobytes() == want.tobytes(), (name, schedule)
    assert r.max_near <= f.n and r.max_far <= f.n
    if len(rows) > 2 and name in cfx.FIXTURES:
        assert r.parked > 0 and r.passes_before_last_landed > 0


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_replay_from_any_chunk(where):
    f = fx.FIXTURES["dense128"]()
    off, tgt, w = csr(f)
    rows = sm.chunk_rows(off, len(f.src) // 16)
    k = {"first": 0, "middle": (len(rows) - 1) // 2, "last": len(rows) - 2}[where]
    start = (rows[k] + rows[k + 1]) // 2
    assert sm.start_chunk(rows, start) == k
    want = oracle.sssp_bellman_ford(off, tgt, w, start)
    for step in (None, 1, 3):
        r = sm.replay(off, tgt, w, start, f.delta, landing=sm.Landing(rows, step))
        assert r.dist.tobytes() == want.tobytes(), (where, step)


def test_stale_filter_after_a_park_is_wrong_on_the_late_improver():
    f = cfx.late_improver()
    off, tgt, w = csr(f)
    rows = sm.chunk_rows(off, cfx.LATE_IMPROVER_ENTRIES)
    want = oracle.sssp_bellman_ford(off, tgt, w, f.start)
    k = 8
    assert want[1] == np.float32(np.float32(0.1) + np.float32(0.1))       # x through p
    assert (want[2:k + 2] < 1.5).all()
    for step in (None, 1, 3):
        good = sm.replay(off, tgt, w, f.start, f.delta, landing=sm.Landing(rows, step))
        assert good.dist.tobytes() == want.tobytes()
        bad = sm.replay(off, tgt, w, f.start, f.delta, landing=sm.Landing(rows, step, stale_filter=True))
        assert bad.dist.tobytes() != want.tobytes()
        assert (bad.dist[2:k + 2] > 5.0).all(), (step, bad.dist[2:k + 2])  # x's chain stays at 5.x
    # without parking the filter is right: every row present, the twin's loop
    assert sm.replay(off, tgt, w, f.start, f.delta).dist.tobytes() == want.tobytes()


# ---- the interface -------------------------------------------------------------------------------------------
OFF = np.array([0, 1, 2, 2], np.uint32)
TGT = np.array([1, 0], np.uint32)
W = np.array([1.0, 2.0], np.float32)


def test_symbols_are_exported_and_declared():
    import graph_b200 as gb
    import graph_b200._capi as capi
    lib = ctypes.CDLL(str(capi.LIB_PATH))
    header = (ROOT / "include" / "graph_b200.h").read_text()
    for name, nargs, decl in (
            ("gb_sssp_csr_u32", 7, "gb_status gb_sssp_csr_u32(int device, uint32_t node_count, const uint32_t* offsets,"),
            ("gb_sssp_csr_info", 1, "gb_status gb_sssp_csr_info(gb_sssp_csr_stats* info);")):
        assert hasattr(lib, name)
        res, args = capi.SIGNATURES[name]
        assert res is ctypes.c_int and len(args) == nargs
        assert decl in header
    assert ctypes.sizeof(capi.SsspCsrInfo) == 8 * 8 + 2 * 4 + 2 * 8
    assert "delta_stepping_csr(" in (ROOT / "include" / "graph_b200.hpp").read_text()
    assert "sssp_csr" in gb.__all__
    r = gb.SsspResult(np.zeros(3, np.float32), 5)
    assert r.info is None and repr(r) == 'SsspResult { distances: "[... 3 values]", took: 5µs }'


def test_missing_device_is_reported():
    import torch
    if torch.cuda.is_available():
        pytest.skip("this box has a GPU")
    import graph_b200 as gb
    with pytest.raises(gb.GraphB200Error, match="no CUDA device"):
        gb.sssp_csr(OFF, TGT, W, start_node=0, delta=1.0)


def test_arrays_must_be_contiguous_and_typed():
    import graph_b200 as gb
    kw = dict(start_node=0, delta=1.0)
    for args in ((OFF.astype(np.int64), TGT, W), (OFF, TGT.astype(np.int32), W), (OFF, TGT, W.astype(np.float64)),
                 (OFF, TGT, np.array([1, 9, 2, 9], np.float32)[::2]), (OFF.tolist(), TGT, W)):
        with pytest.raises(TypeError):
            gb.sssp_csr(*args, **kw)


def test_short_arrays_and_keywords():
    import graph_b200 as gb
    with pytest.raises(ValueError, match="targets hold 1 entries"):
        gb.sssp_csr(OFF, TGT[:1], W, start_node=0, delta=1.0)
    with pytest.raises(ValueError, match="weights hold 1 entries"):
        gb.sssp_csr(OFF, TGT, W[:1], start_node=0, delta=1.0)
    with pytest.raises(ValueError, match="start_node must be non-negative"):
        gb.sssp_csr(OFF, TGT, W, start_node=-1, delta=1.0)
    with pytest.raises(TypeError):
        gb.sssp_csr(OFF, TGT, W, 0, 1.0)
