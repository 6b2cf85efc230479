"""The CPU replay of the delta-stepping queue rules (tools/sssp_model.py) on the fixtures of test_gpu_sssp.py:
its distances are the f32 fixed point, its bucket advance is the header's bit for bit, the old pile rule (one
entry per bucket epoch, all carried over) lets the far pile outgrow the old 2n + 1024 capacity on the comb and
the dense random graphs, and with one entry per vertex (in_pile) every queue stays within n entries (the
capacity sssp.cu allocates)."""
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest

import oracle
import sssp_fixtures as fx

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT / "tools"))
import sssp_model as sm  # noqa: E402


@pytest.fixture(scope="module", params=fx.REPLAYED)
def case(request):
    f = fx.FIXTURES[request.param]()
    off, tgt, w = oracle.csr_build(f.src, f.dst, f.n, oracle.OUTGOING, oracle.SORTED, f.w)
    return request.param, f, (off, tgt, w)


def test_replay_distances_are_the_fixed_point(case):
    name, f, (off, tgt, w) = case
    r = sm.replay(off, tgt, w, f.start, f.delta)
    want = oracle.sssp_bellman_ford(off, tgt, w, f.start)
    assert r.dist.tobytes() == want.tobytes(), name
    assert sm.replay(off, tgt, w, f.start, f.delta, legacy_carry=True).dist.tobytes() == want.tobytes(), name


def test_stamped_split_bounds_every_queue_by_n(case):
    name, f, (off, tgt, w) = case
    r = sm.replay(off, tgt, w, f.start, f.delta)
    assert r.max_near <= f.n and r.max_far <= f.n, (name, r.max_near, r.max_far, f.n)


@pytest.mark.parametrize("name", fx.LEGACY_OVERFLOW)
def test_legacy_split_outgrows_the_old_capacity(name):
    f = fx.FIXTURES[name]()
    off, tgt, w = oracle.csr_build(f.src, f.dst, f.n, oracle.OUTGOING, oracle.SORTED, f.w)
    old = sm.replay(off, tgt, w, f.start, f.delta, legacy_carry=True)
    assert old.max_far > 2 * f.n + 1024, (name, old.max_far)
    if name.startswith(("comb", "star")):   # k chain vertices (or a_i), s targets: the pile reaches k * s
        k = s = int(name[4:])
        assert old.max_far == k * s
    new = sm.replay(off, tgt, w, f.start, f.delta)
    assert new.buckets == old.buckets       # the same buckets in the same order, only the pile is smaller


def test_extremes_fixture_stays_unreached_past_flt_max():
    f = fx.extremes()
    off, tgt, w = oracle.csr_build(f.src, f.dst, f.n, oracle.OUTGOING, oracle.SORTED, f.w)
    d = sm.replay(off, tgt, w, f.start, f.delta).dist
    half = np.float32(fx.FLT_MAX) / np.float32(2)
    assert [d[i] == fx.FLT_MAX for i in (1, 2, 5, 6, 8)] == [True] * 5
    assert d[3] == 0.0 and not np.signbit(d[3]) and d[4] == half and d[7] == half and d[10] == half


def _bits(x):
    return int(np.float32(x).view(np.uint32))


def test_next_bucket_port_matches_header(tmp_path):
    exe = tmp_path / "sssp_bucket_dump"
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", f"-I{ROOT / 'graph_b200' / 'csrc'}",
           str(ROOT / "tests" / "cpp" / "sssp_bucket_dump.cpp"), "-o", str(exe)]
    subprocess.run(cmd, check=True, capture_output=True, text=True)
    f32 = np.float32
    tiny = np.array([1, 2, 3], np.uint32).view(np.float32)
    deltas = [*tiny, 1e-45, 1e-40, np.finfo(f32).tiny, 1e-30, 1e-20, 1e-8, 1e-3, 0.05, 0.1, 0.3, 0.5, 1.0, 2.0,
              1000.0, 1e20, 1e30]
    dmins = [0.0, *tiny, 1e-40, 1e-8, 0.1, 0.2, 0.3, 0.5, 1.0, 2.0, 3.0, 5.0, 1e7, 1e30, fx.FLT_MAX / 2,
             np.nextafter(fx.FLT_MAX, f32(0)), fx.FLT_MAX]
    rng = np.random.default_rng(5)
    dmins += list(rng.integers(0, 0x7F800000, 200).astype(np.uint32).view(np.float32))
    dmins += [f32(k) * f32(0.1) for k in range(1, 40)]
    triples = []
    for delta in deltas:
        delta = f32(delta)
        for dmin in dmins:
            dmin = f32(dmin)
            for old in (f32(0), dmin, np.nextafter(dmin, f32(0)), f32(dmin / f32(2))):
                if old <= dmin:
                    triples.append((dmin, delta, old))
            lo, up, _ = sm.sssp_next_bucket(dmin, delta, f32(0))
            if up < np.inf:                  # the next distance just past the bucket
                triples.append((up, delta, up))
    text = "".join(f"{_bits(a):08x} {_bits(b):08x} {_bits(c):08x}\n" for a, b, c in triples)
    r = subprocess.run([str(exe)], input=text, capture_output=True, text=True, timeout=120, check=True)
    lines = r.stdout.splitlines()
    assert len(lines) == len(triples)
    bad = []
    for (dmin, delta, old), line in zip(triples, lines):
        lo, up, steps = sm.sssp_next_bucket(dmin, delta, old)
        if f"{_bits(lo):08x} {_bits(up):08x} {steps}" != line:
            bad.append((float(dmin), float(delta), float(old), line, _bits(lo), _bits(up), steps))
    assert not bad, bad[:10]
