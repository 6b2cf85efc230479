"""The library under concurrent host threads and CUDA streams.  ctypes releases the GIL for every call, so
Python threads run inside the library together, as the Flight server's gRPC threads and a Rust caller's rayon
threads do.  Every baseline is computed serially on the main thread and checked against the oracle as the other
tests check it (integers and distances bit for bit, EXACT PageRank bit for bit against page_rank_seq, JACOBI
within 1e-6 of the f64-accumulating page_rank_jacobi); every result a thread gets must then equal its baseline
bit for bit, JACOBI included.  Eight threads start together on a barrier and run a fixed job list in a seeded
shuffle, two or three rounds: a correctness check, not a stress loop.  Environment knobs are set before the
threads start and never while they run."""
import ctypes as C
import threading
import time
from types import SimpleNamespace

import numpy as np
import pytest

import graph_b200 as gb
import oracle
from graph_b200 import _capi
from graph_b200._capi import check, lib
from thread_jobs import run_threads

pytestmark = pytest.mark.gpu

THREADS = 8
ROUNDS = 2
PR_RTOL = 1e-6


def P(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def rmat(scale, seed=42):
    src, dst = oracle.rmat_edges(scale, seed=seed)
    n = 1 << scale
    w = oracle.rmat_weights(seed, 0, len(src))
    out_off, out_tgt, out_w = oracle.csr_build(src, dst, n, oracle.OUTGOING, oracle.SORTED, w)
    in_off, in_tgt = oracle.csr_build(src, dst, n, oracle.INCOMING, oracle.SORTED)
    return SimpleNamespace(src=src, dst=dst, w=w, n=n, edges=np.stack([src, dst], 1),
                           out_off=out_off, out_tgt=out_tgt, out_w=out_w, in_off=in_off, in_tgt=in_tgt,
                           und_sorted=oracle.csr_build(src, dst, n, oracle.UNDIRECTED, oracle.SORTED),
                           und_unsorted=oracle.csr_build(src, dst, n, oracle.UNDIRECTED, oracle.UNSORTED))


@pytest.fixture(scope="module")
def r16():
    return rmat(16)


@pytest.fixture(scope="module")
def r14():
    return rmat(14, seed=7)


def pinned(a):
    import torch
    p = torch.empty(max(len(a), 1), dtype=torch.int32, pin_memory=True).numpy().view(a.dtype)[:len(a)]
    p[:] = a
    return p


def copy_csr(g, which):
    """a fresh host copy of one CSR of g (what _Handle._mirror fetches once and caches)"""
    ln = C.c_uint64(0)
    check(lib.gb_graph_csr_len(g._g, which, C.byref(ln)))
    off = np.empty(g.node_count() + 1, np.uint32)
    tgt = np.empty(ln.value, np.uint32)
    check(lib.gb_graph_copy_csr(g._g, which, P(off), P(tgt) if ln.value else None, None))
    return off, tgt


def graph_arrays(g):
    """every array of a twin, as bytes"""
    if isinstance(g, gb.Graph):
        return [a.tobytes() for a in copy_csr(g, _capi.CSR_UNDIRECTED)]
    out = [a.tobytes() for a in copy_csr(g, _capi.CSR_OUT) + copy_csr(g, _capi.CSR_IN)]
    if g._info.has_weights:
        out.append(g.out_weights().tobytes())
    return out


def weighted_edges(off, tgt, w):
    """(row, target, value) triples in one order: parallel edges may hold their values in any order"""
    rows = np.repeat(np.arange(len(off) - 1, dtype=np.uint32), np.diff(off.astype(np.int64)))
    order = np.lexsort((w, tgt, rows))
    return rows[order].tobytes() + tgt[order].tobytes() + w[order].tobytes()


def same_pr(a, b):
    return (a.scores().tobytes() == b.scores().tobytes() and a.ran_iterations == b.ran_iterations
            and a.error == b.error)


def check_jacobi(pr, in_off, in_tgt, out_off, maxit, tol):
    want, it, _ = oracle.page_rank_jacobi(in_off, in_tgt, out_off, maxit, tol, 0.85, acc64=True)
    assert pr.ran_iterations == it
    assert np.max(np.abs(pr.scores() - want) / want) <= PR_RTOL


def set_env(monkeypatch, env):
    for k, v in env.items():
        if v is None:
            monkeypatch.delenv(k, raising=False)
        else:
            monkeypatch.setenv(k, str(v))


# ---- 1. shared twins, every algorithm at once ---------------------------------------------------------------------
EXACT_CONFIGS = [(10, 0.0), (20, 1e-4)]
JACOBI_CONFIGS = [(20, 0.0), (60, 1e-5)]
DELTAS = [0.01, 0.1]


def test_shared_twins_every_algorithm_at_once(r16, tmp_path):
    """One weighted DiGraph, one Graph built Unsorted (its row order still unknown when the threads start, so
    that several of them race to cache it) and one built Sorted, shared by eight threads that all run every
    algorithm, accessor and the serialize / load round trip on them."""
    R = r16
    dg = gb.DiGraph.from_numpy(R.edges, layout=gb.Layout.Sorted, weights=R.w, node_count=R.n)
    ug_unsorted = gb.Graph.from_numpy(R.edges, layout=gb.Layout.Unsorted, node_count=R.n)
    ug_sorted = gb.Graph.from_numpy(R.edges, layout=gb.Layout.Sorted, node_count=R.n)

    # the baselines, each checked against the oracle
    assert [a.tobytes() for a in copy_csr(dg, _capi.CSR_OUT)] == [R.out_off.tobytes(), R.out_tgt.tobytes()]
    assert [a.tobytes() for a in copy_csr(dg, _capi.CSR_IN)] == [R.in_off.tobytes(), R.in_tgt.tobytes()]
    dg_w = dg.out_weights()
    assert weighted_edges(R.out_off, R.out_tgt, dg_w) == weighted_edges(R.out_off, R.out_tgt, R.out_w)
    pr_want = {}
    for maxit, tol in EXACT_CONFIGS:
        pr = dg.page_rank(max_iterations=maxit, tolerance=tol, mode="exact")
        want, it, err = oracle.page_rank_seq(R.in_off, R.in_tgt, R.out_off, maxit, tol, 0.85)
        assert pr.scores().tobytes() == want.tobytes() and pr.ran_iterations == it and pr.error == err
        pr_want[("exact", maxit, tol)] = pr
    for maxit, tol in JACOBI_CONFIGS:
        pr = dg.page_rank(max_iterations=maxit, tolerance=tol, mode="jacobi")
        check_jacobi(pr, R.in_off, R.in_tgt, R.out_off, maxit, tol)
        pr_want[("jacobi", maxit, tol)] = pr
    wcc_want = dg.wcc().components()
    assert wcc_want.tobytes() == oracle.wcc_min_label(R.out_off, R.out_tgt).tobytes()
    deg = np.diff(R.out_off.astype(np.int64))
    starts = [int(np.argmax(deg)), int(np.flatnonzero(deg == 1)[0])]
    sssp_want = {}
    for start in starts:
        bf = oracle.sssp_bellman_ford(R.out_off, R.out_tgt, R.out_w, start)
        for delta in DELTAS:
            d = dg.delta_stepping(start_node=start, delta=delta).distances()
            assert d.tobytes() == bf.tobytes()
            sssp_want[(start, delta)] = d
    tc_sorted = oracle.triangle_count(*R.und_sorted, threads=0)
    tc_unsorted = oracle.triangle_count(*R.und_unsorted, threads=0)
    # the Unsorted graph's count comes from a twin built alike: the shared one must not cache its row order yet
    assert gb.Graph.from_numpy(R.edges, layout=gb.Layout.Unsorted, node_count=R.n).global_triangle_count().triangles \
        == tc_unsorted
    assert ug_sorted.global_triangle_count().triangles == tc_sorted
    assert [a.tobytes() for a in copy_csr(ug_unsorted, _capi.CSR_UNDIRECTED)] == [a.tobytes() for a in R.und_unsorted]
    assert dg.to_undirected(gb.Layout.Sorted).global_triangle_count().triangles == tc_sorted
    parts_want = {}
    for parts in (3, 8):
        got = dg.in_degree_partition(parts)
        assert [a for a, _ in got] + [got[-1][1]] == oracle.in_degree_partition(R.in_off, parts).tolist()
        parts_want[parts] = got
    dg.serialize(tmp_path / "serial.bin")
    file_want = (tmp_path / "serial.bin").read_bytes()
    dg_arrays = graph_arrays(dg)
    assert graph_arrays(gb.DiGraph.load_weighted(tmp_path / "serial.bin", file_format=gb.FileFormat.Binary)) \
        == dg_arrays

    def jobs(t):
        out = []
        for (mode, maxit, tol), want in pr_want.items():
            def pr(mode=mode, maxit=maxit, tol=tol, want=want):
                assert same_pr(dg.page_rank(max_iterations=maxit, tolerance=tol, mode=mode), want)
            out.append((f"page_rank {mode} {maxit} {tol}", pr))
        out.append(("wcc", lambda: assert_bytes(dg.wcc().components(), wcc_want)))
        for (start, delta), want in sssp_want.items():
            out.append((f"delta_stepping {start} {delta}", lambda s=start, d=delta, want=want:
                        assert_bytes(dg.delta_stepping(start_node=s, delta=d).distances(), want)))
        out.append(("tc unsorted", lambda: assert_eq(ug_unsorted.global_triangle_count().triangles, tc_unsorted)))
        out.append(("tc sorted", lambda: assert_eq(ug_sorted.global_triangle_count().triangles, tc_sorted)))
        out.append(("to_undirected + tc", lambda: assert_eq(
            dg.to_undirected(gb.Layout.Sorted).global_triangle_count().triangles, tc_sorted)))
        for parts, want in parts_want.items():
            out.append((f"in_degree_partition {parts}", lambda p=parts, want=want:
                        assert_eq(dg.in_degree_partition(p), want)))
        out.append(("csr out", lambda: assert_eq([a.tobytes() for a in copy_csr(dg, _capi.CSR_OUT)], dg_arrays[:2])))
        out.append(("csr in", lambda: assert_eq([a.tobytes() for a in copy_csr(dg, _capi.CSR_IN)], dg_arrays[2:4])))
        out.append(("csr views", lambda: assert_eq([a.tobytes() for a in dg.csr("out") + dg.csr("in")],
                                                   dg_arrays[:4])))
        out.append(("out_weights", lambda: assert_bytes(dg.out_weights(), dg_w)))

        def round_trip(path=tmp_path / f"thread{t}.bin"):
            dg.serialize(path)
            assert path.read_bytes() == file_want
            assert graph_arrays(gb.DiGraph.load_weighted(path, file_format=gb.FileFormat.Binary)) == dg_arrays
        out.append(("serialize + load", round_trip))
        return out

    run_threads([jobs(t) for t in range(THREADS)], ROUNDS, seed=1)


def assert_bytes(got, want):
    assert got.dtype == want.dtype and got.tobytes() == want.tobytes()


def assert_eq(got, want):
    assert got == want, (got, want)


# ---- 2. separate graphs built in parallel ---------------------------------------------------------------------
def constructions(R):
    """name -> (build(), the oracle's (out CSR with values or None, in CSR) or None for an undirected graph)"""
    e, w, n = R.edges, R.w, R.n
    sorted_w = (R.out_off, R.out_tgt, R.out_w)
    inc = (R.in_off, R.in_tgt)

    def from_torch():
        import torch
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            ts = torch.from_numpy(R.src.view(np.int32)).cuda()
            td = torch.from_numpy(R.dst.astype(np.int64)).cuda()
            tw = torch.from_numpy(w).cuda()
            return gb.DiGraph.from_torch(ts, td, tw, node_count=n, layout=gb.Layout.Sorted)

    return {
        "from_numpy Unsorted": (lambda: gb.DiGraph.from_numpy(e, layout=gb.Layout.Unsorted, weights=w, node_count=n),
                                (oracle.csr_build(R.src, R.dst, n, oracle.OUTGOING, oracle.UNSORTED, w),
                                 oracle.csr_build(R.src, R.dst, n, oracle.INCOMING, oracle.UNSORTED))),
        "from_numpy Sorted": (lambda: gb.DiGraph.from_numpy(e, layout=gb.Layout.Sorted, weights=w, node_count=n),
                              (sorted_w, inc)),
        "from_numpy Deduplicated": (lambda: gb.DiGraph.from_numpy(e, layout=gb.Layout.Deduplicated, node_count=n),
                                    ((*oracle.csr_build(R.src, R.dst, n, oracle.OUTGOING, oracle.DEDUPLICATED), None),
                                     oracle.csr_build(R.src, R.dst, n, oracle.INCOMING, oracle.DEDUPLICATED))),
        "from_csr": (lambda: gb.DiGraph.from_csr(R.out_off, R.out_tgt, R.in_off, R.in_tgt, out_weights=R.out_w),
                     (sorted_w, inc)),
        "rmat": (lambda: gb.DiGraph.rmat(14, seed=7, layout=gb.Layout.Sorted),
                 ((R.out_off, R.out_tgt, None), inc)),
        "for_page_rank": (lambda: gb.DiGraph.for_page_rank(R.in_off, R.in_tgt, R.out_off), None),
        "from_torch": (from_torch, (sorted_w, inc)),
        "Graph from_numpy": (lambda: gb.Graph.from_numpy(e, layout=gb.Layout.Sorted, node_count=n), "undirected"),
    }


def fingerprint(name, g):
    """what the algorithms give on g, and its arrays"""
    if name == "for_page_rank":
        return {"page_rank": g.page_rank(max_iterations=20, tolerance=0.0, mode="jacobi").scores().tobytes()}
    if isinstance(g, gb.Graph):
        return {"arrays": graph_arrays(g), "tc": g.global_triangle_count().triangles}
    return {"arrays": graph_arrays(g),
            "page_rank": g.page_rank(max_iterations=20, tolerance=0.0, mode="jacobi").scores().tobytes(),
            "wcc": g.wcc().components().tobytes()}


def test_separate_graphs_built_in_parallel(r14):
    """Every thread builds its own graphs through every constructor and runs the algorithms on them, then frees
    them: concurrent device builds (CUB sorts, the memory pool, buffer releases that synchronise the device)."""
    R = r14
    builds = constructions(R)
    want = {}
    for name, (build, ref) in builds.items():
        g = build()
        fp = fingerprint(name, g)
        if ref == "undirected":
            assert fp["arrays"] == [a.tobytes() for a in R.und_sorted]
            assert fp["tc"] == oracle.triangle_count(*R.und_sorted, threads=0)
        else:
            (oo, ot, ow), (io, it) = ref if ref is not None else ((R.out_off, None, None), (R.in_off, R.in_tgt))
            pr = g.page_rank(max_iterations=20, tolerance=0.0, mode="jacobi")
            check_jacobi(pr, io, it, oo, 20, 0.0)
            if ref is not None:
                assert fp["arrays"][:4] == [oo.tobytes(), ot.tobytes(), io.tobytes(), it.tobytes()]
                if ow is not None:
                    got_w = np.frombuffer(fp["arrays"][4], np.float32)
                    assert weighted_edges(oo, ot, got_w) == weighted_edges(oo, ot, ow)
                assert fp["wcc"] == oracle.wcc_min_label(oo, ot).tobytes()
        want[name] = fp

    def job(name, build):
        def fn():
            g = build()
            assert fingerprint(name, g) == want[name]
            del g
        return (name, fn)

    run_threads([[job(name, b) for name, (b, _) in builds.items()] for _ in range(THREADS)], ROUNDS, seed=2)


# ---- 3. one-shot calls in parallel, with thread-local statistics -------------------------------------------------
SSSP_INFO = ("chunks", "chunk_entries", "h2d_bytes", "pinned", "start_chunk")
TC_INFO = ("chunks", "chunk_entries", "h2d_bytes", "pinned", "sorted_chunks", "list_chunks", "first_list_chunk")


def page_rank_csr(R, maxit=20):
    """gb_page_rank_csr_u32 (JACOBI): (scores, iterations, error)"""
    cfg = _capi.PageRankConfig(maxit, 0.0, 0.85, _capi.PR_JACOBI)
    scores = np.empty(R.n, np.float32)
    it, err = C.c_uint64(0), C.c_double(0.0)
    check(lib.gb_page_rank_csr_u32(0, R.n, P(R.in_off), P(R.in_tgt), P(R.out_off), C.byref(cfg), P(scores),
                                   C.byref(it), C.byref(err)))
    return scores, int(it.value), float(err.value)


@pytest.mark.parametrize("knobs", ["default", "fed"])
def test_one_shot_calls_in_parallel(r16, monkeypatch, knobs):
    """sssp_csr (pinned and pageable), triangle_count_csr on a sorted and an unsorted CSR, wcc_csr and the streamed
    gb_page_rank_csr_u32 at once.  Each call's statistics equal the serial call's on every field that does not
    depend on timing: one thread's never show up in another's."""
    R = r16
    m, um = int(R.out_off[-1]), int(R.und_sorted[0][-1])
    env = {"GB_PR_FEED_MIN_EDGES": 0, "GB_SSSP_FEED_ENTRIES": None, "GB_SSSP_FEED_STEP": None,
           "GB_TC_FEED_ENTRIES": None, "GB_WCC_FEED_EDGES": None, "GB_PR_FEED_CHUNKS": None}
    if knobs == "fed":
        env.update({"GB_SSSP_FEED_ENTRIES": m // 40, "GB_SSSP_FEED_STEP": 1, "GB_TC_FEED_ENTRIES": um // 9,
                    "GB_WCC_FEED_EDGES": m // 16 // 4 * 4, "GB_PR_FEED_CHUNKS": 7})
    set_env(monkeypatch, env)
    start = int(np.argmax(np.diff(R.out_off.astype(np.int64))))
    host = (R.out_off, R.out_tgt, R.out_w)
    pin = tuple(pinned(a) for a in host)
    usorted, uunsorted = R.und_sorted, R.und_unsorted
    usorted_pin = tuple(pinned(a) for a in usorted)

    calls = {
        "sssp_csr pageable": lambda: gb.sssp_csr(*host, start_node=start, delta=0.1),
        "sssp_csr pinned": lambda: gb.sssp_csr(*pin, start_node=start, delta=0.1),
        "tc_csr sorted": lambda: gb.triangle_count_csr(*usorted),
        "tc_csr sorted pinned": lambda: gb.triangle_count_csr(*usorted_pin),
        "tc_csr unsorted": lambda: gb.triangle_count_csr(*uunsorted),
        "wcc_csr": lambda: gb.wcc_csr(R.out_off, R.out_tgt),
        "page_rank_csr": lambda: page_rank_csr(R),
    }

    def key(name, r):
        """the deterministic part of a result: values and the statistics that do not depend on timing"""
        if name.startswith("sssp"):
            return r.distances().tobytes(), {k: r.info[k] for k in SSSP_INFO}
        if name.startswith("tc"):
            return r.triangles, {k: r.info[k] for k in TC_INFO}
        if name == "wcc_csr":
            return r.components().tobytes()
        return r[0].tobytes(), r[1], r[2]

    want = {name: key(name, call()) for name, call in calls.items()}
    bf = oracle.sssp_bellman_ford(R.out_off, R.out_tgt, R.out_w, start).tobytes()
    assert want["sssp_csr pageable"][0] == bf and want["sssp_csr pinned"][0] == bf
    assert want["sssp_csr pinned"][1]["pinned"] == 1 and want["sssp_csr pageable"][1]["pinned"] == 0
    assert want["tc_csr sorted"][0] == want["tc_csr sorted pinned"][0] == oracle.triangle_count(*usorted, threads=0)
    assert want["tc_csr unsorted"][0] == oracle.triangle_count(*uunsorted, threads=0)
    assert want["tc_csr unsorted"][1]["list_chunks"] > 0 and want["tc_csr sorted"][1]["list_chunks"] == 0
    assert want["wcc_csr"] == oracle.wcc_min_label(R.out_off, R.out_tgt).tobytes()
    scores, it, _ = page_rank_csr(R)
    jw, jit, _ = oracle.page_rank_jacobi(R.in_off, R.in_tgt, R.out_off, 20, 0.0, 0.85, acc64=True)
    assert it == jit and np.max(np.abs(scores - jw) / jw) <= PR_RTOL
    if knobs == "fed":
        assert want["sssp_csr pageable"][1]["chunks"] >= 40 and want["tc_csr sorted"][1]["chunks"] >= 9

    def job(name, call):
        return (name, lambda: assert_eq(key(name, call()), want[name]))

    run_threads([[job(name, c) for name, c in calls.items()] for _ in range(THREADS)], ROUNDS, seed=3)


# ---- 4. errors stay on their thread ------------------------------------------------------------------------------
def sssp_info():
    info = _capi.SsspCsrInfo()
    check(lib.gb_sssp_csr_info(C.byref(info)))
    return info.as_dict()


def tc_info():
    info = _capi.TcCsrInfo()
    check(lib.gb_triangle_count_csr_info(C.byref(info)))
    return info.as_dict()


def all_zero(info):
    return all(v == 0 for v in info.values())


def test_errors_stay_on_their_thread(r16, tmp_path):
    """Five threads make failing calls whose messages are known from serial runs and read gb_last_error() right
    after; three others make calls that succeed.  After a failed one-shot call the thread's statistics are all zero,
    while the succeeding threads' equal their serial calls'."""
    R = r16
    n = R.n
    dg = gb.DiGraph.from_csr(R.out_off, R.out_tgt, R.in_off, R.in_tgt, out_weights=R.out_w)
    start = int(np.argmax(np.diff(R.out_off.astype(np.int64))))
    bad_tgt = R.out_tgt.copy()
    bad_tgt[len(bad_tgt) // 2] = n
    bad_off = R.und_sorted[0].copy()
    bad_off[1000] = bad_off[2000]

    def failing(kind, t):
        """the failing call: (status, gb_last_error() read right after it)"""
        if kind == "sssp_csr target out of range":
            st = call_status(lambda: gb.sssp_csr(R.out_off, bad_tgt, R.out_w, start_node=start, delta=0.1))
        elif kind == "triangle_count_csr offsets not monotone":
            st = call_status(lambda: gb.triangle_count_csr(bad_off, R.und_sorted[1]))
        elif kind == "delta_stepping bad start":
            st = call_status(lambda: dg.delta_stepping(start_node=n + t, delta=0.1))
        elif kind == "load missing file":
            out = C.c_void_p()
            st = lib.gb_digraph_load_u32(0, str(tmp_path / f"missing{t}.el").encode(), 1, 1, 0, C.byref(out))
        else:  # page_rank without a stop rule
            st = call_status(lambda: dg.page_rank(max_iterations=0, tolerance=0.0, mode="jacobi"))
        return st, lib.gb_last_error().decode()

    kinds = ["sssp_csr target out of range", "triangle_count_csr offsets not monotone", "delta_stepping bad start",
             "load missing file", "page_rank without a stop rule"]
    msg = {}
    for t, kind in enumerate(kinds):
        st, msg[kind] = failing(kind, t)
        assert st != 0 and msg[kind], kind
    assert "targets >= node_count" in msg[kinds[0]] and "not monotone" in msg[kinds[1]]
    assert f"missing{3}.el" in msg[kinds[3]]
    sssp_ok = gb.sssp_csr(R.out_off, R.out_tgt, R.out_w, start_node=start, delta=0.1)
    tc_ok = gb.triangle_count_csr(*R.und_sorted)
    assert sssp_ok.distances().tobytes() == oracle.sssp_bellman_ford(R.out_off, R.out_tgt, R.out_w, start).tobytes()
    assert tc_ok.triangles == oracle.triangle_count(*R.und_sorted, threads=0)
    pr_ok = dg.page_rank(max_iterations=20, tolerance=0.0, mode="jacobi")
    check_jacobi(pr_ok, R.in_off, R.in_tgt, R.out_off, 20, 0.0)
    wcc_ok = dg.wcc().components()
    assert wcc_ok.tobytes() == oracle.wcc_min_label(R.out_off, R.out_tgt).tobytes()
    sssp_stats = {k: sssp_ok.info[k] for k in SSSP_INFO}
    tc_stats = {k: tc_ok.info[k] for k in TC_INFO}

    def fail_job(kind, t):
        def fn():
            st, got = failing(kind, t)
            assert st != 0 and got == msg[kind], f"read {got!r}, its own is {msg[kind]!r}"
            if kind == kinds[0]:
                assert all_zero(sssp_info())
            if kind == kinds[1]:
                assert all_zero(tc_info())
        return (kind, fn)

    def ok_jobs():
        def sssp():
            r = gb.sssp_csr(R.out_off, R.out_tgt, R.out_w, start_node=start, delta=0.1)
            assert_bytes(r.distances(), sssp_ok.distances())
            info = sssp_info()
            assert {k: info[k] for k in SSSP_INFO} == sssp_stats and not all_zero(info)

        def tc():
            r = gb.triangle_count_csr(*R.und_sorted)
            assert r.triangles == tc_ok.triangles
            info = tc_info()
            assert {k: info[k] for k in TC_INFO} == tc_stats and not all_zero(info)
        return [("sssp_csr", sssp), ("triangle_count_csr", tc),
                ("page_rank", lambda: assert_eq(same_pr(dg.page_rank(max_iterations=20, tolerance=0.0,
                                                                     mode="jacobi"), pr_ok), True)),
                ("wcc", lambda: assert_bytes(dg.wcc().components(), wcc_ok))]

    per_thread = [[fail_job(kind, t)] * 3 for t, kind in enumerate(kinds)]
    per_thread += [ok_jobs() for _ in range(THREADS - len(kinds))]
    run_threads(per_thread, 3, seed=4)


def call_status(fn):
    try:
        fn()
    except ValueError:
        return _capi.GB_ERR_INVALID
    return _capi.GB_OK


# ---- 5. handle info and timing while another thread plans -----------------------------------------------------------
def test_info_and_timing_while_another_thread_plans(r16):
    """Thread A drops the PageRank layout and runs a JACOBI page_rank, a fixed number of times; thread B polls
    device_bytes() and last_timing() until A is done.  B must only ever see the twin's bytes with or without the
    layout's, and a timing that is all zero or that of a whole serial reset-then-run."""
    R = r16
    g = gb.DiGraph.from_csr(R.out_off, R.out_tgt, R.in_off, R.in_tgt)
    assert all(v == 0 for v in g.last_timing().values())
    bare = g.device_bytes()
    check(lib.gb_page_rank_plan_reset(g._g))
    want = g.page_rank(max_iterations=20, tolerance=0.0, mode="jacobi")
    check_jacobi(want, R.in_off, R.in_tgt, R.out_off, 20, 0.0)
    planned = g.device_bytes()
    timing = g.last_timing()
    assert planned > bare and timing["total_ms"] > 0 and timing["kernel_launches"] > 0
    assert g.device_bytes() == planned and g.last_timing()["kernel_launches"] == timing["kernel_launches"]
    done = threading.Event()
    seen = {"bytes": set(), "polls": 0}

    def plan_and_run():
        try:
            for _ in range(6):
                check(lib.gb_page_rank_plan_reset(g._g))
                assert same_pr(g.page_rank(max_iterations=20, tolerance=0.0, mode="jacobi"), want)
        finally:
            done.set()

    def poll():
        deadline = time.monotonic() + 300
        while not done.is_set() and time.monotonic() < deadline:
            b = g.device_bytes()
            assert b in (bare, planned), (b, bare, planned)
            seen["bytes"].add(b)
            t = g.last_timing()
            if any(v != 0 for v in t.values()):
                assert t["total_ms"] > 0, t
                assert (t["kernel_launches"], t["hot_kernel_launches"]) == \
                    (timing["kernel_launches"], timing["hot_kernel_launches"]), t
            seen["polls"] += 1

    run_threads([[("reset + page_rank x 6", plan_and_run)], [("poll info and timing", poll)]], 1, seed=5)
    assert seen["polls"] > 0


# ---- 6. concurrent file loads share or bypass the pinned-ring cache -------------------------------------------------
def test_concurrent_file_loads(r14, tmp_path, monkeypatch):
    """Four threads load a Graph500 file, a text edge list, a weighted text edge list and a binary file at the same
    time through the device path (GB_LOAD_CHUNK_BYTES=4096), while a fifth serialises another graph.  One load at a
    time may hold the cached pinned ring; the others stream through rings of their own.  Every graph must be the host
    reader's, byte for byte, and report the serial load's statistics: a buffer shared by two loads would corrupt
    one of them."""
    R = r14
    monkeypatch.setenv("GB_LOAD_CHUNK_BYTES", "4096")
    files = {"g500": str(tmp_path / "r.graph500"), "el": str(tmp_path / "r.el"), "wel": str(tmp_path / "r.wel"),
             "bin": str(tmp_path / "r.bin")}
    gb.write_graph500(files["g500"], R.src, R.dst)
    np.savetxt(files["el"], R.edges, fmt="%d")
    with open(files["wel"], "w") as f:
        f.write("".join(f"{a} {b} {x:.9g}\n" for a, b, x in zip(R.src.tolist(), R.dst.tolist(), R.w.tolist())))
    gb.DiGraph.from_numpy(R.edges, layout=gb.Layout.Sorted, weights=R.w, node_count=R.n).serialize(files["bin"])
    S = gb.Layout.Sorted
    loads = {
        "g500": lambda: gb.DiGraph.load(files["g500"], S, gb.FileFormat.Graph500),
        "el": lambda: gb.DiGraph.load(files["el"], S, gb.FileFormat.EdgeList),
        "wel": lambda: gb.DiGraph.load_weighted(files["wel"], S),
        "bin": lambda: gb.DiGraph.load_weighted(files["bin"], S, gb.FileFormat.Binary),
    }
    src, dst, n = gb._read_graph500(files["g500"])
    oo, ot, ow, io, it = gb._decode_binary(open(files["bin"], "rb").read(), True, with_values=True)
    host = {
        "g500": gb.DiGraph._from_edges(src, dst, None, n, S),
        "el": gb.DiGraph._from_edges(*gb._read_edge_list(files["el"]), None, 0, S),
        "wel": gb.DiGraph._from_edges(*gb._read_edge_list(files["wel"], with_values=True), 0, S),
        "bin": gb.DiGraph.from_csr(oo, ot, io, it, out_weights=ow),
    }
    want = {k: graph_arrays(h) for k, h in host.items()}
    info = {}
    for k, load in loads.items():
        g = load()
        assert graph_arrays(g) == want[k], k
        info[k] = g.load_info()
        assert info[k]["chunks"] > 1, (k, info[k])
    other = gb.Graph.from_numpy(R.edges, layout=gb.Layout.Sorted, node_count=R.n)
    other.serialize(tmp_path / "other.bin")
    other_bytes = (tmp_path / "other.bin").read_bytes()

    def load_job(k):
        def fn():
            g = loads[k]()
            assert graph_arrays(g) == want[k]
            assert g.load_info() == info[k]
        return [(f"load {k}", fn)]

    def serialize_job():
        path = tmp_path / "other_thread.bin"
        other.serialize(path)
        assert path.read_bytes() == other_bytes
    run_threads([load_job(k) for k in loads] + [[("serialize", serialize_job)]], 3, seed=6)


# ---- 7. from_torch waits for the caller's stream -------------------------------------------------------------------
SLEEP_CYCLES = 100_000_000  # about 60 ms at the H100's clocks: a delay ahead of the real ids on the stream


@pytest.fixture(scope="module")
def torch_edges(r14):
    import torch
    R = r14
    real = {"src32": torch.from_numpy(R.src.view(np.int32)).cuda(),
            "dst32": torch.from_numpy(R.dst.view(np.int32)).cuda(),
            "src64": torch.from_numpy(R.src.astype(np.int64)).cuda(),
            "dst64": torch.from_numpy(R.dst.astype(np.int64)).cuda(),
            "w": torch.from_numpy(R.w).cuda()}
    torch.cuda.synchronize()
    want_d = graph_arrays(gb.DiGraph.from_numpy(R.edges, layout=gb.Layout.Sorted, weights=R.w, node_count=R.n))
    want_u = graph_arrays(gb.Graph.from_numpy(R.edges, layout=gb.Layout.Sorted, node_count=R.n))
    assert want_d[:4] == [a.tobytes() for a in (R.out_off, R.out_tgt, R.in_off, R.in_tgt)]
    assert want_u == [a.tobytes() for a in R.und_sorted]
    return R, real, want_d, want_u


def delayed_build(torch_edges, case):
    """On a fresh side stream: id and weight tensors filled with a wrong pattern and synchronised; then, on that
    stream, a sleep, the copy of the real values into them and at once the build on that stream.  A build that did
    not wait for the stream would read the wrong pattern."""
    import torch
    R, real, want_d, want_u = torch_edges
    m, n = len(R.src), R.n
    bits = 64 if case.endswith("int64") else 32
    dt = torch.int64 if bits == 64 else torch.int32
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        ts = torch.zeros(m, dtype=dt, device="cuda")
        td = torch.zeros(m, dtype=dt, device="cuda")
        tw = torch.full((m,), -1.0, dtype=torch.float32, device="cuda")
    s.synchronize()
    S = _capi.LAYOUT_SORTED
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        ts.copy_(real[f"src{bits}"])
        td.copy_(real[f"dst{bits}"])
        if case.startswith("public"):
            if "Graph" in case:
                g = gb.Graph.from_torch(ts, td, node_count=n, layout=gb.Layout.Sorted)
            else:
                tw.copy_(real["w"])
                g = gb.DiGraph.from_torch(ts, td, tw, node_count=n, layout=gb.Layout.Sorted)
        else:
            if bits == 64:
                # gb_ids_to_u32 runs on the stream and waits for it; the weights are copied after a second sleep
                us = torch.empty(m, dtype=torch.int32, device="cuda")
                ud = torch.empty(m, dtype=torch.int32, device="cuda")
                check(lib.gb_ids_to_u32(0, ts.data_ptr(), 8, m, us.data_ptr(), s.cuda_stream))
                check(lib.gb_ids_to_u32(0, td.data_ptr(), 8, m, ud.data_ptr(), s.cuda_stream))
                ts, td = us, ud
                torch.cuda._sleep(SLEEP_CYCLES)
            out = C.c_void_p()
            if "Graph" in case:
                check(lib.gb_graph_from_device_edges_u32(0, ts.data_ptr(), td.data_ptr(), m, n, S, s.cuda_stream,
                                                         C.byref(out)))
                g = gb.Graph(out)
            else:
                tw.copy_(real["w"])
                check(lib.gb_digraph_from_device_edges_u32(0, ts.data_ptr(), td.data_ptr(), tw.data_ptr(), m, n, S,
                                                           s.cuda_stream, C.byref(out)))
                g = gb.DiGraph(out)
    assert graph_arrays(g) == (want_u if "Graph" in case else want_d), case


DELAYED = ["DiGraph int32", "DiGraph int64", "Graph int32", "Graph int64", "public DiGraph int32",
           "public DiGraph int64", "public Graph int64"]


@pytest.mark.parametrize("case", DELAYED)
def test_from_device_edges_waits_for_the_callers_stream(torch_edges, case):
    delayed_build(torch_edges, case)


def test_from_device_edges_on_four_streams_at_once(torch_edges):
    jobs = [(case, lambda c=case: delayed_build(torch_edges, c)) for case in DELAYED]
    run_threads([jobs for _ in range(4)], ROUNDS, seed=7)


# ---- 8. a shared communicator serialises its PageRank calls ---------------------------------------------------------
@pytest.mark.parametrize("devices", ["one", "all"])
def test_shared_communicator(devices):
    """Threads share one communicator: page_rank_csr on RMAT-14 and RMAT-16 (different n, so the sweep buffers are
    reallocated between calls) and page_rank on resident RMAT-16 twins, while another thread runs wcc_csr on it.
    Every result must be bit-equal to the serial call on the same communicator."""
    import torch
    ndev = torch.cuda.device_count()
    if devices == "all" and ndev < 2:
        pytest.skip("one GPU: the all-device communicator is the one-device one")
    devs = [0] if devices == "one" else list(range(ndev))
    R14, R16 = rmat(14, seed=3), rmat(16)
    twins = []
    try:
        for d in devs:
            gb.set_device(d)
            twins.append(gb.DiGraph.from_csr(R16.out_off, R16.out_tgt, R16.in_off, R16.in_tgt))
    finally:
        gb.set_device(0)
    comm = gb.Comm(devs)
    calls = {
        "page_rank_csr rmat14": (R14, 20, 0.0, lambda: comm.page_rank_csr(R14.in_off, R14.in_tgt, R14.out_off,
                                                                          max_iterations=20, tolerance=0.0)),
        "page_rank_csr rmat16": (R16, 20, 0.0, lambda: comm.page_rank_csr(R16.in_off, R16.in_tgt, R16.out_off,
                                                                          max_iterations=20, tolerance=0.0)),
        "page_rank_csr rmat16 tol": (R16, 60, 1e-5, lambda: comm.page_rank_csr(
            R16.in_off, R16.in_tgt, R16.out_off, max_iterations=60, tolerance=1e-5)),
        "page_rank twins": (R16, 20, 0.0, lambda: comm.page_rank(twins, max_iterations=20, tolerance=0.0)),
    }
    want = {}
    for name, (R, maxit, tol, call) in calls.items():
        want[name] = call()
        check_jacobi(want[name], R.in_off, R.in_tgt, R.out_off, maxit, tol)
    wcc_want = comm.wcc_csr(R16.out_off, R16.out_tgt).components()
    assert wcc_want.tobytes() == oracle.wcc_min_label(R16.out_off, R16.out_tgt).tobytes()
    pr_jobs = [(name, lambda c=call, w=want[name]: assert_eq(same_pr(c(), w), True))
               for name, (_, _, _, call) in calls.items()]
    wcc_job = ("wcc_csr", lambda: assert_bytes(comm.wcc_csr(R16.out_off, R16.out_tgt).components(), wcc_want))
    run_threads([pr_jobs for _ in range(THREADS - 1)] + [[wcc_job] * 4], ROUNDS, seed=8)
    # the communicator still works alone afterwards
    assert same_pr(calls["page_rank_csr rmat14"][3](), want["page_rank_csr rmat14"])
