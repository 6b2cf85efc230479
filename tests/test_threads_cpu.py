"""gb_last_error() is thread-local: host threads that call the host-only decoders (gb_graph500_decode,
gb_binary_decode) with different malformed inputs at the same time each read back their own message.  The
decoders run on the CPU, so this holds on machines without a GPU too.  ctypes releases the GIL for every call,
so the threads are inside the library together, and between a failed call and the gb_last_error() that follows
it other threads' calls fail and set their messages."""
import ctypes as C

import numpy as np

import binary_restatement as br
import graph_b200 as gb
from thread_jobs import run_threads

THREADS = 8
ROUNDS = 3
CALLS = 40  # failing calls per thread and round


def graph500_with_wide_id(t):
    """packed records whose high word is set in record t: an id of 2^32 or more"""
    m = 1 << 16
    rec = np.zeros((m, 3), np.uint32)
    rec[:, 0] = np.arange(m) % 1000
    rec[:, 1] = (np.arange(m) * 7) % 1000
    rec[(t * 997) % m, 2] = 1
    return rec.tobytes()


def directed_csrs():
    o, t = br.sorted_csr(br.EDGES, 4)
    i, it = br.sorted_csr([(d, s) for s, d in br.EDGES], 4)
    return (o, t), (i, it)


def binary_bad_header(t):
    """an unknown id type name, one per thread"""
    (o, tg), (i, it) = directed_csrs()
    good = br.write([(o, tg, None), (i, it, None)])
    bad = f"bad{t}"
    return good[:8] + np.array([len(bad)], "<u8").tobytes() + bad.encode() + good[8 + 8 + 3:]


def binary_bad_offsets(t):
    """offsets that decrease at t + 1 rows (the message counts them)"""
    n = 64
    off = np.arange(n + 1, dtype=np.uint64) * 4
    for r in range(t + 1):
        off[2 * r + 1] = off[2 * r + 2] + 1
    tgt = np.arange(4 * n, dtype=np.uint64) % n
    return br.write([(off, tgt, None)])


def binary_bad_targets(t):
    """t + 1 targets >= node_count (the message counts them)"""
    n = 64
    off = np.arange(n + 1, dtype=np.uint64) * 4
    tgt = np.arange(4 * n, dtype=np.uint64) % n
    tgt[: t + 1] = n + np.arange(t + 1)
    return br.write([(off, tgt, None)])


def call(kind, data):
    """the failing decode; the message read from gb_last_error() right after it, on this thread"""
    raw = np.frombuffer(data, np.uint8)
    if kind == "graph500":
        m = len(data) // 12
        src, dst = np.empty(m, np.uint32), np.empty(m, np.uint32)
        got, n = C.c_uint64(0), C.c_uint32(0)
        st = gb.lib.gb_graph500_decode(gb._ptr(raw), raw.size, gb._ptr(src), gb._ptr(dst), C.byref(got), C.byref(n))
    else:
        try:
            gb._decode_binary(data, kind == "bad_header")
            st = 0
        except ValueError:
            st = 1
    return st, gb.lib.gb_last_error().decode()


KINDS = [("graph500", graph500_with_wide_id), ("bad_header", binary_bad_header),
         ("bad_offsets", binary_bad_offsets), ("bad_targets", binary_bad_targets)]


def test_each_thread_reads_its_own_error():
    inputs = []
    for t in range(THREADS):
        kind, make = KINDS[t % len(KINDS)]
        inputs.append((kind, make(t)))
    # the messages, from serial calls on this thread
    want = []
    for kind, data in inputs:
        st, msg = call(kind, data)
        assert st != 0 and msg
        want.append(msg)
    assert want[0] == "Graph500 node id does not fit 32 bits"
    assert 'got "bad1"' in want[1]
    assert want[2] == "csr offsets are not monotone (3 rows)"
    assert want[3] == "csr CSR holds 4 targets >= node_count 64"
    assert len(set(want[1:4] + want[5:8])) == 6   # distinct per thread, besides the fixed Graph500 message

    def job(t):
        def fn():
            for _ in range(CALLS):
                st, msg = call(*inputs[t])
                assert st != 0 and msg == want[t], f"read {msg!r}, its own is {want[t]!r}"
        return [(f"{inputs[t][0]} x {CALLS}", fn)]

    run_threads([job(t) for t in range(THREADS)], ROUNDS)
