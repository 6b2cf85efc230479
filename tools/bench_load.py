"""Load time of Graph500 and text edge-list files: the device loader (DiGraph.load / load_weighted, csrc/load.cu)
against the host readers it replaced (_read_graph500 / _read_edge_list + _from_edges) and against the pread
floor (the file read into pinned memory by 4 threads in 64 MiB pieces, nothing else).

    python tools/bench_load.py [--scales 20,24] [--with-26] [--runs 3] [--json out.json]

The workloads are written into a temporary directory that is removed on exit: an RMAT Graph500 file
(device generator + write_graph500), an unweighted text edge list and a weighted one with %.6g values, plus
the golden fixtures.  Every file is read once before it is timed, so the page cache is warm: the numbers
are not disk numbers.  Per workload: one warm-up of each path, then --runs timed runs alternating old and
new; the CSRs of both paths are compared byte for byte.  Peak device bytes are the high-water mark of the
device's default memory pool during one load (the pool the library allocates from)."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import graph_b200 as gb  # noqa: E402

FORMATTER = r"""
#include <stdint.h>
#include <stdio.h>
#include <stddef.h>
static char* put_u32(char* p, uint32_t v) {
  char b[10]; int n = 0;
  do { b[n++] = (char)('0' + v % 10); v /= 10; } while (v);
  while (n) *p++ = b[--n];
  return p;
}
size_t format_edges(const uint32_t* s, const uint32_t* d, const float* w, size_t m, char* out) {
  char* p = out;
  for (size_t i = 0; i < m; ++i) {
    p = put_u32(p, s[i]); *p++ = ' '; p = put_u32(p, d[i]);
    if (w) p += sprintf(p, " %.6g", (double)w[i]);
    *p++ = '\n';
  }
  return (size_t)(p - out);
}
"""


def formatter(tmp: Path):
    src = tmp / "fmt.c"
    so = tmp / "fmt.so"
    src.write_text(FORMATTER)
    subprocess.run(["cc", "-O2", "-shared", "-fPIC", str(src), "-o", str(so)], check=True)
    f = C.CDLL(str(so)).format_edges
    f.restype = C.c_size_t
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    return f


def write_text(fmt, path, src, dst, w=None, block=1 << 22):
    blocks = [(i, min(i + block, len(src))) for i in range(0, len(src), block)]

    def one(b):
        s, d = src[b[0]:b[1]], dst[b[0]:b[1]]
        ww = None if w is None else w[b[0]:b[1]]
        out = np.empty((b[1] - b[0]) * (36 if w is not None else 22), np.uint8)
        n = fmt(s.ctypes.data, d.ctypes.data, None if ww is None else ww.ctypes.data, len(s), out.ctypes.data)
        return out[:n]

    with open(path, "wb") as f, ThreadPoolExecutor(8) as ex:
        for chunk in ex.map(one, blocks):
            f.write(chunk.data)


class Pool:
    """High-water mark of the default memory pool of device 0 (libcudart is shared with the library)."""

    def __init__(self):
        self.rt = C.CDLL("libcudart.so.12")
        self.pool = C.c_void_p()
        assert self.rt.cudaDeviceGetDefaultMemPool(C.byref(self.pool), 0) == 0

    def reset(self):
        zero = C.c_uint64(0)
        self.rt.cudaMemPoolSetAttribute(self.pool, 8, C.byref(zero))  # cudaMemPoolAttrUsedMemHigh

    def high(self) -> int:
        v = C.c_uint64(0)
        self.rt.cudaMemPoolGetAttribute(self.pool, 8, C.byref(v))
        return int(v.value)


def pread_floor(path, pinned, threads=4, piece=64 << 20):
    size = os.path.getsize(path)
    fd = os.open(path, os.O_RDONLY)
    try:
        def reader(r):
            view = memoryview(pinned[r * piece:(r + 1) * piece].numpy())
            for off in range(r * piece, size, threads * piece):
                n = min(piece, size - off)
                got = os.preadv(fd, [view[:n]], off)
                assert got == n
        t0 = time.perf_counter()
        with ThreadPoolExecutor(threads) as ex:
            list(ex.map(reader, range(threads)))
        return time.perf_counter() - t0
    finally:
        os.close(fd)


def old_path(path, fmt, weighted):
    if fmt is gb.FileFormat.Graph500:
        src, dst, n = gb._read_graph500(path)
        return gb.DiGraph._from_edges(src, dst, None, n, gb.Layout.Sorted)
    if weighted:
        src, dst, w = gb._read_edge_list(path, with_values=True)
        return gb.DiGraph._from_edges(src, dst, w, 0, gb.Layout.Sorted)
    src, dst = gb._read_edge_list(path)
    return gb.DiGraph._from_edges(src, dst, None, 0, gb.Layout.Sorted)


def new_path(path, fmt, weighted):
    if weighted:
        return gb.DiGraph.load_weighted(path, layout=gb.Layout.Sorted)
    return gb.DiGraph.load(path, layout=gb.Layout.Sorted, file_format=fmt)


def same_csr(a, b, weighted):
    arrs = lambda g: list(g.csr("out")) + list(g.csr("in")) + ([g.out_weights()] if weighted else [])  # noqa: E731
    return a.node_count() == b.node_count() and all(x.tobytes() == y.tobytes() for x, y in zip(arrs(a), arrs(b)))


def bench(name, path, fmt, weighted, runs, pool, pinned):
    with open(path, "rb") as f:  # warm the page cache
        while f.read(1 << 26):
            pass
    res = {"workload": name, "file_bytes": os.path.getsize(path)}
    a, b = old_path(path, fmt, weighted), new_path(path, fmt, weighted)
    res["csr_byte_equal"] = same_csr(a, b, weighted)
    res["edges"] = b.load_info()["edges"]
    res["fallback_lines"] = b.load_info()["fallback_lines"]
    res["chunks"] = b.load_info()["chunks"]
    del a, b
    floor, old, new = [], [], []
    for _ in range(runs):
        floor.append(pread_floor(path, pinned))
        for fn, acc in ((old_path, old), (new_path, new)):
            t0 = time.perf_counter()
            g = fn(path, fmt, weighted)
            acc.append(time.perf_counter() - t0)
            del g
    for fn, key in ((old_path, "old"), (new_path, "new")):
        pool.reset()
        g = fn(path, fmt, weighted)
        res[f"peak_device_bytes_{key}"] = pool.high()
        del g
    res["pread_floor_s"] = min(floor)
    res["old_s"] = min(old)
    res["new_s"] = min(new)
    res["old_runs_s"] = old
    res["new_runs_s"] = new
    res["new_over_floor"] = res["new_s"] / res["pread_floor_s"]
    res["old_over_new"] = res["old_s"] / res["new_s"]
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="20,24")
    ap.add_argument("--with-26", action="store_true", help="also scale 26 (12.9 GB Graph500 + ~18 GB of text)")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": card, "page_cache": "warm (every file is read once before timing)"}), flush=True)
    pool = Pool()
    pinned = torch.empty(4 * (64 << 20), dtype=torch.uint8, pin_memory=True)
    scales = [int(s) for s in args.scales.split(",") if s] + ([26] if args.with_26 else [])
    out = {"card": card, "page_cache": "warm", "results": []}
    tmp = Path(tempfile.mkdtemp(prefix="bench_load_"))
    try:
        golden = ROOT / "tests" / "golden"
        for name, fmt, w in [("scale_8.graph500", gb.FileFormat.Graph500, False),
                             ("test.el", gb.FileFormat.EdgeList, False), ("test.wel", gb.FileFormat.EdgeList, True)]:
            out["results"].append(bench(f"golden {name}", str(golden / name), fmt, w, args.runs, pool, pinned))
        fmt_fn = formatter(tmp)
        for s in scales:
            m = 16 << s
            src = np.empty(m, np.uint32)
            dst = np.empty(m, np.uint32)
            gb.check(gb.lib.gb_rmat_edges(0, s, 42, 0, m, gb._ptr(src), gb._ptr(dst)))
            wts = np.random.default_rng(s).random(m, dtype=np.float32)
            files = [(f"rmat{s}.graph500", gb.FileFormat.Graph500, False),
                     (f"rmat{s}.el", gb.FileFormat.EdgeList, False), (f"rmat{s}.wel", gb.FileFormat.EdgeList, True)]
            gb.write_graph500(tmp / files[0][0], src, dst)
            write_text(fmt_fn, tmp / files[1][0], src, dst)
            write_text(fmt_fn, tmp / files[2][0], src, dst, wts)
            del src, dst, wts
            for name, fmt, w in files:
                out["results"].append(bench(name, str(tmp / name), fmt, w, args.runs, pool, pinned))
                os.unlink(tmp / name)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.json:
        Path(args.json).write_text(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
