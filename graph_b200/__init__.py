"""graph_b200 — H100-native drop-in for the CSR hot path of neo4j-labs/graph.

The public names mirror the reference's Python module ``graph_mate`` (crates/mate/graph_mate.pyi:
``DiGraph``, ``Graph``, ``Layout``, ``FileFormat``, ``PageRankResult``, ``WccResult``,
``TriangleCountResult``) so that the reference's own pytest suite reads the same against this
package.  Every algorithm call goes through the C ABI of ``libgraph_b200.so``
(include/graph_b200.h) and runs on the GPU; there is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
import sys
import time
from pathlib import Path

import numpy as np

from . import _capi
from ._capi import GraphB200Error, check, lib

__all__ = ["DiGraph", "Graph", "Layout", "FileFormat", "PageRankResult", "WccResult",
           "TriangleCountResult", "SsspResult", "PageRankConfig", "WccConfig", "DeltaSteppingConfig",
           "GraphB200Error", "device_count", "set_device", "write_graph500", "wcc_csr",
           "triangle_count_csr"]

_device = 0


def device_count() -> int:
    return int(lib.gb_device_count())


def set_device(index: int) -> None:
    """CUDA device new graphs are created on (one process per GPU sets this to LOCAL_RANK)."""
    global _device
    _device = int(index)


class Comm:
    """Single-process multi-GPU communicator (gb_comm_*): one host thread, N devices, no torch / NCCL.

        comm = Comm([0, 1])
        graphs = [DiGraph.rmat(22) under set_device(d) for d in comm.devices]   # the same graph on each
        result = comm.page_rank(graphs, max_iterations=20, tolerance=0.0)
    """

    def __init__(self, devices):
        self.devices = [int(d) for d in devices]
        arr = (C.c_int * len(self.devices))(*self.devices)
        self._c = C.c_void_p()
        check(lib.gb_comm_init(len(self.devices), arr, C.byref(self._c)))

    def __del__(self):
        c, self._c = getattr(self, "_c", None), None
        if c:
            try:
                lib.gb_comm_free(c)
            except Exception:
                pass

    @property
    def multicast(self) -> bool:
        n, mc = C.c_int(0), C.c_int(0)
        check(lib.gb_comm_info(self._c, C.byref(n), C.byref(mc)))
        return bool(mc.value)

    def page_rank(self, graphs, *, max_iterations: int = 20, tolerance: float = 1e-4, damping_factor: float = 0.85):
        """page_rank over the communicator's devices (JACOBI schedule); graphs[i] must live on devices[i]."""
        if len(graphs) != len(self.devices):
            raise ValueError("one graph per device of the communicator")
        cfg = _capi.PageRankConfig(int(max_iterations), float(tolerance), float(damping_factor), _capi.PR_JACOBI)
        arr = (C.c_void_p * len(graphs))(*[g._g for g in graphs])
        scores = np.empty(graphs[0].node_count(), np.float32)
        it, err = C.c_uint64(0), C.c_double(0.0)

        def go():
            check(lib.gb_page_rank_multi(self._c, arr, C.byref(cfg), _ptr(scores), C.byref(it), C.byref(err)))
        _, micros = _timed(go)
        return PageRankResult(scores, int(it.value), float(err.value), micros)

    def page_rank_csr(self, in_offsets, in_targets, out_offsets, *, max_iterations: int = 20,
                      tolerance: float = 1e-4, damping_factor: float = 0.85) -> "PageRankResult":
        """page_rank of a host CSR over the communicator's devices, with no resident twin
        (gb_page_rank_csr_multi_u32): each device uploads about 1/ndev of the arrays over its own bus, every rank
        gathers its rows from the parts and builds its shard, and the sweeps are those of page_rank (JACOBI).
        Same arrays and checks as DiGraph.for_page_rank; pass pinned arrays to overlap the upload."""
        io, it_, oo = _page_rank_csr_arrays(in_offsets, in_targets, out_offsets, "page_rank_csr")
        cfg = _capi.PageRankConfig(int(max_iterations), float(tolerance), float(damping_factor), _capi.PR_JACOBI)
        scores = np.empty(len(io) - 1, np.float32)
        it, err = C.c_uint64(0), C.c_double(0.0)

        def go():
            check(lib.gb_page_rank_csr_multi_u32(self._c, len(io) - 1, _ptr(io), _ptr(it_) if len(it_) else None,
                                                 _ptr(oo), C.byref(cfg), _ptr(scores), C.byref(it), C.byref(err)))
        _, micros = _timed(go)
        return PageRankResult(scores, int(it.value), float(err.value), micros)

    def pr_shards_csr(self, in_offsets, in_targets, out_offsets, *, ranks_per_device: int = 1):
        """The shards of page_rank_csr (gb_pr_shards_csr_u32) as multigpu.CudaShardBackend objects, rank r on
        devices[r // ranks_per_device], for a caller that drives the sweeps itself."""
        from .multigpu import CudaShardBackend
        io, it_, oo = _page_rank_csr_arrays(in_offsets, in_targets, out_offsets, "pr_shards_csr")
        world = len(self.devices) * int(ranks_per_device)
        arr = (C.c_void_p * max(world, 1))()
        check(lib.gb_pr_shards_csr_u32(self._c, int(ranks_per_device), len(io) - 1, _ptr(io),
                                       _ptr(it_) if len(it_) else None, _ptr(oo), arr))
        return [CudaShardBackend.from_handle(arr[r], r, world, len(io) - 1,
                                             f"cuda:{self.devices[r // int(ranks_per_device)]}")
                for r in range(world)]

    def wcc_csr(self, offsets, targets, *, chunk_size: int | None = None, neighbor_rounds: int | None = None,
                sampling_size: int | None = None, out=None):
        """graph_b200.wcc_csr over the communicator's devices (gb_wcc_csr_multi_u32): each device streams and
        links about 1/ndev of the edges over its own bus, the forests merge over NVLink, and the labels are
        the same.  Same checks and `out` as wcc_csr; a config value left at None is WccConfig's default."""
        d = WccConfig()
        return _wcc_csr_call(lib.gb_wcc_csr_multi_u32, self._c, offsets, targets,
                             d.chunk_size if chunk_size is None else chunk_size,
                             d.neighbor_rounds if neighbor_rounds is None else neighbor_rounds,
                             d.sampling_size if sampling_size is None else sampling_size, out)


# ---- enums (crates/mate/src/graphs/mod.rs Layout / FileFormat; csr.rs:35-45) --------------------
class _Enum:
    def __init__(self, cls_name: str, name: str, value: int):
        self._cls, self.name, self.value = cls_name, name, value

    def __repr__(self):
        return f"{self._cls}.{self.name}"

    def __int__(self):
        return self.value


class Layout:
    """How neighbor lists are organised inside the CSR target array (csr.rs:35-45)."""
    Unsorted = _Enum("Layout", "Unsorted", _capi.LAYOUT_UNSORTED)
    Sorted = _Enum("Layout", "Sorted", _capi.LAYOUT_SORTED)
    Deduplicated = _Enum("Layout", "Deduplicated", _capi.LAYOUT_DEDUPLICATED)


class FileFormat:
    Graph500 = _Enum("FileFormat", "Graph500", 0)
    EdgeList = _Enum("FileFormat", "EdgeList", 1)
    Binary = _Enum("FileFormat", "Binary", 2)  # SerializeGraphOp's file (input/binary.rs); see serialize()


def _layout_value(layout) -> int:
    if layout is None:
        return _capi.LAYOUT_UNSORTED  # CsrLayout::default(), csr.rs:35-45
    if isinstance(layout, _Enum) and layout._cls == "Layout":
        return layout.value
    raise TypeError(f"layout must be a graph_b200.Layout, got {layout!r}")


# ---- configs (plain structs with the reference defaults) -----------------------------------------
class PageRankConfig:
    """crates/algos/src/page_rank.rs:14-56"""
    DEFAULT_MAX_ITERATIONS = 20
    DEFAULT_TOLERANCE = 1e-4
    DEFAULT_DAMPING_FACTOR = 0.85

    def __init__(self, max_iterations=DEFAULT_MAX_ITERATIONS, tolerance=DEFAULT_TOLERANCE,
                 damping_factor=DEFAULT_DAMPING_FACTOR):
        self.max_iterations, self.tolerance, self.damping_factor = max_iterations, tolerance, damping_factor


class WccConfig:
    """crates/algos/src/wcc.rs:40-79"""
    DEFAULT_CHUNK_SIZE = 16384
    DEFAULT_NEIGHBOR_ROUNDS = 2
    DEFAULT_SAMPLING_SIZE = 1024

    def __init__(self, chunk_size=DEFAULT_CHUNK_SIZE, neighbor_rounds=DEFAULT_NEIGHBOR_ROUNDS,
                 sampling_size=DEFAULT_SAMPLING_SIZE):
        self.chunk_size, self.neighbor_rounds, self.sampling_size = chunk_size, neighbor_rounds, sampling_size


class DeltaSteppingConfig:
    """crates/algos/src/sssp.rs:18-36"""

    def __init__(self, start_node: int, delta: float):
        self.start_node, self.delta = start_node, delta


# ---- results (crates/mate/src/{page_rank,wcc,triangle_count}.rs) ----------------------------------
def _took(micros: int) -> str:
    return f"{micros / 1000.0:.3f}ms" if micros >= 1000 else f"{micros}µs"


class PageRankResult:
    def __init__(self, scores, ran_iterations, error, micros):
        scores.flags.writeable = False
        self._scores, self.ran_iterations, self.error, self.micros = scores, ran_iterations, error, micros

    def scores(self) -> np.ndarray:
        return self._scores

    def __repr__(self):
        return (f'PageRankResult {{ scores: "[... {len(self._scores)} values]", ran_iterations: '
                f"{self.ran_iterations}, error: {self.error}, took: {_took(self.micros)} }}")


class WccResult:
    def __init__(self, components, micros):
        components.flags.writeable = False
        self._components, self.micros = components, micros

    def components(self) -> np.ndarray:
        return self._components

    def __repr__(self):
        return f'WccResult {{ components: "[... {len(self._components)} values]", took: {_took(self.micros)} }}'


class TriangleCountResult:
    def __init__(self, triangles, micros, info=None):
        self.triangles, self.micros = triangles, micros
        self.info = info  # triangle_count_csr: the call's gb_tc_csr_info as a dict

    def __repr__(self):
        return f"TriangleCountResult {{ triangles: {self.triangles}, took: {_took(self.micros)} }}"


class SsspResult:
    def __init__(self, distances, micros):
        distances.flags.writeable = False
        self._distances, self.micros = distances, micros

    def distances(self) -> np.ndarray:
        return self._distances

    def __repr__(self):
        return f'SsspResult {{ distances: "[... {len(self._distances)} values]", took: {_took(self.micros)} }}'


# ---- input files (crates/builder/src/input/{graph500,edgelist}.rs) --------------------------------
# DiGraph.load / Graph.load stream the file to the device and parse it there (csrc/load.cu).  The host
# readers below (csrc/io.cu) give the same edges; they serve the Flight server's weighted undirected graphs
# and are the reference the device loader is tested against.
def _load_args(path, file_format, layout):
    """(path bytes, format value, layout value) for gb_*_load_u32; raises what opening the file raises."""
    if file_format in (FileFormat.Graph500, FileFormat.EdgeList, FileFormat.Binary):
        fmt = file_format.value
    else:
        raise TypeError(f"unknown file format {file_format!r}")
    path = os.fspath(path)
    open(path, "rb").close()  # FileNotFoundError / IsADirectoryError / PermissionError as before
    return os.fsencode(path), fmt, _layout_value(layout)


def _read_graph500(path) -> tuple[np.ndarray, np.ndarray, int]:
    """Packed 12-byte edges {v0_low, v1_low, high} (graph500.rs:111-127); node_count = edges/16 (:74)."""
    raw = np.fromfile(path, dtype=np.uint8)
    m = raw.size // 12
    src = np.empty(m, np.uint32)
    dst = np.empty(m, np.uint32)
    got, n = C.c_uint64(0), C.c_uint32(0)
    check(lib.gb_graph500_decode(_ptr(raw) if raw.size else None, raw.size, _ptr(src), _ptr(dst), C.byref(got),
                                 C.byref(n)))
    return src, dst, int(n.value)


def write_graph500(path, src, dst) -> None:
    """Writes edges as the packed Graph500 file the reference reads (`app -f graph500 --use-32-bit`,
    `DiGraph.load(path)`); the reader derives node_count = edge_count / 16 (graph500.rs:74)."""
    src = np.ascontiguousarray(src, dtype=np.uint32)
    dst = np.ascontiguousarray(dst, dtype=np.uint32)
    if len(src) != len(dst):
        raise ValueError("src and dst must have the same length")
    raw = np.empty(12 * len(src), np.uint8)
    check(lib.gb_graph500_encode(_ptr(src), _ptr(dst), len(src), _ptr(raw)))
    raw.tofile(path)


def _read_edge_list(path, with_values=False):
    """Text lines `<src> <dst>[ <value>]` with \\n or \\r\\n endings (edgelist.rs:181-279)."""
    text = Path(path).read_bytes()
    m = C.c_uint64(0)
    check(lib.gb_edge_list_parse(text, len(text), None, None, None, C.byref(m)))
    src = np.empty(m.value, np.uint32)
    dst = np.empty(m.value, np.uint32)
    w = np.empty(m.value, np.float32) if with_values else None
    check(lib.gb_edge_list_parse(text, len(text), _ptr(src), _ptr(dst), _ptr(w), C.byref(m)))
    return (src, dst, w) if with_values else (src, dst)


def _decode_binary(data: bytes, directed: bool, with_values: bool = False):
    """The host decoder of binary graph files (gb_binary_decode): (out_offsets, out_targets, out_values,
    in_offsets, in_targets) for a directed file, (offsets, targets) for an undirected one.  out_values is None
    unless with_values; in-CSR values are never returned."""
    raw = np.frombuffer(data, np.uint8)
    kind = _capi.KIND_DIRECTED if directed else _capi.KIND_UNDIRECTED
    n, m, hv = C.c_uint32(0), C.c_uint64(0), C.c_int(0)
    args = (_ptr(raw) if raw.size else None, raw.size, kind, C.byref(n), C.byref(m), C.byref(hv))
    check(lib.gb_binary_decode(*args, None, None, None, None, None))
    if with_values and not hv.value:
        raise ValueError("the binary graph file holds no edge values")
    csrs = [(np.empty(n.value + 1, np.uint32), np.empty(m.value, np.uint32)) for _ in range(2 if directed else 1)]
    w = np.empty(m.value, np.float32) if with_values else None
    inc = csrs[1] if directed else (None, None)
    check(lib.gb_binary_decode(*args, _ptr(csrs[0][0]), _ptr(csrs[0][1]), _ptr(w), _ptr(inc[0]), _ptr(inc[1])))
    return (*csrs[0], w, *csrs[1]) if directed else csrs[0]


def _check_host_csr(off: np.ndarray, tgt: np.ndarray, what: str) -> None:
    """The C side reads off[n] and copies off[n] targets: reject arrays that are too short here."""
    if off.ndim != 1 or len(off) < 2:
        raise ValueError(f"{what} offsets need node_count + 1 >= 2 entries")
    if tgt.ndim != 1 or len(tgt) < int(off[-1]):
        raise ValueError(f"{what} targets hold {len(tgt)} entries but the offsets end at {int(off[-1])}")


def _edges_from_numpy(arr) -> tuple[np.ndarray, np.ndarray]:
    a = np.asarray(arr)
    if a.ndim != 2 or a.shape[1] < 2:
        # crates/mate/src/graphs/mod.rs:441-449
        raise TypeError("Can only create a graph from a 2-dimensional array with at least 2 columns")
    if a.dtype != np.uint32:
        if not np.issubdtype(a.dtype, np.integer) or (a.size and (a.min() < 0 or a.max() > 0xFFFFFFFF)):
            raise TypeError("node ids must be 32-bit unsigned integers")
        a = a.astype(np.uint32)
    return np.ascontiguousarray(a[:, 0]), np.ascontiguousarray(a[:, 1])


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _torch_edges(src, dst, weights):
    """Device u32 id tensors (narrowed and range-checked on the device), the weights, and torch's current
    stream on the graph's device, for gb_*_from_device_edges_u32."""
    import torch  # only this constructor needs torch

    dev = torch.device("cuda", _device)

    def check_tensor(t, what, dtypes):
        if not isinstance(t, torch.Tensor) or t.device != dev:
            raise ValueError(f"{what} must be a tensor on {dev}")
        if t.dim() != 1 or not t.is_contiguous():
            raise ValueError(f"{what} must be a contiguous 1-D tensor")
        if t.dtype not in dtypes:
            raise TypeError(f"{what} must be a tensor of {' or '.join(map(str, dtypes))}")

    check_tensor(src, "src", (torch.int32, torch.int64))
    check_tensor(dst, "dst", (torch.int32, torch.int64))
    m = src.numel()
    if dst.numel() != m:
        raise ValueError("src and dst must have the same length")
    if weights is not None:
        check_tensor(weights, "weights", (torch.float32,))
        if weights.numel() != m:
            raise ValueError("weights must have one entry per edge")
    stream = torch.cuda.current_stream(dev)
    ids = []
    for t in (src, dst):
        u = torch.empty(m, dtype=torch.int32, device=dev)  # holds the u32 bit patterns
        try:
            check(lib.gb_ids_to_u32(_device, t.data_ptr(), t.element_size(), m, u.data_ptr(), stream.cuda_stream))
        except ValueError:
            raise TypeError("node ids must be 32-bit unsigned integers") from None
        ids.append(u)
    return ids[0], ids[1], weights, m, stream


# ---- graph handles ---------------------------------------------------------------------------
class _Handle:
    """Owns a gb_graph* and a lazily materialised read-only host mirror for neighbor views."""

    def __init__(self, raw_ptr, load_micros=0):
        self._g = raw_ptr
        self.load_micros = int(load_micros)
        info = _capi.GraphInfo()
        check(lib.gb_graph_get_info(self._g, C.byref(info)))
        self._info = info
        self._host = {}

    def __del__(self):
        g, self._g = getattr(self, "_g", None), None
        if g:
            try:
                lib.gb_graph_free(g)
            except Exception:  # interpreter shutdown
                pass

    def _refresh(self):
        check(lib.gb_graph_get_info(self._g, C.byref(self._info)))

    def _mirror(self, which: int):
        """(offsets, targets[, weights]) host copy of one CSR, fetched once (csr.rs:97-117 views)."""
        if which not in self._host:
            n = self._info.node_count
            ln = C.c_uint64(0)
            check(lib.gb_graph_csr_len(self._g, which, C.byref(ln)))
            off = np.empty(n + 1, np.uint32)
            tgt = np.empty(ln.value, np.uint32)
            check(lib.gb_graph_copy_csr(self._g, which, _ptr(off), _ptr(tgt) if ln.value else None, None))
            off.flags.writeable = False
            tgt.flags.writeable = False  # views are read-only (shared_slice.rs:128)
            self._host[which] = (off, tgt)
        return self._host[which]

    def _views_alive(self) -> bool:
        # a numpy view keeps a reference to its base array
        for off, tgt in self._host.values():
            if sys.getrefcount(tgt) > 3:  # tuple entry + loop variable + getrefcount argument
                return True
        return False

    def _row(self, which: int, node: int) -> np.ndarray:
        off, tgt = self._mirror(which)
        n = self._info.node_count
        if not 0 <= node < n:
            raise IndexError(f"node {node} out of range for a graph with {n} nodes")
        return tgt[off[node]:off[node + 1]]

    def _degree(self, which: int, node: int) -> int:
        off, _ = self._mirror(which)
        n = self._info.node_count
        if not 0 <= node < n:
            raise IndexError(f"node {node} out of range for a graph with {n} nodes")
        return int(off[node + 1]) - int(off[node])

    def node_count(self) -> int:
        return int(self._info.node_count)

    def edge_count(self) -> int:
        return int(self._info.edge_count)

    def device_bytes(self) -> int:
        self._refresh()
        return int(self._info.device_bytes)

    def last_timing(self) -> dict:
        t = _capi.Timing()
        check(lib.gb_graph_last_timing(self._g, C.byref(t)))
        return {"total_ms": t.total_ms, "hot_kernel_ms": t.hot_kernel_ms,
                "hot_kernel_launches": int(t.hot_kernel_launches), "kernel_launches": int(t.kernel_launches)}

    def cuda_stream(self) -> int:
        return int(lib.gb_graph_stream(self._g) or 0)

    def load_info(self) -> dict:
        """Statistics of the file load that created this graph (zeros for graphs made otherwise):
        file_bytes, chunks, edges, fallback_lines (values re-parsed on the host), h2d_bytes."""
        info = _capi.LoadInfo()
        check(lib.gb_graph_load_info(self._g, C.byref(info)))
        return info.as_dict()

    def serialize(self, path) -> None:
        """SerializeGraphOp::serialize (graph_ops.rs:232-238): writes the graph as the binary file that
        `load(path, file_format=FileFormat.Binary)` here and DeserializeGraphOp in the reference read (NI = u32;
        a weighted digraph writes Target<u32, f32> records for both CSRs).  The file is written next to `path`
        under a temporary name and renamed over it."""
        check(lib.gb_graph_serialize(self._g, os.fsencode(os.fspath(path))))

    def __repr__(self):
        return (f"{type(self).__name__} {{ node_count: {self.node_count()}, edge_count: {self.edge_count()}, "
                f"load_took: {_took(self.load_micros)} }}")


def _timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, max(1, int((time.perf_counter() - t0) * 1e6))


def _construct(cls, fn, *args):
    """cls around the graph the C constructor fn(*args, &graph) makes, with the call's time as load_micros."""
    out = C.c_void_p()
    _, micros = _timed(lambda: check(fn(*args, C.byref(out))))
    return cls(out, micros)


_PR_MODES = {"auto": _capi.PR_AUTO, "exact": _capi.PR_EXACT, "jacobi": _capi.PR_JACOBI}


class DiGraph(_Handle):
    """A directed graph using 32 bits for node ids — device twin of DirectedCsrGraph<u32>
    (crates/builder/src/graph/csr.rs:364-368; Python surface crates/mate/graph_mate.pyi:46-118)."""

    # -- construction --
    @staticmethod
    def _from_edges(src, dst, weights, node_count, layout) -> "DiGraph":
        return _construct(DiGraph, lib.gb_digraph_from_edges_u32, _device, _ptr(src), _ptr(dst), _ptr(weights),
                          len(src), node_count, _layout_value(layout))

    @staticmethod
    def load(path, layout=None, file_format=FileFormat.Graph500) -> "DiGraph":
        """Load a graph from the provided format (crates/mate/src/graphs/digraph.rs:35-44); the file is
        parsed on the device."""
        return _construct(DiGraph, lib.gb_digraph_load_u32, _device, *_load_args(path, file_format, layout), 0)

    @staticmethod
    def load_weighted(path, layout=None, file_format=FileFormat.EdgeList) -> "DiGraph":
        """Weighted text edge list `<src> <dst> <f32>`, or a binary file with Target<NI, f32> records
        (DirectedCsrGraph<u32, (), f32>, for sssp)."""
        if file_format is FileFormat.Graph500:
            raise ValueError("Graph500 files carry no edge values")
        return _construct(DiGraph, lib.gb_digraph_load_u32, _device, *_load_args(path, file_format, layout), 1)

    @staticmethod
    def from_torch(src, dst, weights=None, node_count: int = 0, layout=None) -> "DiGraph":
        """From contiguous 1-D CUDA tensors on the graph's device (ids int32 or int64, weights float32),
        without a host copy.  node_count 0 means max id + 1."""
        s, d, w, m, stream = _torch_edges(src, dst, weights)
        return _construct(DiGraph, lib.gb_digraph_from_device_edges_u32, _device, s.data_ptr(), d.data_ptr(),
                          None if w is None else w.data_ptr(), m, int(node_count), _layout_value(layout),
                          stream.cuda_stream)

    @staticmethod
    def from_numpy(arr, layout=None, weights=None, node_count: int = 0) -> "DiGraph":
        src, dst = _edges_from_numpy(arr)
        w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float32)
        if w is not None and len(w) != len(src):
            raise ValueError("weights must have one entry per edge")
        return DiGraph._from_edges(src, dst, w, node_count, layout)

    @staticmethod
    def from_pandas(df, layout=None) -> "DiGraph":
        return DiGraph.from_numpy(df.to_numpy(), layout)  # crates/mate/src/graphs/mod.rs:169-189

    @staticmethod
    def from_csr(out_offsets, out_targets, in_offsets, in_targets, out_weights=None) -> "DiGraph":
        """Device twin of an already built DirectedCsrGraph (host CSR arrays are uploaded as is)."""
        oo = np.ascontiguousarray(out_offsets, np.uint32)
        ot = np.ascontiguousarray(out_targets, np.uint32)
        io = np.ascontiguousarray(in_offsets, np.uint32)
        it = np.ascontiguousarray(in_targets, np.uint32)
        ow = None if out_weights is None else np.ascontiguousarray(out_weights, np.float32)
        _check_host_csr(oo, ot, "out")
        _check_host_csr(io, it, "in")
        if len(io) != len(oo):
            raise ValueError("in and out offsets must have the same length (node_count + 1)")
        if ow is not None and len(ow) != len(ot):
            raise ValueError("out_weights must have one entry per out target")
        return _construct(DiGraph, lib.gb_digraph_from_csr_u32, _device, len(oo) - 1, _ptr(oo), _ptr(ot), _ptr(ow),
                          _ptr(io), _ptr(it))

    @staticmethod
    def for_page_rank(in_offsets, in_targets, out_offsets) -> "DiGraph":
        """Device twin holding only what page_rank reads: the in-CSR and the out-degrees (as out offsets).
        Arrays are used as given (pass pinned uint32 arrays to upload at PCIe speed)."""
        io, it, oo = _page_rank_csr_arrays(in_offsets, in_targets, out_offsets, "for_page_rank")
        return _construct(DiGraph, lib.gb_digraph_for_page_rank_u32, _device, len(io) - 1, _ptr(io), _ptr(it),
                          _ptr(oo))

    @staticmethod
    def rmat(scale: int, edge_factor: int = 16, seed: int = 42, layout=Layout.Sorted, weights=False) -> "DiGraph":
        """Synthetic R-MAT graph generated and built on device (the BASELINE.json workload)."""
        return _construct(DiGraph, lib.gb_digraph_rmat, _device, scale, edge_factor, seed, _layout_value(layout),
                          int(bool(weights)))

    # -- accessors --
    def out_degree(self, node: int) -> int:
        return self._degree(_capi.CSR_OUT, node)

    def in_degree(self, node: int) -> int:
        return self._degree(_capi.CSR_IN, node)

    def out_neighbors(self, node: int) -> np.ndarray:
        return self._row(_capi.CSR_OUT, node)

    def in_neighbors(self, node: int) -> np.ndarray:
        return self._row(_capi.CSR_IN, node)

    def copy_out_neighbors(self, node: int) -> list:
        return self._row(_capi.CSR_OUT, node).tolist()

    def copy_in_neighbors(self, node: int) -> list:
        return self._row(_capi.CSR_IN, node).tolist()

    def out_weights(self) -> np.ndarray:
        """f32 edge values aligned with the out-CSR targets (SoA twin of Target<u32, f32>)."""
        ln = C.c_uint64(0)
        check(lib.gb_graph_csr_len(self._g, _capi.CSR_OUT, C.byref(ln)))
        off = np.empty(self.node_count() + 1, np.uint32)
        w = np.empty(ln.value, np.float32)
        check(lib.gb_graph_copy_csr(self._g, _capi.CSR_OUT, _ptr(off), None, _ptr(w)))
        return w

    def csr(self, which: str = "out"):
        """(offsets, targets) host arrays of the out or in CSR (read-only)."""
        return self._mirror(_capi.CSR_OUT if which == "out" else _capi.CSR_IN)

    def to_undirected(self, layout=None) -> "Graph":
        """New, unrelated undirected graph (graph_ops.rs:229; csr.rs:391-464)."""
        return _construct(Graph, lib.gb_to_undirected, self._g, _layout_value(layout))

    def in_degree_partition(self, parts: int) -> list:
        """graph_ops.rs:431-439 — ranges as [(start, end), ...]"""
        r = np.zeros(parts + 1, np.uint32)
        check(lib.gb_in_degree_partition(self._g, parts, _ptr(r)))
        out = [(int(r[i]), int(r[i + 1])) for i in range(parts) if r[i + 1] > r[i]]
        return out

    def page_rank_plan_info(self) -> dict:
        """Statistics of the device layout the JACOBI page_rank sweeps (built on first use)."""
        st = _capi.PrShardStats()
        check(lib.gb_page_rank_plan_info(self._g, C.byref(st)))
        return st.as_dict()

    def page_rank_plan_shape(self) -> dict:
        """Diagnostics: the launch shape of the JACOBI sweep kernels (built on first use)."""
        sh = _capi.PrPlanShape()
        check(lib.gb_page_rank_plan_shape(self._g, C.byref(sh)))
        return sh.as_dict()

    # -- algorithms --
    def page_rank(self, *, max_iterations: int = PageRankConfig.DEFAULT_MAX_ITERATIONS,
                  tolerance: float = PageRankConfig.DEFAULT_TOLERANCE,
                  damping_factor: float = PageRankConfig.DEFAULT_DAMPING_FACTOR,
                  mode: str = "auto") -> PageRankResult:
        """page_rank(&graph, PageRankConfig) (page_rank.rs:58-111); keyword-only like
        crates/mate/src/graphs/digraph.rs:126-142.  `mode`: "auto" | "exact" | "jacobi"."""
        cfg = _capi.PageRankConfig(int(max_iterations), float(tolerance), float(damping_factor), _PR_MODES[mode])
        scores = np.empty(self.node_count(), np.float32)
        it, err = C.c_uint64(0), C.c_double(0.0)

        def go():
            check(lib.gb_page_rank(self._g, C.byref(cfg), _ptr(scores), C.byref(it), C.byref(err)))
        _, micros = _timed(go)
        return PageRankResult(scores, int(it.value), float(err.value), micros)

    def wcc(self, *, chunk_size: int = WccConfig.DEFAULT_CHUNK_SIZE,
            neighbor_rounds: int = WccConfig.DEFAULT_NEIGHBOR_ROUNDS,
            sampling_size: int = WccConfig.DEFAULT_SAMPLING_SIZE) -> WccResult:
        """wcc_afforest(&graph, WccConfig).to_vec() (wcc.rs:127-139); keyword-only (digraph.rs:144-160)."""
        cfg = _capi.WccConfig(int(chunk_size), int(neighbor_rounds), int(sampling_size))
        comp = np.empty(self.node_count(), np.uint32)

        def go():
            check(lib.gb_wcc(self._g, C.byref(cfg), _ptr(comp)))
        _, micros = _timed(go)
        return WccResult(comp, micros)

    def wcc_afforest_dss(self, **kw) -> WccResult:
        """wcc_afforest_dss(&graph, config) (wcc.rs:144-156), as `Components::component` reports it: the
        minimum node id of every node's component — the same labels as wcc().  The reference variant
        differs only in its backing union-find (DisjointSetStruct, dss.rs), whose raw `to_vec()` may hold
        non-root ancestors that depend on the thread schedule; nothing consumes it (crates/app/src/app.rs:15
        drops the result), so the device path does not imitate it (DESIGN.md §2)."""
        return self.wcc(**kw)

    def wcc_baseline(self, **kw) -> WccResult:
        """wcc_baseline(&graph, config) (wcc.rs:103-123): union over every out-edge; same component labels."""
        return self.wcc(**kw)

    def delta_stepping(self, *, start_node: int, delta: float) -> SsspResult:
        """delta_stepping(&graph, DeltaSteppingConfig) (sssp.rs:38-102); needs f32 edge values."""
        if start_node < 0:
            raise ValueError("start_node must be non-negative")
        cfg = _capi.SsspConfig(int(start_node), float(delta))
        dist = np.empty(self.node_count(), np.float32)

        def go():
            check(lib.gb_sssp(self._g, C.byref(cfg), _ptr(dist)))
        _, micros = _timed(go)
        return SsspResult(dist, micros)


class Graph(_Handle):
    """An undirected graph using 32 bits for node ids — device twin of UndirectedCsrGraph<u32>
    (csr.rs:658-661; Python surface graph_mate.pyi:120-168)."""

    @staticmethod
    def _from_edges(src, dst, node_count, layout) -> "Graph":
        return _construct(Graph, lib.gb_graph_from_edges_u32, _device, _ptr(src), _ptr(dst), len(src), node_count,
                          _layout_value(layout))

    @staticmethod
    def load(path, layout=None, file_format=FileFormat.Graph500) -> "Graph":
        return _construct(Graph, lib.gb_graph_load_u32, _device, *_load_args(path, file_format, layout))

    @staticmethod
    def from_torch(src, dst, node_count: int = 0, layout=None) -> "Graph":
        """From contiguous 1-D int32 / int64 CUDA tensors on the graph's device, without a host copy."""
        s, d, _, m, stream = _torch_edges(src, dst, None)
        return _construct(Graph, lib.gb_graph_from_device_edges_u32, _device, s.data_ptr(), d.data_ptr(), m,
                          int(node_count), _layout_value(layout), stream.cuda_stream)

    @staticmethod
    def from_numpy(arr, layout=None, node_count: int = 0) -> "Graph":
        src, dst = _edges_from_numpy(arr)
        return Graph._from_edges(src, dst, node_count, layout)

    @staticmethod
    def from_pandas(df, layout=None) -> "Graph":
        return Graph.from_numpy(df.to_numpy(), layout)

    @staticmethod
    def from_csr(offsets, targets) -> "Graph":
        off = np.ascontiguousarray(offsets, np.uint32)
        tgt = np.ascontiguousarray(targets, np.uint32)
        _check_host_csr(off, tgt, "undirected")
        return _construct(Graph, lib.gb_graph_from_csr_u32, _device, len(off) - 1, _ptr(off), _ptr(tgt))

    @staticmethod
    def rmat(scale: int, edge_factor: int = 16, seed: int = 42, layout=Layout.Sorted) -> "Graph":
        return _construct(Graph, lib.gb_graph_rmat, _device, scale, edge_factor, seed, _layout_value(layout))

    def degree(self, node: int) -> int:
        return self._degree(_capi.CSR_UNDIRECTED, node)

    def neighbors(self, node: int) -> np.ndarray:
        return self._row(_capi.CSR_UNDIRECTED, node)

    def copy_neighbors(self, node: int) -> list:
        return self._row(_capi.CSR_UNDIRECTED, node).tolist()

    def csr(self):
        return self._mirror(_capi.CSR_UNDIRECTED)

    def make_degree_ordered(self) -> None:
        """Relabel by descending degree, in place (graph_ops.rs:173, 511-638)."""
        if self._views_alive():
            # crates/mate/src/graphs/mod.rs:264-276
            raise ValueError("Graph cannot be reordered because there are references to this graph from neighbor lists.")

        def go():
            check(lib.gb_make_degree_ordered(self._g))
        _, micros = _timed(go)
        self._host.clear()
        self.load_micros += micros

    def global_triangle_count(self) -> TriangleCountResult:
        """global_triangle_count(&graph) (triangle_count.rs:22-86)."""
        tri = C.c_uint64(0)

        def go():
            check(lib.gb_triangle_count(self._g, C.byref(tri)))
        _, micros = _timed(go)
        return TriangleCountResult(int(tri.value), micros)


def _page_rank_csr_arrays(in_offsets, in_targets, out_offsets, what: str):
    """The host arrays of a page-rank CSR as given: contiguous uint32, consistent lengths."""
    io, it, oo = (np.asarray(a) for a in (in_offsets, in_targets, out_offsets))
    for a in (io, it, oo):
        if a.dtype != np.uint32 or not a.flags.c_contiguous:
            raise TypeError(f"{what} needs contiguous uint32 arrays")
    _check_host_csr(io, it, "in")
    if len(oo) != len(io):
        raise ValueError("in and out offsets must have the same length (node_count + 1)")
    return io, it, oo


def _host_csr_arrays(offsets, targets, what: str, kind: str):
    """The host arrays of a one-shot call as given: contiguous uint32 (pinned arrays stay pinned)."""
    off, tgt = np.asarray(offsets), np.asarray(targets)
    for a in (off, tgt):
        if a.dtype != np.uint32 or not a.flags.c_contiguous:
            raise TypeError(f"{what} needs contiguous uint32 arrays")
    _check_host_csr(off, tgt, kind)
    return off, tgt


def _wcc_csr_call(fn, first, offsets, targets, chunk_size, neighbor_rounds, sampling_size, out) -> WccResult:
    """fn(first, node_count, offsets, targets, &config, components): gb_wcc_csr_u32 or gb_wcc_csr_multi_u32."""
    off, tgt = _host_csr_arrays(offsets, targets, "wcc_csr", "out")
    cfg = _capi.WccConfig(int(chunk_size), int(neighbor_rounds), int(sampling_size))
    if out is None:
        comp = np.empty(len(off) - 1, np.uint32)
    else:
        comp = out
        if not isinstance(comp, np.ndarray) or comp.dtype != np.uint32 or not comp.flags.c_contiguous:
            raise TypeError("out must be a contiguous uint32 numpy array")
        if comp.shape != (len(off) - 1,) or not comp.flags.writeable:
            raise ValueError(f"out must be a writeable array of node_count = {len(off) - 1} entries")

    def go():
        check(fn(first, len(off) - 1, _ptr(off), _ptr(tgt) if len(tgt) else None, C.byref(cfg), _ptr(comp)))
    _, micros = _timed(go)
    return WccResult(comp if out is None else comp.view(), micros)  # a view: `out` itself stays writeable


def wcc_csr(offsets, targets, *, chunk_size: int = WccConfig.DEFAULT_CHUNK_SIZE,
            neighbor_rounds: int = WccConfig.DEFAULT_NEIGHBOR_ROUNDS,
            sampling_size: int = WccConfig.DEFAULT_SAMPLING_SIZE, out=None) -> WccResult:
    """wcc_baseline (wcc.rs:103-123) of a host out-CSR without a resident twin: the offsets are uploaded, the
    targets streamed through a ring of device buffers and linked as they land.  Same labels as
    DiGraph.wcc() on the twin (the minimum node id of each component); the config is checked and otherwise
    ignored.  Arrays are used as given: pass pinned contiguous uint32 arrays to overlap the links with the copy.
    `out`, a contiguous uint32 array of node_count entries (e.g. a pinned torch buffer viewed as numpy), receives
    the labels instead of a new array; it is left untouched when the call fails."""
    return _wcc_csr_call(lib.gb_wcc_csr_u32, _device, offsets, targets, chunk_size, neighbor_rounds,
                         sampling_size, out)


def triangle_count_csr(offsets, targets) -> TriangleCountResult:
    """global_triangle_count (triangle_count.rs:22-86) of a host undirected CSR without a resident twin: the
    number Graph.from_csr(offsets, targets).global_triangle_count() gives, rows in any order.  The offsets are
    uploaded first, the targets in row-aligned chunks, and each chunk is checked and counted as soon as its rows
    are on the device while the next ones are on the bus; the CSR is freed before the call returns.  Arrays are
    used as given: pass pinned contiguous uint32 arrays to overlap the counts with the copy.  `info` on the
    result holds the call's chunk count, h2d bytes, chunks per kernel path and device times."""
    off, tgt = _host_csr_arrays(offsets, targets, "triangle_count_csr", "undirected")
    tri = C.c_uint64(0)

    def go():
        check(lib.gb_triangle_count_csr_u32(_device, len(off) - 1, _ptr(off), _ptr(tgt) if len(tgt) else None,
                                            C.byref(tri)))
    _, micros = _timed(go)
    info = _capi.TcCsrInfo()
    check(lib.gb_triangle_count_csr_info(C.byref(info)))
    return TriangleCountResult(int(tri.value), micros, info.as_dict())
