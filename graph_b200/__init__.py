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
import threading
import time
from pathlib import Path

import numpy as np

from . import _capi
from ._capi import GraphB200Error, check, lib

__all__ = ["DiGraph", "Graph", "Layout", "FileFormat", "PageRankResult", "WccResult",
           "TriangleCountResult", "SsspResult", "LabelStats", "NodeLabelIndex", "NeighborLabelFrequencies",
           "NeighborLabelFrequency", "PageRankConfig", "WccConfig", "DeltaSteppingConfig",
           "GraphB200Error", "device_count", "set_device", "write_graph500", "wcc_csr", "wcc_file", "wcc_file_info",
           "triangle_count_csr", "sssp_csr", "DirectedALGraph", "UndirectedALGraph"]

_device = 0


def device_count() -> int:
    return int(lib.gb_device_count())


def set_device(index: int) -> None:
    """CUDA device new graphs are created on (one process per GPU sets this to LOCAL_RANK)."""
    global _device
    _device = int(index)


class Comm:
    """Single-process multi-GPU communicator (gb_comm_*): the calling thread drives all N devices, no torch /
    NCCL.  Threads may share one; its PageRank calls run one at a time.

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
    # node-labelled .graph file (input/dotgraph.rs); load() drops the labels, load_labeled() keeps them.
    # load_labeled(file_format=Binary) reads the labelled binary file that serialize_labeled() writes.
    DotGraph = _Enum("FileFormat", "DotGraph", 3)


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
    def __init__(self, distances, micros, info=None):
        distances.flags.writeable = False
        self._distances, self.micros = distances, micros
        self.info = info  # sssp_csr: the call's gb_sssp_csr_stats as a dict

    def distances(self) -> np.ndarray:
        return self._distances

    def __repr__(self):
        return f'SsspResult {{ distances: "[... {len(self._distances)} values]", took: {_took(self.micros)} }}'


# ---- structures over a labelled graph (crates/builder/src/input/dotgraph.rs) ------------------------
class LabelStats:
    """LabelStats (dotgraph.rs:213-219): max_degree is the largest degree of the graph, label_count the number
    of distinct labels, label_frequency a dict label -> number of nodes."""

    def __init__(self, max_degree, label_count, max_label, max_label_frequency, label_frequency):
        self.max_degree, self.label_count, self.max_label = max_degree, label_count, max_label
        self.max_label_frequency, self.label_frequency = max_label_frequency, label_frequency

    def __repr__(self):
        return (f"LabelStats {{ max_degree: {self.max_degree}, label_count: {self.label_count}, "
                f"max_label: {self.max_label}, max_label_frequency: {self.max_label_frequency} }}")


class NodeLabelIndex:
    """NodeLabelIndex (dotgraph.rs:430-532): a CSR with max_label + 1 rows; nodes(label) lists the nodes with that
    label, ascending (read-only)."""

    def __init__(self, offsets, nodes):
        offsets.flags.writeable = False
        nodes.flags.writeable = False
        self.offsets, self._nodes = offsets, nodes

    def nodes(self, label: int) -> np.ndarray:
        if not 0 <= label < len(self.offsets) - 1:
            raise IndexError(f"label {label} out of range for an index of {len(self.offsets) - 1} labels")
        return self._nodes[self.offsets[label]:self.offsets[label + 1]]


class NeighborLabelFrequency:
    """NeighborLabelFrequency (dotgraph.rs:337-365): the labels of one node's neighbours and how often each
    occurs.  get(label) is None for a label that does not occur; iteration yields (label, count) pairs, labels
    ascending."""

    def __init__(self, labels, counts):
        self._labels, self._counts = labels, counts

    def get(self, label: int):
        i = int(np.searchsorted(self._labels, label))
        if i < len(self._labels) and int(self._labels[i]) == label:
            return int(self._counts[i])
        return None

    def __len__(self):
        return len(self._labels)

    def is_empty(self) -> bool:
        return len(self._labels) == 0

    def __iter__(self):
        return zip(self._labels.tolist(), self._counts.tolist())

    iter = __iter__


class NeighborLabelFrequencies:
    """NeighborLabelFrequencies (dotgraph.rs:367-427) as a pair CSR: node u's (label, count) pairs are
    labels / counts[offsets[u]:offsets[u + 1]], labels ascending.  `micros` is the call's time, `device_ms` the
    CUDA-event time of its device work."""

    def __init__(self, offsets, labels, counts, micros=0, device_ms=0.0):
        for a in (offsets, labels, counts):
            a.flags.writeable = False
        self.offsets, self.labels, self.counts = offsets, labels, counts
        self.micros, self.device_ms = micros, device_ms

    def neighbor_frequency(self, node: int) -> NeighborLabelFrequency:
        if not 0 <= node < len(self.offsets) - 1:
            raise IndexError(f"node {node} out of range for a graph with {len(self.offsets) - 1} nodes")
        a, b = int(self.offsets[node]), int(self.offsets[node + 1])
        return NeighborLabelFrequency(self.labels[a:b], self.counts[a:b])


# ---- input files (crates/builder/src/input/{graph500,edgelist}.rs) --------------------------------
# DiGraph.load / Graph.load stream the file to the device and parse it there (csrc/load.cu).  The host
# readers below (csrc/io.cu) give the same edges; they are the reference the device loader is tested against.
def _load_args(path, file_format, layout):
    """(path bytes, format value, layout value) for gb_*_load_u32; raises what opening the file raises."""
    if file_format in (FileFormat.Graph500, FileFormat.EdgeList, FileFormat.Binary, FileFormat.DotGraph):
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


def _decode_binary_labeled(data: bytes, directed: bool, label_bytes: int = 4, with_values: bool = False):
    """The host decoder of labelled binary graph files (gb_binary_decode_labeled): the labels, then what
    _decode_binary returns.  label_bytes is NV's width (4: u32, 8: u64 / usize), which the file does not state."""
    raw = np.frombuffer(data, np.uint8)
    kind = _capi.KIND_DIRECTED if directed else _capi.KIND_UNDIRECTED
    n, m, hv = C.c_uint32(0), C.c_uint64(0), C.c_int(0)
    args = (_ptr(raw) if raw.size else None, raw.size, kind, label_bytes, C.byref(n), C.byref(m), C.byref(hv))
    check(lib.gb_binary_decode_labeled(*args, None, None, None, None, None, None))
    if with_values and not hv.value:
        raise ValueError("the binary graph file holds no edge values")
    labels = np.empty(n.value, np.uint32)
    csrs = [(np.empty(n.value + 1, np.uint32), np.empty(m.value, np.uint32)) for _ in range(2 if directed else 1)]
    w = np.empty(m.value, np.float32) if with_values else None
    inc = csrs[1] if directed else (None, None)
    check(lib.gb_binary_decode_labeled(*args, _ptr(labels), _ptr(csrs[0][0]), _ptr(csrs[0][1]), _ptr(w),
                                       _ptr(inc[0]), _ptr(inc[1])))
    return (labels, *csrs[0], w, *csrs[1]) if directed else (labels, *csrs[0])


def _load_labeled(cls, dot_fn, binary_fn, path, layout, file_format, label_bytes):
    """load_labeled: a DotGraph file through dot_fn, or a binary file with NodeValues of label_bytes each through
    binary_fn."""
    if file_format is FileFormat.Binary:
        p, _, lay = _load_args(path, file_format, layout)
        return _construct(cls, binary_fn, _device, p, lay, int(label_bytes))
    if file_format is not FileFormat.DotGraph:
        raise ValueError(f"labelled graphs load from DotGraph or Binary files, not {file_format!r}")
    if label_bytes != 4:
        raise ValueError("label_bytes is the width of a binary file's node values; a DotGraph file's labels are u32")
    p, _, lay = _load_args(path, FileFormat.DotGraph, layout)
    return _construct(cls, dot_fn, _device, p, lay)


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


def _node_values(values, node_count: int) -> np.ndarray:
    """The labels of from_numpy(node_values=...): one u32 per node; their number is the node count."""
    v = np.asarray(values)
    if v.ndim != 1 or len(v) == 0:
        raise ValueError("node_values must be a non-empty 1-D array with one label per node")
    if v.dtype != np.uint32:
        if not np.issubdtype(v.dtype, np.integer) or v.min() < 0 or v.max() > 0xFFFFFFFF:
            raise TypeError("node values must be 32-bit unsigned integers")
    if node_count and node_count != len(v):
        raise ValueError(f"node_count {node_count} differs from the {len(v)} node values")
    return np.ascontiguousarray(v, dtype=np.uint32)


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
        for key, entry in self._host.items():
            if key == "labels":
                continue
            off, tgt = entry
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

    def node_values(self) -> np.ndarray:
        """NodeValues of a labelled graph: one label per node (read-only).  A graph without labels raises
        ValueError."""
        if "labels" not in self._host:
            labels = np.empty(self.node_count(), np.uint32)
            check(lib.gb_graph_node_values(self._g, _ptr(labels)))
            labels.flags.writeable = False
            self._host["labels"] = labels
        return self._host["labels"]

    def node_value(self, node: int) -> int:
        """NodeValues::node_value (csr.rs:64-76)."""
        labels = self.node_values()
        if not 0 <= node < len(labels):
            raise IndexError(f"node {node} out of range for a graph with {len(labels)} nodes")
        return int(labels[node])

    def has_node_values(self) -> bool:
        return lib.gb_graph_node_values(self._g, None) == _capi.GB_OK

    def serialize(self, path) -> None:
        """SerializeGraphOp::serialize (graph_ops.rs:232-238): writes the graph as the binary file that
        `load(path, file_format=FileFormat.Binary)` here and DeserializeGraphOp in the reference read (NI = u32;
        a weighted digraph writes Target<u32, f32> records for both CSRs).  The file is written next to `path`
        under a temporary name and renamed over it."""
        check(lib.gb_graph_serialize(self._g, os.fsencode(os.fspath(path))))

    def serialize_labeled(self, path) -> None:
        """SerializeGraphOp::serialize of a labelled graph (DirectedCsrGraph<u32, u32> / UndirectedCsrGraph<u32,
        u32>): NodeValues<u32>, then the CSRs as serialize() writes them, without edge values.  The file loads
        with `load_labeled(path, file_format=FileFormat.Binary)`.  After make_degree_ordered() the labels are
        written as stored, which are not permuted.  A graph without labels raises ValueError."""
        check(lib.gb_graph_serialize_labeled(self._g, os.fsencode(os.fspath(path))))

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
    def load_labeled(path, layout=None, file_format=FileFormat.DotGraph, label_bytes: int = 4) -> "DiGraph":
        """A DotGraph (.graph) file as DirectedCsrGraph<u32, u32>: node_count = N, one label per node
        (input/dotgraph.rs; GraphBuilder::file_format(DotGraphInput)).  Parsed on the device when large.
        FileFormat.Binary: the file serialize_labeled() writes, or a DirectedCsrGraph<NI, NV> file of the reference
        with NV of label_bytes (4: u32, 8: u64 / usize, narrowed); its rows are kept as stored."""
        return _load_labeled(DiGraph, lib.gb_digraph_load_labeled_u32, lib.gb_digraph_load_labeled_binary_u32, path,
                             layout, file_format, label_bytes)

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
    def from_numpy(arr, layout=None, weights=None, node_count: int = 0, node_values=None) -> "DiGraph":
        """node_values: one u32 label per node (GraphBuilder::edges(..).node_values(..), builder.rs:388, 425);
        the node count is then their number."""
        src, dst = _edges_from_numpy(arr)
        if node_values is not None:
            if weights is not None:
                raise ValueError("a graph with node values carries no edge weights")
            labels = _node_values(node_values, node_count)
            return _construct(DiGraph, lib.gb_digraph_from_edges_labeled_u32, _device, _ptr(src), _ptr(dst), len(src),
                              _ptr(labels), len(labels), _layout_value(layout))
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

    def to_undirected(self, layout=None, *, weights=False) -> "Graph":
        """New, unrelated undirected graph (graph_ops.rs:229; csr.rs:391-464).  weights=True keeps the out-CSR's
        f32 values (UndirectedCsrGraph<u32, (), f32>) and needs a weighted digraph."""
        fn = lib.gb_to_undirected_weighted if weights else lib.gb_to_undirected
        return _construct(Graph, fn, self._g, _layout_value(layout))

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
    def _from_edges(src, dst, node_count, layout, weights=None) -> "Graph":
        if weights is not None:
            return _construct(Graph, lib.gb_graph_from_weighted_edges_u32, _device, _ptr(src), _ptr(dst),
                              _ptr(weights), len(src), node_count, _layout_value(layout))
        return _construct(Graph, lib.gb_graph_from_edges_u32, _device, _ptr(src), _ptr(dst), len(src), node_count,
                          _layout_value(layout))

    @staticmethod
    def load(path, layout=None, file_format=FileFormat.Graph500) -> "Graph":
        return _construct(Graph, lib.gb_graph_load_u32, _device, *_load_args(path, file_format, layout))

    @staticmethod
    def load_labeled(path, layout=None, file_format=FileFormat.DotGraph, label_bytes: int = 4) -> "Graph":
        """A DotGraph (.graph) file as UndirectedCsrGraph<u32, u32>: node_count = N, one label per node.
        FileFormat.Binary: a labelled binary file, as DiGraph.load_labeled reads one."""
        return _load_labeled(Graph, lib.gb_graph_load_labeled_u32, lib.gb_graph_load_labeled_binary_u32, path, layout,
                             file_format, label_bytes)

    @staticmethod
    def load_weighted(path, layout=None, file_format=FileFormat.EdgeList) -> "Graph":
        """Weighted text edge list `<src> <dst> <f32>`, or a binary file with Target<NI, f32> records, as
        UndirectedCsrGraph<u32, (), f32> (the reference's `loading --undirected --weighted`)."""
        if file_format is FileFormat.Graph500:
            raise ValueError("Graph500 files carry no edge values")
        if file_format is FileFormat.DotGraph:
            raise ValueError("DotGraph files carry no edge values")
        return _construct(Graph, lib.gb_graph_load_weighted_u32, _device, *_load_args(path, file_format, layout))

    @staticmethod
    def from_torch(src, dst, node_count: int = 0, layout=None, weights=None) -> "Graph":
        """From contiguous 1-D int32 / int64 CUDA tensors on the graph's device, without a host copy.  weights:
        one float32 value per edge on the same device, for UndirectedCsrGraph<u32, (), f32>."""
        s, d, w, m, stream = _torch_edges(src, dst, weights)
        if w is not None:
            return _construct(Graph, lib.gb_graph_from_device_weighted_edges_u32, _device, s.data_ptr(),
                              d.data_ptr(), w.data_ptr(), m, int(node_count), _layout_value(layout),
                              stream.cuda_stream)
        return _construct(Graph, lib.gb_graph_from_device_edges_u32, _device, s.data_ptr(), d.data_ptr(), m,
                          int(node_count), _layout_value(layout), stream.cuda_stream)

    @staticmethod
    def from_numpy(arr, layout=None, node_count: int = 0, node_values=None, weights=None) -> "Graph":
        """node_values: one u32 label per node; the node count is then their number.  weights: one f32 value
        per edge, which both entries of the edge carry (UndirectedCsrGraph<u32, (), f32>)."""
        src, dst = _edges_from_numpy(arr)
        if node_values is not None:
            if weights is not None:
                raise ValueError("a graph with node values carries no edge weights")
            labels = _node_values(node_values, node_count)
            return _construct(Graph, lib.gb_graph_from_edges_labeled_u32, _device, _ptr(src), _ptr(dst), len(src),
                              _ptr(labels), len(labels), _layout_value(layout))
        w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float32)
        if w is not None and (w.ndim != 1 or len(w) != len(src)):
            raise ValueError("weights must have one entry per edge")
        return Graph._from_edges(src, dst, node_count, layout, w)

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

    def weights(self) -> np.ndarray:
        """f32 edge values aligned with the csr() targets (SoA twin of Target<u32, f32>); a graph without values
        raises ValueError."""
        ln = C.c_uint64(0)
        check(lib.gb_graph_csr_len(self._g, _capi.CSR_UNDIRECTED, C.byref(ln)))
        off = np.empty(self.node_count() + 1, np.uint32)
        w = np.empty(ln.value, np.float32)
        check(lib.gb_graph_copy_csr(self._g, _capi.CSR_UNDIRECTED, _ptr(off), None, _ptr(w)))
        return w

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

    def label_stats(self) -> LabelStats:
        """LabelStats::from_graph (dotgraph.rs:220-313) of a labelled graph."""
        st = _capi.LabelStatsInfo()
        check(lib.gb_label_stats(self._g, C.byref(st), None, None))
        labels = np.empty(st.label_count, np.uint32)
        counts = np.empty(st.label_count, np.uint64)
        check(lib.gb_label_stats(self._g, C.byref(st), _ptr(labels), _ptr(counts)))
        return LabelStats(int(st.max_degree), int(st.label_count), int(st.max_label), int(st.max_label_frequency),
                          dict(zip(labels.tolist(), counts.tolist())))

    def node_label_index(self) -> NodeLabelIndex:
        """NodeLabelIndex::from_stats(node_count, &label_stats, node_value) (dotgraph.rs:430-532)."""
        max_label = C.c_uint32(0)
        check(lib.gb_node_label_index(self._g, C.byref(max_label), None, None))
        offsets = np.empty(max_label.value + 2, np.uint32)
        nodes = np.empty(self.node_count(), np.uint32)
        check(lib.gb_node_label_index(self._g, None, _ptr(offsets), _ptr(nodes)))
        return NodeLabelIndex(offsets, nodes)

    def neighbor_label_frequencies(self) -> NeighborLabelFrequencies:
        """NeighborLabelFrequencies::from_graph (dotgraph.rs:367-427), computed on the device."""
        cap = int(self._info.target_count)
        offsets = np.empty(self.node_count() + 1, np.uint32)
        labels = np.empty(max(cap, 1), np.uint32)
        counts = np.empty(max(cap, 1), np.uint32)

        def go():
            check(lib.gb_neighbor_label_frequencies(self._g, _ptr(offsets), _ptr(labels), _ptr(counts)))
        _, micros = _timed(go)
        pairs = int(offsets[-1])
        return NeighborLabelFrequencies(offsets, labels[:pairs].copy(), counts[:pairs].copy(), micros,
                                        self.last_timing()["total_ms"])

    def global_triangle_count(self) -> TriangleCountResult:
        """global_triangle_count(&graph) (triangle_count.rs:22-86)."""
        tri = C.c_uint64(0)

        def go():
            check(lib.gb_triangle_count(self._g, C.byref(tri)))
        _, micros = _timed(go)
        return TriangleCountResult(int(tri.value), micros)


# ---- adjacency-list graphs (crates/builder/src/graph/adj_list.rs) ----------------------------------------
def _batch_arrays(src, dst, values, with_values: bool):
    """Host edge arrays of add_edges as contiguous uint32 / float32."""
    s = np.asarray(src)
    d = np.asarray(dst)
    for a in (s, d):
        if a.ndim != 1:
            raise ValueError("src and dst must be 1-D arrays")
        if a.dtype != np.uint32 and (not np.issubdtype(a.dtype, np.integer)
                                     or (a.size and (a.min() < 0 or a.max() > 0xFFFFFFFF))):
            raise TypeError("node ids must be 32-bit unsigned integers")
    if len(s) != len(d):
        raise ValueError("src and dst must have the same length")
    w = None
    if with_values:
        if values is None:
            raise ValueError("the graph carries edge values: add_edges needs values")
        w = np.ascontiguousarray(values, dtype=np.float32)
        if w.ndim != 1 or len(w) != len(s):
            raise ValueError("values must have one entry per edge")
    elif values is not None:
        raise ValueError("the graph carries no edge values")
    return np.ascontiguousarray(s, np.uint32), np.ascontiguousarray(d, np.uint32), w


class _ALGraph:
    """Owns a gb_algraph*: adjacency lists on the device that take new edges.  Neighbour accessors return owned
    copies, because rows move when edges are added.  The algorithms run on a snapshot (to_graph()) that is kept
    until the next add_edges."""
    _KIND = _capi.KIND_DIRECTED
    _SNAPSHOT = None  # DiGraph / Graph

    def __init__(self, raw_ptr, load_micros=0, layout=None, values=False):
        self._g = raw_ptr
        self.load_micros = int(load_micros)
        self.layout = layout
        self._values = bool(values)
        self._lock = threading.Lock()
        self._version = 0
        self._snap = (None, None)

    def __del__(self):
        g, self._g = getattr(self, "_g", None), None
        if g:
            try:
                lib.gb_algraph_free(g)
            except Exception:  # interpreter shutdown
                pass

    # -- construction --
    @classmethod
    def _make(cls, fn, *args, layout=None, values=False):
        out = C.c_void_p()
        _, micros = _timed(lambda: check(fn(*args, C.byref(out))))
        return cls(out, micros, layout if layout is not None else Layout.Unsorted, values)

    @classmethod
    def from_numpy(cls, arr, layout=None, weights=None, node_count: int = 0):
        """From an (m, 2) array of edges (DirectedALGraph / UndirectedALGraph From<(E, CsrLayout)>, adj_list.rs:
        406-450, 559-595); weights: one f32 value per edge (EV = f32).  node_count 0 means max id + 1."""
        src, dst = _edges_from_numpy(arr)
        w = None if weights is None else np.ascontiguousarray(weights, dtype=np.float32)
        if w is not None and (w.ndim != 1 or len(w) != len(src)):
            raise ValueError("weights must have one entry per edge")
        return cls._make(lib.gb_algraph_from_edges_u32, _device, cls._KIND, _ptr(src), _ptr(dst), _ptr(w), len(src),
                         int(node_count), _layout_value(layout), int(w is not None), layout=layout,
                         values=w is not None)

    @classmethod
    def from_torch(cls, src, dst, weights=None, node_count: int = 0, layout=None):
        """From contiguous 1-D CUDA tensors on the graph's device (ids int32 or int64, weights float32)."""
        s, d, w, m, stream = _torch_edges(src, dst, weights)
        return cls._make(lib.gb_algraph_from_device_edges_u32, _device, cls._KIND, s.data_ptr(), d.data_ptr(),
                         None if w is None else w.data_ptr(), m, int(node_count), _layout_value(layout),
                         int(w is not None), stream.cuda_stream, layout=layout, values=w is not None)

    @classmethod
    def load(cls, path, layout=None, file_format=FileFormat.Graph500):
        """A Graph500 or text edge-list file, streamed to the device and parsed there."""
        p, fmt, lay = _load_args(path, file_format, layout)
        return cls._make(lib.gb_algraph_load_u32, _device, cls._KIND, p, fmt, lay, 0, layout=layout)

    @classmethod
    def load_weighted(cls, path, layout=None):
        """A weighted text edge list `<src> <dst> <f32>` (EV = f32)."""
        p, fmt, lay = _load_args(path, FileFormat.EdgeList, layout)
        return cls._make(lib.gb_algraph_load_u32, _device, cls._KIND, p, fmt, lay, 1, layout=layout, values=True)

    # -- accessors --
    def _info(self):
        info = _capi.GraphInfo()
        check(lib.gb_algraph_get_info(self._g, C.byref(info)))
        return info

    def node_count(self) -> int:
        return int(self._info().node_count)

    def edge_count(self) -> int:
        return int(self._info().edge_count)

    def device_bytes(self) -> int:
        return int(self._info().device_bytes)

    def has_values(self) -> bool:
        return self._values

    def load_info(self) -> dict:
        info = _capi.LoadInfo()
        check(lib.gb_algraph_load_info(self._g, C.byref(info)))
        return info.as_dict()

    def last_batch(self) -> dict:
        """What the last add_edges did: entries inserted, rows touched and moved, compactions, device times."""
        info = _capi.AlBatchInfo()
        check(lib.gb_algraph_last_batch(self._g, C.byref(info)))
        return info.as_dict()

    def _degree(self, which: int, node: int) -> int:
        ln = C.c_uint32(0)
        self._check_node(node)
        check(lib.gb_algraph_copy_row(self._g, which, node, 0, None, None, C.byref(ln)))
        return int(ln.value)

    def _check_node(self, node: int) -> None:
        n = self.node_count()
        if not 0 <= node < n:
            raise IndexError(f"node {node} out of range for a graph with {n} nodes")

    def _row(self, which: int, node: int, with_values: bool = False):
        if with_values and not self._values:
            raise ValueError("the graph carries no edge values")
        cap = self._degree(which, node)
        while True:  # another thread may add edges between the two calls
            tgt = np.empty(cap, np.uint32)
            val = np.empty(cap, np.float32) if with_values else None
            ln = C.c_uint32(0)
            check(lib.gb_algraph_copy_row(self._g, which, node, cap, _ptr(tgt), _ptr(val), C.byref(ln)))
            if ln.value <= cap:
                n = int(ln.value)
                return (tgt[:n], val[:n]) if with_values else tgt[:n]
            cap = int(ln.value)

    def _csr(self, which: int, with_values: bool = False):
        """(offsets, targets[, values]) of one list as a compacted CSR."""
        if with_values and not self._values:
            raise ValueError("the graph carries no edge values")
        off = np.empty(self.node_count() + 1, np.uint32)
        count = C.c_uint64(0)
        check(lib.gb_algraph_copy_csr(self._g, which, 0, _ptr(off), None, None, C.byref(count)))
        while True:  # the arrays are filled only when they can hold the list as it is at the call
            m = int(count.value)
            tgt = np.empty(max(m, 1), np.uint32)
            val = np.empty(max(m, 1), np.float32) if with_values else None
            check(lib.gb_algraph_copy_csr(self._g, which, m, _ptr(off), _ptr(tgt), _ptr(val), C.byref(count)))
            if int(count.value) <= m:
                k = int(count.value)
                return (off, tgt[:k], val[:k]) if with_values else (off, tgt[:k])

    # -- mutation --
    def add_edge(self, source: int, target: int, value=None) -> None:
        """EdgeMutation::add_edge / EdgeMutationWithValues::add_edge_with_value (adj_list.rs:381-404, 534-557).
        A missing node raises ValueError: node "<id>" does not exist in the graph."""
        if (value is None) == self._values:
            raise ValueError("add_edge needs a value exactly when the graph carries edge values")
        for x in (source, target):
            if not 0 <= int(x) <= 0xFFFFFFFF:
                raise ValueError(f'node "{int(x)}" does not exist in the graph')
        self.add_edges([source], [target], None if value is None else [value])

    def add_edges(self, src, dst, values=None) -> None:
        """len(src) add_edge calls in array order, as one device batch: all or nothing.  numpy arrays (or lists)
        or CUDA tensors on the graph's device (ids int32 / int64, values float32)."""
        try:
            import torch
            on_device = isinstance(src, torch.Tensor)
        except ImportError:
            on_device = False
        if on_device:
            if (values is None) == self._values:
                raise ValueError("add_edges needs values exactly when the graph carries edge values")
            s, d, w, m, stream = _torch_edges(src, dst, values)
            check(lib.gb_algraph_add_device_edges_u32(self._g, s.data_ptr(), d.data_ptr(),
                                                      None if w is None else w.data_ptr(), m, stream.cuda_stream))
        else:
            s, d, w = _batch_arrays(src, dst, values, self._values)
            check(lib.gb_algraph_add_edges_u32(self._g, _ptr(s), _ptr(d), _ptr(w), len(s)))
        with self._lock:
            self._version += 1
            self._snap = (None, None)

    # -- snapshot and algorithms --
    def to_graph(self):
        """A fresh, immutable DiGraph / Graph with this graph's rows (and out values), byte for byte."""
        return _construct(self._SNAPSHOT, lib.gb_algraph_to_graph, self._g)

    def _snapshot(self):
        with self._lock:
            version, snap = self._snap
            if snap is None or version != self._version:
                snap = self.to_graph()
                self._snap = (self._version, snap)
            return snap

    def __repr__(self):
        return f"{type(self).__name__} {{ node_count: {self.node_count()}, edge_count: {self.edge_count()} }}"


class DirectedALGraph(_ALGraph):
    """Device twin of DirectedALGraph<u32, (), EV> (crates/builder/src/graph/adj_list.rs:279-450), EV = () or
    f32: an out-list and an in-list that take new edges."""
    _KIND = _capi.KIND_DIRECTED
    _SNAPSHOT = DiGraph

    def out_degree(self, node: int) -> int:
        return self._degree(_capi.CSR_OUT, node)

    def in_degree(self, node: int) -> int:
        return self._degree(_capi.CSR_IN, node)

    def out_neighbors(self, node: int) -> np.ndarray:
        return self._row(_capi.CSR_OUT, node)

    def in_neighbors(self, node: int) -> np.ndarray:
        return self._row(_capi.CSR_IN, node)

    def out_neighbors_with_values(self, node: int):
        """(targets, values) of out-row `node` (DirectedNeighborsWithValues, adj_list.rs:355-369)."""
        return self._row(_capi.CSR_OUT, node, True)

    def in_neighbors_with_values(self, node: int):
        return self._row(_capi.CSR_IN, node, True)

    def csr(self, which: str = "out", with_values: bool = False):
        return self._csr(_capi.CSR_OUT if which == "out" else _capi.CSR_IN, with_values)

    def page_rank(self, *, max_iterations: int = PageRankConfig.DEFAULT_MAX_ITERATIONS,
                  tolerance: float = PageRankConfig.DEFAULT_TOLERANCE,
                  damping_factor: float = PageRankConfig.DEFAULT_DAMPING_FACTOR, mode: str = "auto") -> PageRankResult:
        """DiGraph.page_rank on the snapshot."""
        return self._snapshot().page_rank(max_iterations=max_iterations, tolerance=tolerance,
                                          damping_factor=damping_factor, mode=mode)

    def wcc(self, *, chunk_size: int = WccConfig.DEFAULT_CHUNK_SIZE,
            neighbor_rounds: int = WccConfig.DEFAULT_NEIGHBOR_ROUNDS,
            sampling_size: int = WccConfig.DEFAULT_SAMPLING_SIZE) -> WccResult:
        """DiGraph.wcc on the snapshot."""
        return self._snapshot().wcc(chunk_size=chunk_size, neighbor_rounds=neighbor_rounds,
                                    sampling_size=sampling_size)

    def delta_stepping(self, *, start_node: int, delta: float) -> SsspResult:
        """DiGraph.delta_stepping on the snapshot; needs f32 edge values."""
        return self._snapshot().delta_stepping(start_node=start_node, delta=delta)


class UndirectedALGraph(_ALGraph):
    """Device twin of UndirectedALGraph<u32, (), EV> (adj_list.rs:452-595), EV = () or f32: one list that takes
    new edges."""
    _KIND = _capi.KIND_UNDIRECTED
    _SNAPSHOT = Graph

    def degree(self, node: int) -> int:
        return self._degree(_capi.CSR_UNDIRECTED, node)

    def neighbors(self, node: int) -> np.ndarray:
        return self._row(_capi.CSR_UNDIRECTED, node)

    def neighbors_with_values(self, node: int):
        """(targets, values) of row `node` (UndirectedNeighborsWithValues, adj_list.rs:512-522)."""
        return self._row(_capi.CSR_UNDIRECTED, node, True)

    def csr(self, with_values: bool = False):
        return self._csr(_capi.CSR_UNDIRECTED, with_values)

    def global_triangle_count(self) -> TriangleCountResult:
        """Graph.global_triangle_count on the snapshot."""
        return self._snapshot().global_triangle_count()


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


def wcc_file(path, file_format=FileFormat.Graph500, *, chunk_size: int = WccConfig.DEFAULT_CHUNK_SIZE,
             neighbor_rounds: int = WccConfig.DEFAULT_NEIGHBOR_ROUNDS,
             sampling_size: int = WccConfig.DEFAULT_SAMPLING_SIZE) -> WccResult:
    """wcc of a graph file in one pass, without building the graph (gb_wcc_file_u32): the file is read as
    DiGraph.load(path, file_format=file_format) reads it, and each chunk's edges are linked on the device as soon as
    they are decoded, so no edge array or CSR is ever held and Graph500, edge-list and DotGraph files of 2^32 - 1
    edges or more are accepted.  The labels are those of DiGraph.load(...).wcc() (the minimum node id of each
    component), and every other file fails as the load fails, with FileNotFoundError or the same ValueError.  The
    config is checked and otherwise ignored; wcc_file_info() describes the call."""
    p, fmt, _ = _load_args(path, file_format, None)
    cfg = _capi.WccConfig(int(chunk_size), int(neighbor_rounds), int(sampling_size))
    h = C.c_void_p()

    def go():
        check(lib.gb_wcc_file_u32(_device, p, fmt, C.byref(cfg), C.byref(h)))
        try:
            n = C.c_uint32(0)
            check(lib.gb_components_node_count(h, C.byref(n)))
            comp = np.empty(n.value, np.uint32)
            check(lib.gb_components_copy(h, _ptr(comp)))
        finally:
            lib.gb_components_free(h)
        return comp
    comp, micros = _timed(go)
    return WccResult(comp, micros)


def wcc_file_info() -> dict:
    """Statistics of the calling thread's last wcc_file (all zero after a failed call): file_bytes, chunks, edges,
    h2d_bytes, device_bytes (the most the call held on the device at once), node_count and total_ms (CUDA-event time
    from the first copy to the last link)."""
    info = _capi.WccFileStats()
    check(lib.gb_wcc_file_info(C.byref(info)))
    return info.as_dict()


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


def sssp_csr(offsets, targets, weights, *, start_node: int, delta: float) -> SsspResult:
    """delta_stepping (sssp.rs:38-102) of a host weighted out-CSR without a resident twin and without its
    transpose: the distances DiGraph.from_csr(...).delta_stepping() gives for the same arrays, bit for bit.  The
    offsets are uploaded first; the targets and their f32 weights follow in row-aligned chunks, from the start's
    chunk on, and the bucket loop runs while they land: a queued vertex whose row is not on the device yet is
    parked and relaxed once it is.  The CSR is freed before the call returns.  Arrays are used as given: pass
    pinned contiguous arrays (uint32 offsets and targets, float32 weights) to overlap the passes with the copy.
    `weights` may be None only when there are no edges.  `info` on the result holds the call's chunk count, h2d
    bytes, parked vertices, pass counts and device times."""
    off, tgt = _host_csr_arrays(offsets, targets, "sssp_csr", "out")
    w = None
    if weights is not None:
        w = np.asarray(weights)
        if w.dtype != np.float32 or not w.flags.c_contiguous:
            raise TypeError("sssp_csr needs contiguous float32 weights")
        if w.ndim != 1 or len(w) < int(off[-1]):
            raise ValueError(f"weights hold {len(w)} entries but the offsets end at {int(off[-1])}")
    if start_node < 0:
        raise ValueError("start_node must be non-negative")
    cfg = _capi.SsspConfig(int(start_node), float(delta))
    dist = np.empty(len(off) - 1, np.float32)

    def go():
        check(lib.gb_sssp_csr_u32(_device, len(off) - 1, _ptr(off), _ptr(tgt) if len(tgt) else None,
                                  _ptr(w) if w is not None and len(w) else None, C.byref(cfg), _ptr(dist)))
    _, micros = _timed(go)
    info = _capi.SsspCsrInfo()
    check(lib.gb_sssp_csr_info(C.byref(info)))
    return SsspResult(dist, micros, info.as_dict())
