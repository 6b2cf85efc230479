"""graph_b200.flight — the Arrow Flight front end of the reference (crates/server) over the H100 hot path.

What a client of the reference's server sees is kept: the six JSON actions of actions.rs:28-55
(`create`, `list`, `remove`, `compute`, `to_relabeled`, `to_undirected`), `do_put` with a
`CreateGraphCommand` descriptor and two int64 columns (server.rs:110-176), `do_get` with a JSON
`PropertyId` ticket that streams the stored property in record batches of 10 000 rows (server.rs:33,
catalog.rs:262-287), the result documents (`CreateActionResult`, `MutateResult{property_id, algo_result}`,
…) and the error classes (invalid argument for an algorithm on the wrong kind of graph, not found for an
unknown graph or property).  The reference's example clients (crates/server/examples/*.py) run unchanged.

How it is built differs: one synchronous dispatcher over an ENGINE object with eight methods.  The default
engine is this package (every graph lives in HBM, every algorithm is a C-ABI call); the catalog and the
property store are two dicts behind one lock.  Node ids are u32 on the device: a `do_put` stream with ids
>= 2^32 is rejected as an invalid argument (the reference holds u64 ids).

    python -m graph_b200.flight [host] [port]        # main.rs: defaults ::1 / 50051; here 127.0.0.1 / 50051
"""
from __future__ import annotations

import json
import threading
import time

import numpy as np
import pyarrow as pa
import pyarrow.flight as fl

CHUNK_SIZE = 10_000  # rows per record batch of a stored property (server.rs:33)

ACTION_TYPES = [  # actions.rs:28-55
    ("create", "Create a new graph."),
    ("list", "List all graphs."),
    ("remove", "Remove a graph."),
    ("compute", "Compute a graph algorithm on a graph."),
    ("to_relabeled", "Relabels the node ids of a graph in degree-descending order"),
    ("to_undirected", "Converts a directed graph to an undirected graph"),
]
FILE_FORMATS = ("EdgeList", "EdgeListWeighted", "Graph500")
LAYOUTS = ("Sorted", "Unsorted", "Deduplicated")
ORIENTATIONS = ("Directed", "Undirected")


class JsonError(fl.FlightInternalError):
    """serde_json failures surface as Status::internal("JsonError: ...") (actions.rs:318-320)."""


def _json(body, what: str) -> dict:
    try:
        doc = json.loads(bytes(body).decode("utf-8"))
    except Exception as e:  # noqa: BLE001
        raise JsonError(f"JsonError: {e}") from None
    if not isinstance(doc, dict):
        raise JsonError(f"JsonError: expected a JSON object for {what}")
    return doc


def _field(doc: dict, name: str, kinds, default=None, choices=None):
    if name not in doc:
        if default is not None:
            return default
        raise JsonError(f"JsonError: missing field `{name}`")
    v = doc[name]
    if isinstance(v, bool) or not isinstance(v, kinds):
        raise JsonError(f"JsonError: invalid type for field `{name}`")
    if choices is not None and v not in choices:
        raise JsonError(f"JsonError: unknown variant `{v}`, expected one of {', '.join(choices)}")
    return v


def _millis(t0: float) -> int:
    return int((time.perf_counter() - t0) * 1000)


class B200Engine:
    """The algorithms and graph operations the front end needs, on the device twin (graph_b200)."""

    def __init__(self):
        import graph_b200 as gb  # loads libgraph_b200.so; constructors fail loudly without a CUDA device
        self.gb = gb

    def _layout(self, name: str):
        return getattr(self.gb.Layout, name)

    # a catalog entry is (kind, handle); kind is the reference's GraphType display string (catalog.rs:21-35)
    def load(self, path: str, file_format: str, orientation: str, layout: str):
        gb = self.gb
        weighted = file_format == "EdgeListWeighted"
        if orientation == "Directed":
            if weighted:
                return "directed+weighted", gb.DiGraph.load_weighted(path, self._layout(layout))
            fmt = gb.FileFormat.Graph500 if file_format == "Graph500" else gb.FileFormat.EdgeList
            return "directed", gb.DiGraph.load(path, self._layout(layout), fmt)
        if weighted:
            return "undirected+weighted", gb.Graph.load_weighted(path, self._layout(layout))
        fmt = gb.FileFormat.Graph500 if file_format == "Graph500" else gb.FileFormat.EdgeList
        return "undirected", gb.Graph.load(path, self._layout(layout), fmt)

    def from_edges(self, src: np.ndarray, dst: np.ndarray, orientation: str, layout: str):
        edges = np.stack([src, dst], 1)
        if orientation == "Directed":
            return "directed", self.gb.DiGraph.from_numpy(edges, self._layout(layout))
        return "undirected", self.gb.Graph.from_numpy(edges, self._layout(layout))

    def page_rank(self, g, max_iterations: int, tolerance: float, damping_factor: float):
        r = g.page_rank(max_iterations=max_iterations, tolerance=tolerance, damping_factor=damping_factor)
        return r.scores(), int(r.ran_iterations), float(r.error)

    def wcc(self, g, chunk_size: int, neighbor_rounds: int, sampling_size: int) -> np.ndarray:
        return g.wcc(chunk_size=chunk_size, neighbor_rounds=neighbor_rounds, sampling_size=sampling_size).components()

    def sssp(self, g, start_node: int, delta: float) -> np.ndarray:
        return g.delta_stepping(start_node=start_node, delta=delta).distances()

    def triangle_count(self, g) -> int:
        return int(g.global_triangle_count().triangles)

    def make_degree_ordered(self, g) -> None:
        g.make_degree_ordered()

    def to_undirected(self, g, layout: str):
        # a "directed+weighted" twin becomes an "undirected+weighted" one with its values (server.rs:390-391)
        return g.to_undirected(self._layout(layout), weights=bool(g._info.has_weights))


class GraphFlightServer(fl.FlightServerBase):
    """FlightServiceImpl of server.rs:36-52: a graph catalog and a property store behind Flight."""

    def __init__(self, location: str = "grpc://127.0.0.1:50051", engine=None, **kwargs):
        super().__init__(location, **kwargs)
        self.engine = engine if engine is not None else B200Engine()
        self._lock = threading.RLock()
        self._graphs: dict[str, tuple[str, object]] = {}       # GraphCatalog (catalog.rs:146-205)
        self._properties: dict[tuple[str, str], pa.Table] = {}  # PropertyStore (catalog.rs:246-265)

    # ---- catalog -----------------------------------------------------------------------------------
    def _get(self, name: str):
        with self._lock:
            if name not in self._graphs:
                raise KeyError(f"Graph with name '{name}' not found")  # Status::not_found, catalog.rs:200-205
            return self._graphs[name]

    def _info(self, name: str, kind: str, g) -> dict:
        return {"graph_name": name, "graph_type": kind, "node_count": int(g.node_count()),
                "edge_count": int(g.edge_count())}

    # ---- Flight surface ----------------------------------------------------------------------------
    def list_actions(self, context):
        return ACTION_TYPES

    def do_action(self, context, action):
        kind = action.type
        body = action.body.to_pybytes() if action.body is not None else b""
        handlers = {"create": self._create, "list": self._list, "remove": self._remove, "compute": self._compute,
                    "to_relabeled": self._to_relabeled, "to_undirected": self._to_undirected}
        if kind not in handlers:
            raise pa.ArrowInvalid(f"Unknown action type: {kind}")  # actions.rs:85-87
        result = handlers[kind](body)
        return iter([fl.Result(json.dumps(result).encode("utf-8"))])

    def do_get(self, context, ticket):
        doc = _json(ticket.ticket, "PropertyId")
        key = (_field(doc, "graph_name", str), _field(doc, "property_key", str))
        with self._lock:
            if key not in self._properties:
                raise KeyError(f"Property Id not found: PropertyId {{ graph_name: {key[0]!r}, property_key: {key[1]!r} }}")
            table = self._properties[key]
        return fl.GeneratorStream(table.schema, iter(table.to_batches(max_chunksize=CHUNK_SIZE)))

    def do_put(self, context, descriptor, reader, writer):
        if descriptor.descriptor_type != fl.DescriptorType.CMD:
            raise pa.ArrowInvalid(f"Expected command, got {descriptor.descriptor_type}")  # actions.rs:150-163
        cmd = _json(descriptor.command, "CreateGraphCommand")
        name = _field(cmd, "graph_name", str)
        _field(cmd, "edge_count", int)  # a capacity hint in the reference (server.rs:134)
        layout = _field(cmd, "csr_layout", str, "Unsorted", LAYOUTS)
        orientation = _field(cmd, "orientation", str, "Directed", ORIENTATIONS)
        t0 = time.perf_counter()
        table = reader.read_all()
        if table.num_columns < 2:
            raise pa.ArrowInvalid("expected two int64 columns: source ids, target ids")
        cols = []
        for c in (0, 1):
            a = table.column(c).combine_chunks()
            if not pa.types.is_int64(a.type) or a.null_count:
                raise pa.ArrowInvalid("expected two non-null int64 columns: source ids, target ids")
            v = a.to_numpy(zero_copy_only=False) if len(a) else np.empty(0, np.int64)
            if len(v) and (v.min() < 0 or v.max() >= 1 << 32):
                raise pa.ArrowInvalid("node ids must fit u32 on the device twin")
            cols.append(np.ascontiguousarray(v, dtype=np.uint32))
        kind, g = self.engine.from_edges(cols[0], cols[1], orientation, layout)
        result = {"node_count": int(g.node_count()), "edge_count": int(g.edge_count()), "create_millis": _millis(t0)}
        with self._lock:
            self._graphs[name] = (kind, g)
        writer.write(pa.py_buffer(json.dumps(result).encode("utf-8")))

    # ---- actions -----------------------------------------------------------------------------------
    def _create(self, body) -> dict:  # create_graph, server.rs:295-322
        cfg = _json(body, "CreateGraphFromFileConfig")
        name = _field(cfg, "graph_name", str)
        file_format = _field(cfg, "file_format", str, choices=FILE_FORMATS)
        path = _field(cfg, "path", str)
        layout = _field(cfg, "csr_layout", str, "Unsorted", LAYOUTS)
        orientation = _field(cfg, "orientation", str, "Directed", ORIENTATIONS)
        t0 = time.perf_counter()
        try:
            kind, g = self.engine.load(path, file_format, orientation, layout)
        except (OSError, ValueError) as e:
            raise fl.FlightInternalError(f"GraphError: {e}") from None  # catalog.rs:141-143
        result = {"node_count": int(g.node_count()), "edge_count": int(g.edge_count()), "create_millis": _millis(t0)}
        with self._lock:
            self._graphs[name] = (kind, g)
        return result

    def _list(self, body) -> dict:
        with self._lock:
            return {"graph_infos": [self._info(n, k, g) for n, (k, g) in self._graphs.items()]}

    def _remove(self, body) -> dict:
        name = _field(_json(body, "RemoveGraphConfig"), "graph_name", str)
        with self._lock:
            kind, g = self._get(name)
            info = self._info(name, kind, g)
            del self._graphs[name]
        return info

    def _to_relabeled(self, body) -> dict:  # server.rs:341-368: undirected, unweighted graphs only
        name = _field(_json(body, "ToRelabeledConfig"), "graph_name", str)
        with self._lock:
            kind, g = self._get(name)
            if kind != "undirected":
                raise pa.ArrowInvalid("Relabelling directed graphs is not supported.")
            t0 = time.perf_counter()
            self.engine.make_degree_ordered(g)
            return {"to_relabeled_millis": _millis(t0)}

    def _to_undirected(self, body) -> dict:  # server.rs:370-407
        cfg = _json(body, "ToUndirectedConfig")
        name = _field(cfg, "graph_name", str)
        layout = _field(cfg, "csr_layout", str, "Unsorted", LAYOUTS)
        with self._lock:
            kind, g = self._get(name)
            t0 = time.perf_counter()
            if kind.startswith("directed"):
                self._graphs[name] = (kind.replace("directed", "undirected", 1), self.engine.to_undirected(g, layout))
            return {"to_undirected_millis": _millis(t0)}

    def _compute(self, body) -> dict:  # server.rs:214-262
        cfg = _json(body, "ComputeConfig")
        name = _field(cfg, "graph_name", str)
        key = _field(cfg, "property_key", str)
        if "algorithm" not in cfg:
            raise JsonError("JsonError: missing field `algorithm`")
        algo = cfg["algorithm"]
        if isinstance(algo, str):  # serde's unit variant: "TriangleCount"
            algo = {algo: None}
        if not isinstance(algo, dict) or len(algo) != 1:
            raise JsonError("JsonError: expected an externally tagged `Algorithm`")
        (variant, params), = algo.items()
        params = params if isinstance(params, dict) else {}
        kind, g = self._get(name)
        t0 = time.perf_counter()
        if variant == "PageRank":
            p = (_field(params, "max_iterations", int), float(_field(params, "tolerance", (int, float))),
                 float(_field(params, "damping_factor", (int, float))))
            if kind != "directed":
                raise pa.ArrowInvalid("Page Rank requires a directed graph")
            scores, iterations, error = self.engine.page_rank(g, *p)
            result = {"iterations": iterations, "error": error, "compute_millis": _millis(t0)}
            return self._mutate(name, key, "page_rank", pa.array(scores, pa.float32()), result)
        if variant == "TriangleCount":
            if kind != "undirected":
                raise pa.ArrowInvalid("Triangle count requires an undirected graph")
            tc = self.engine.triangle_count(g)
            return {"triangle_count": int(tc), "compute_millis": _millis(t0)}  # no property (server.rs:453-477)
        if variant == "Sssp":
            p = (_field(params, "start_node", int), float(_field(params, "delta", (int, float))))
            if kind != "directed+weighted":
                raise pa.ArrowInvalid("Sssp requires a directed, weighted graph")
            dist = self.engine.sssp(g, *p)
            return self._mutate(name, key, "distance", pa.array(dist, pa.float32()), {"compute_millis": _millis(t0)})
        if variant == "Wcc":
            p = (_field(params, "chunk_size", int), _field(params, "neighbor_rounds", int),
                 _field(params, "sampling_size", int))
            if kind != "directed":
                raise pa.ArrowInvalid("Wcc requires a directed graph")
            comp = np.asarray(self.engine.wcc(g, *p)).astype(np.uint64)
            return self._mutate(name, key, "component", pa.array(comp, pa.uint64()), {"compute_millis": _millis(t0)})
        raise JsonError(f"JsonError: unknown variant `{variant}`, expected one of PageRank, TriangleCount, Sssp, Wcc")

    def _mutate(self, name: str, key: str, column: str, values: pa.Array, algo_result: dict) -> dict:
        schema = pa.schema([pa.field(column, values.type, nullable=False)])
        with self._lock:
            self._properties[(name, key)] = pa.Table.from_arrays([values], schema=schema)
        return {"property_id": {"graph_name": name, "property_key": key}, "algo_result": algo_result}


def main(argv=None) -> None:
    import argparse
    ap = argparse.ArgumentParser(description="Graph Arrow Server (H100)")
    ap.add_argument("host", nargs="?", default="127.0.0.1")
    ap.add_argument("port", nargs="?", type=int, default=50051)
    a = ap.parse_args(argv)
    server = GraphFlightServer(f"grpc://{a.host}:{a.port}")
    print(f"Starting server at {a.host}:{server.port}", flush=True)
    server.serve()


if __name__ == "__main__":
    main()
