"""The Flight front end under parallel clients, with its default engine (the device twin).  gRPC serves the requests
on a thread pool and the server runs each algorithm outside its catalog lock, so requests on distinct graphs and on
one shared graph reach the library together, and `to_relabeled` rewrites a graph that TriangleCount requests are
counting.  That graph is Deduplicated: the reference's count on parallel edges and self-loops depends on the labels
(an RMAT-14 multigraph counts 21787594, 22471534 and 22471742 after none, one and two relabellings), a simple graph's
does not.  Every result and every stored property fetched with do_get must equal the serial request's, which is
checked against the oracle first.  The file name sorts last: it starts a gRPC server inside the test process."""
import json

import numpy as np
import pytest

import oracle
from thread_jobs import run_threads

pytestmark = pytest.mark.gpu

pa = pytest.importorskip("pyarrow")
fl = pytest.importorskip("pyarrow.flight")

CLIENTS = 7   # plus one that relabels the shared undirected graph
ROUNDS = 2
PAGE_RANK = {"PageRank": {"max_iterations": 20, "tolerance": 1e-4, "damping_factor": 0.85}}
WCC = {"Wcc": {"chunk_size": 16384, "neighbor_rounds": 2, "sampling_size": 1024}}


@pytest.fixture(scope="module")
def server():
    from graph_b200.flight import GraphFlightServer
    s = GraphFlightServer("grpc://127.0.0.1:0")
    yield s
    s.shutdown()


def act(client, kind, doc):
    return json.loads(next(client.do_action(fl.Action(kind, json.dumps(doc).encode()))).body.to_pybytes())


def prop(client, property_id) -> bytes:
    col = client.do_get(fl.Ticket(json.dumps(property_id).encode())).read_all().column(0)
    return col.to_numpy().tobytes()


@pytest.fixture(scope="module")
def inputs(tmp_path_factory, golden_dir):
    """name -> (path, file format, CSR layout, the oracle's CSRs of the file's edges in that layout)"""
    d = tmp_path_factory.mktemp("flight_threads")
    src, dst = oracle.rmat_edges(14, seed=11)
    w = oracle.rmat_weights(11, 0, len(src))
    np.savetxt(d / "rmat14.el", np.stack([src, dst], 1), fmt="%d")
    with open(d / "rmat14.wel", "w") as f:
        f.write("".join(f"{a} {b} {x:.9g}\n" for a, b, x in zip(src.tolist(), dst.tolist(), w.tolist())))
    out = {}
    for name, path, fmt, layout in (("example", golden_dir / "example.el", "EdgeList", "Sorted"),
                                    ("scale8", golden_dir / "scale_8.graph500", "Graph500", "Sorted"),
                                    ("rmat", d / "rmat14.el", "EdgeList", "Sorted"),
                                    ("rmat_dd", d / "rmat14.el", "EdgeList", "Deduplicated"),
                                    ("rmat_w", d / "rmat14.wel", "EdgeListWeighted", "Sorted")):
        raw = path.read_bytes()
        vals = None
        if fmt == "Graph500":
            s, t, n = oracle.graph500_decode(raw)
        elif fmt == "EdgeListWeighted":
            s, t, vals = oracle.edgelist_parse(raw, with_values=True)
            n = oracle.node_count(s, t)
        else:
            s, t = oracle.edgelist_parse(raw)
            n = oracle.node_count(s, t)
        lay = oracle.SORTED if layout == "Sorted" else oracle.DEDUPLICATED
        out[name] = (str(path), fmt, layout, {
            "out": oracle.csr_build(s, t, n, oracle.OUTGOING, lay, vals),
            "in": oracle.csr_build(s, t, n, oracle.INCOMING, lay),
            "und": oracle.csr_build(s, t, n, oracle.UNDIRECTED, lay)})
    return out


def create(client, graph, inp, orientation):
    path, fmt, layout, _ = inp
    act(client, "create", {"graph_name": graph, "file_format": fmt, "path": path, "csr_layout": layout,
                           "orientation": orientation})


def graphs_of(prefix, inputs):
    """(graph name, input, orientation) of every graph one client creates"""
    out = [(f"{prefix}{k}_d", k, "Directed") for k in inputs]
    out += [(f"{prefix}{k}_u", k, "Undirected") for k in inputs if k != "rmat_w"]
    return out


def requests(graph, key, inputs):
    """the compute requests a graph takes, as (label, property key or None, request)"""
    name, orientation = graph.rsplit("_", 1)
    k = name.split(":")[-1]
    if orientation == "u":
        return [("TriangleCount", None, {"graph_name": graph, "property_key": key + "tc",
                                         "algorithm": {"TriangleCount": None}})]
    if k == "rmat_w":
        off = inputs[k][3]["out"][0]
        start = int(np.argmax(np.diff(off.astype(np.int64))))
        return [("Sssp", key + "sssp", {"graph_name": graph, "property_key": key + "sssp",
                                        "algorithm": {"Sssp": {"start_node": start, "delta": 0.1}}})]
    return [("PageRank", key + "pr", {"graph_name": graph, "property_key": key + "pr", "algorithm": PAGE_RANK}),
            ("Wcc", key + "wcc", {"graph_name": graph, "property_key": key + "wcc", "algorithm": WCC})]


def result_of(client, label, req):
    """the deterministic part of a compute request's answer: its numbers and the stored property's bytes"""
    r = act(client, "compute", req)
    if label == "TriangleCount":
        return r["triangle_count"]
    got = prop(client, r["property_id"])
    if label == "PageRank":
        return r["algo_result"]["iterations"], r["algo_result"]["error"], got
    return got


def check_oracle(label, k, want, csrs):
    if label == "TriangleCount":
        assert want == oracle.triangle_count(*csrs["und"], threads=0)
    elif label == "Sssp":
        off, tgt, w = csrs["out"]
        start = int(np.argmax(np.diff(off.astype(np.int64))))
        assert want == oracle.sssp_bellman_ford(off, tgt, w, start).tobytes()
    elif label == "Wcc":
        assert want == oracle.wcc_min_label(*csrs["out"][:2]).astype(np.uint64).tobytes()
    else:
        scores, it, err = oracle.page_rank_seq(csrs["in"][0], csrs["in"][1], csrs["out"][0], 20, 1e-4, 0.85)
        assert want == (it, err, scores.tobytes()), k


def test_parallel_clients(server, inputs):
    url = f"grpc://127.0.0.1:{server.port}"
    main = fl.connect(url)
    # the serial answers, from graphs the main client creates
    want = {}
    for graph, k, orientation in graphs_of("serial:", inputs):
        create(main, graph, inputs[k], orientation)
        for label, _, req in requests(graph, "serial", inputs):
            want[(k, orientation, label)] = result_of(main, label, req)
            check_oracle(label, k, want[(k, orientation, label)], inputs[k][3])
    for graph, k, orientation in graphs_of("shared:", inputs):
        create(main, graph, inputs[k], orientation)

    clients = [fl.connect(url) for _ in range(CLIENTS + 1)]
    # every client creates its own graphs, all at once
    run_threads([[(f"create {g}", lambda c=clients[t], g=g, k=k, o=o: create(c, g, inputs[k], o))
                  for g, k, o in graphs_of(f"t{t}:", inputs)] for t in range(CLIENTS)], 1, seed=9)

    def compute_jobs(t):
        c = clients[t]
        jobs = []
        for prefix in (f"t{t}:", "shared:"):
            for graph, k, orientation in graphs_of(prefix, inputs):
                for label, _, req in requests(graph, f"t{t}", inputs):
                    w = want[(k, orientation, label)]
                    jobs.append((f"{label} on {graph}", lambda req=req, label=label, w=w:
                                 assert_eq(result_of(c, label, req), w)))
        return jobs

    relabel = clients[CLIENTS]
    relabel_jobs = [("to_relabeled shared:rmat_dd_u",
                     lambda: act(relabel, "to_relabeled", {"graph_name": "shared:rmat_dd_u"}))] * 6
    run_threads([compute_jobs(t) for t in range(CLIENTS)] + [relabel_jobs], ROUNDS, seed=10)
    # the relabelled graph still counts the same
    tc = act(main, "compute", {"graph_name": "shared:rmat_dd_u", "property_key": "tc", "algorithm": "TriangleCount"})
    assert tc["triangle_count"] == want[("rmat_dd", "Undirected", "TriangleCount")]
    for c in clients + [main]:
        c.close()


def assert_eq(got, want):
    assert got == want
