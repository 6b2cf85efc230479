"""Graph construction (graph_b200/csrc/graph.cu): host and device edge arrays share the argument checks, the
node_count inference and the id check, and every host CSR reaches the device through one upload that checks
its offsets and targets.  The same malformed input must fail the same way whichever entry point takes it."""
import ctypes as C

import numpy as np
import pytest

import graph_b200 as gb
from graph_b200 import _capi
from graph_b200._capi import lib

pytestmark = pytest.mark.gpu

# a 6-node ring; the out offsets have the ring's edge count, but row 1 ends before it starts
IN_OFF = np.arange(7, dtype=np.uint32)
IN_TGT = np.array([5, 0, 1, 2, 3, 4], np.uint32)
BAD_OUT_OFF = np.array([0, 2, 1, 3, 4, 6, 6], np.uint32)


def test_for_page_rank_rejects_non_monotone_out_offsets():
    with pytest.raises(ValueError, match="out offsets are not monotone"):
        gb.DiGraph.for_page_rank(IN_OFF, IN_TGT, BAD_OUT_OFF)


@pytest.mark.parametrize("min_edges", [None, "0"], ids=["resident", "streamed"])
def test_page_rank_csr_rejects_non_monotone_out_offsets(monkeypatch, min_edges):
    """Below GB_PR_FEED_MIN_EDGES the one-shot entry uploads the whole CSR first; at 0 it streams the targets.
    Both must reject the same out offsets."""
    monkeypatch.delenv("GB_PR_FEED_CHUNKS", raising=False)
    if min_edges is None:
        monkeypatch.delenv("GB_PR_FEED_MIN_EDGES", raising=False)
    else:
        monkeypatch.setenv("GB_PR_FEED_MIN_EDGES", min_edges)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    cfg = _capi.PageRankConfig(5, 0.0, 0.85, _capi.PR_JACOBI)
    scores = np.empty(len(IN_OFF) - 1, np.float32)
    it, err = C.c_uint64(0), C.c_double(0.0)
    st = lib.gb_page_rank_csr_u32(0, len(IN_OFF) - 1, P(IN_OFF), P(IN_TGT), P(BAD_OUT_OFF), C.byref(cfg), P(scores),
                                  C.byref(it), C.byref(err))
    assert st == _capi.GB_ERR_INVALID
    assert b"out offsets are not monotone" in lib.gb_last_error()


def host_and_device_error(cls, edges, node_count):
    import torch
    e = np.asarray(edges, np.uint32).reshape(-1, 2)
    t = torch.from_numpy(e.astype(np.int64)).cuda()
    errs = []
    for make in (lambda: cls.from_numpy(e, node_count=node_count),
                 lambda: cls.from_torch(t[:, 0].contiguous(), t[:, 1].contiguous(), node_count=node_count)):
        with pytest.raises(Exception) as ei:
            make()
        errs.append((type(ei.value), str(ei.value)))
    assert errs[0] == errs[1]
    return errs[0]


@pytest.mark.parametrize("cls", [gb.DiGraph, gb.Graph], ids=lambda c: c.__name__)
@pytest.mark.parametrize("edges,node_count,message", [
    ([], 0, "cannot infer node_count from an empty edge list"),
    ([[0, 4294967295]], 0, "node id 2^32-1 leaves no room for node_count"),
    ([[0, 1], [2, 7]], 4, "1 edge endpoints are >= node_count 4"),
], ids=["empty", "max_id", "beyond_node_count"])
def test_host_and_device_edges_fail_alike(cls, edges, node_count, message):
    t, msg = host_and_device_error(cls, edges, node_count)
    assert t is ValueError and msg == message
