"""ctypes binding of libgraph_b200.so (include/graph_b200.h).  No CPU fallback: importing this
module fails loudly when the CUDA library has not been built."""
from __future__ import annotations

import ctypes as C
from pathlib import Path

_HERE = Path(__file__).resolve().parent
LIB_PATH = _HERE / "libgraph_b200.so"

GB_OK, GB_ERR_INVALID, GB_ERR_CUDA, GB_ERR_OOM, GB_ERR_UNSUPPORTED = range(5)
LAYOUT_UNSORTED, LAYOUT_SORTED, LAYOUT_DEDUPLICATED = 0, 1, 2
KIND_DIRECTED, KIND_UNDIRECTED = 0, 1
CSR_OUT, CSR_IN, CSR_UNDIRECTED = 0, 1, 2
PR_AUTO, PR_EXACT, PR_JACOBI = 0, 1, 2
WCC_INIT, WCC_SAMPLE, WCC_COMPRESS, WCC_MERGE, WCC_LINK_REMAINING = range(5)


class GraphInfo(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("node_count", C.c_uint32), ("edge_count", C.c_uint64),
                ("target_count", C.c_uint64), ("has_weights", C.c_uint32), ("device", C.c_int32),
                ("device_bytes", C.c_uint64)]


class PageRankConfig(C.Structure):
    _fields_ = [("max_iterations", C.c_uint64), ("tolerance", C.c_double),
                ("damping_factor", C.c_float), ("mode", C.c_uint32)]


class WccConfig(C.Structure):
    _fields_ = [("chunk_size", C.c_uint64), ("neighbor_rounds", C.c_uint64),
                ("sampling_size", C.c_uint64)]


class SsspConfig(C.Structure):
    _fields_ = [("start_node", C.c_uint64), ("delta", C.c_float)]


class Timing(C.Structure):
    _fields_ = [("total_ms", C.c_double), ("hot_kernel_ms", C.c_double),
                ("hot_kernel_launches", C.c_uint64), ("kernel_launches", C.c_uint64)]


class PrShardStats(C.Structure):
    _fields_ = [("rank", C.c_uint32), ("world", C.c_uint32), ("active_rows", C.c_uint32),
                ("local_rows", C.c_uint32), ("local_edges", C.c_uint64), ("block_edges", C.c_uint64),
                ("block_entries", C.c_uint32), ("hot_blocks", C.c_uint32), ("segments", C.c_uint64),
                ("groups", C.c_uint64), ("chunks", C.c_uint32), ("tasks", C.c_uint32),
                ("cut_segments", C.c_uint32), ("chunk_groups", C.c_uint32),
                ("launches_per_sweep", C.c_uint32), ("device_bytes", C.c_uint64),
                ("vblock_parts", C.c_uint32), ("vblock_pairs", C.c_uint64), ("vblock_edges", C.c_uint64),
                ("vblock_wide_steps", C.c_uint32), ("vblock_slots", C.c_uint64), ("vblock_sectors", C.c_uint32)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class PrPlanShape(C.Structure):
    _fields_ = [("hot_blocks", C.c_uint32), ("n_cb", C.c_uint32), ("n_fin", C.c_uint32),
                ("n_fin_warp", C.c_uint32), ("fin_u", C.c_uint32), ("fin_hub_ctas", C.c_uint32),
                ("grid_cb", C.c_uint32), ("grid_sell", C.c_uint32), ("grid_fin", C.c_uint32),
                ("n_mega", C.c_uint32), ("n_fix", C.c_uint32), ("fix_in_sell", C.c_uint32), ("dual", C.c_uint32),
                ("last_hot_block", C.c_uint32)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class LoadInfo(C.Structure):
    _fields_ = [("file_bytes", C.c_uint64), ("chunks", C.c_uint64), ("edges", C.c_uint64),
                ("fallback_lines", C.c_uint64), ("h2d_bytes", C.c_uint64)]

    def as_dict(self):
        return {k: int(getattr(self, k)) for k, _ in self._fields_}


class TcCsrInfo(C.Structure):
    _fields_ = [("chunks", C.c_uint64), ("chunk_entries", C.c_uint64), ("h2d_bytes", C.c_uint64),
                ("sorted_chunks", C.c_uint64), ("list_chunks", C.c_uint64), ("first_list_chunk", C.c_uint64),
                ("kernel_launches", C.c_uint64), ("pinned", C.c_uint32), ("reserved", C.c_uint32),
                ("upload_ms", C.c_double), ("total_ms", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


class SsspCsrInfo(C.Structure):
    _fields_ = [("chunks", C.c_uint64), ("chunk_entries", C.c_uint64), ("h2d_bytes", C.c_uint64),
                ("parked", C.c_uint64), ("unpark_rounds", C.c_uint64), ("passes", C.c_uint64),
                ("passes_before_last_landed", C.c_uint64), ("kernel_launches", C.c_uint64),
                ("pinned", C.c_uint32), ("start_chunk", C.c_uint32), ("upload_ms", C.c_double),
                ("total_ms", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class WccFileStats(C.Structure):
    _fields_ = [("file_bytes", C.c_uint64), ("chunks", C.c_uint64), ("edges", C.c_uint64),
                ("h2d_bytes", C.c_uint64), ("device_bytes", C.c_uint64), ("node_count", C.c_uint32),
                ("reserved", C.c_uint32), ("total_ms", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_ if k != "reserved"}


class LabelStatsInfo(C.Structure):
    _fields_ = [("max_degree", C.c_uint32), ("max_label", C.c_uint32), ("label_count", C.c_uint64),
                ("max_label_frequency", C.c_uint64)]


class AlBatchInfo(C.Structure):
    _fields_ = [("edges", C.c_uint64), ("inserted", C.c_uint64), ("touched_rows", C.c_uint64),
                ("relocated_rows", C.c_uint64), ("compactions", C.c_uint64), ("total_compactions", C.c_uint64),
                ("pool_entries", C.c_uint64), ("pool_used", C.c_uint64), ("total_ms", C.c_double),
                ("compaction_ms", C.c_double)]

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


class GraphB200Error(RuntimeError):
    """CUDA / allocation failure inside libgraph_b200."""


_P = C.c_void_p
_U32P = C.POINTER(C.c_uint32)
_F32P = C.POINTER(C.c_float)

# every symbol include/graph_b200.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "gb_abi_version": (C.c_int, []),
    "gb_last_error": (C.c_char_p, []),
    "gb_device_count": (C.c_int, []),
    "gb_set_profiling": (None, [C.c_int]),
    "gb_digraph_from_csr_u32": (C.c_int, [C.c_int, C.c_uint32, _P, _P, _P, _P, _P, C.POINTER(_P)]),
    "gb_graph_from_csr_u32": (C.c_int, [C.c_int, C.c_uint32, _P, _P, C.POINTER(_P)]),
    "gb_digraph_from_edges_u32": (C.c_int, [C.c_int, _P, _P, _P, C.c_uint64, C.c_uint32, C.c_int, C.POINTER(_P)]),
    "gb_graph_from_edges_u32": (C.c_int, [C.c_int, _P, _P, C.c_uint64, C.c_uint32, C.c_int, C.POINTER(_P)]),
    "gb_graph_from_weighted_edges_u32": (C.c_int, [C.c_int, _P, _P, _P, C.c_uint64, C.c_uint32, C.c_int,
                                                   C.POINTER(_P)]),
    "gb_digraph_rmat": (C.c_int, [C.c_int, C.c_uint32, C.c_uint32, C.c_uint64, C.c_int, C.c_int, C.POINTER(_P)]),
    "gb_graph_rmat": (C.c_int, [C.c_int, C.c_uint32, C.c_uint32, C.c_uint64, C.c_int, C.POINTER(_P)]),
    "gb_rmat_edges": (C.c_int, [C.c_int, C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint64, _P, _P]),
    "gb_graph500_decode": (C.c_int, [_P, C.c_uint64, _P, _P, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]),
    "gb_graph500_encode": (C.c_int, [_P, _P, C.c_uint64, _P]),
    "gb_edge_list_parse": (C.c_int, [C.c_char_p, C.c_uint64, _P, _P, _P, C.POINTER(C.c_uint64)]),
    "gb_binary_decode": (C.c_int, [_P, C.c_uint64, C.c_int, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64),
                                   C.POINTER(C.c_int), _P, _P, _P, _P, _P]),
    "gb_graph_serialize": (C.c_int, [_P, C.c_char_p]),
    "gb_digraph_load_u32": (C.c_int, [C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "gb_graph_load_u32": (C.c_int, [C.c_int, C.c_char_p, C.c_int, C.c_int, C.POINTER(_P)]),
    "gb_graph_load_weighted_u32": (C.c_int, [C.c_int, C.c_char_p, C.c_int, C.c_int, C.POINTER(_P)]),
    "gb_graph_load_info": (C.c_int, [_P, C.POINTER(LoadInfo)]),
    "gb_digraph_load_labeled_u32": (C.c_int, [C.c_int, C.c_char_p, C.c_int, C.POINTER(_P)]),
    "gb_graph_load_labeled_u32": (C.c_int, [C.c_int, C.c_char_p, C.c_int, C.POINTER(_P)]),
    "gb_digraph_from_edges_labeled_u32": (C.c_int, [C.c_int, _P, _P, C.c_uint64, _P, C.c_uint32, C.c_int,
                                                    C.POINTER(_P)]),
    "gb_graph_from_edges_labeled_u32": (C.c_int, [C.c_int, _P, _P, C.c_uint64, _P, C.c_uint32, C.c_int,
                                                  C.POINTER(_P)]),
    "gb_digraph_load_labeled_binary_u32": (C.c_int, [C.c_int, C.c_char_p, C.c_int, C.c_uint32, C.POINTER(_P)]),
    "gb_graph_load_labeled_binary_u32": (C.c_int, [C.c_int, C.c_char_p, C.c_int, C.c_uint32, C.POINTER(_P)]),
    "gb_graph_serialize_labeled": (C.c_int, [_P, C.c_char_p]),
    "gb_binary_decode_labeled": (C.c_int, [_P, C.c_uint64, C.c_int, C.c_uint32, C.POINTER(C.c_uint32),
                                           C.POINTER(C.c_uint64), C.POINTER(C.c_int), _P, _P, _P, _P, _P, _P]),
    "gb_graph_node_values": (C.c_int, [_P, _P]),
    "gb_label_stats": (C.c_int, [_P, C.POINTER(LabelStatsInfo), _P, _P]),
    "gb_node_label_index": (C.c_int, [_P, C.POINTER(C.c_uint32), _P, _P]),
    "gb_neighbor_label_frequencies": (C.c_int, [_P, _P, _P, _P]),
    "gb_digraph_from_device_edges_u32": (C.c_int, [C.c_int, _P, _P, _P, C.c_uint64, C.c_uint32, C.c_int, _P,
                                                   C.POINTER(_P)]),
    "gb_graph_from_device_edges_u32": (C.c_int, [C.c_int, _P, _P, C.c_uint64, C.c_uint32, C.c_int, _P,
                                                 C.POINTER(_P)]),
    "gb_graph_from_device_weighted_edges_u32": (C.c_int, [C.c_int, _P, _P, _P, C.c_uint64, C.c_uint32, C.c_int,
                                                          _P, C.POINTER(_P)]),
    "gb_ids_to_u32": (C.c_int, [C.c_int, _P, C.c_int, C.c_uint64, _P, _P]),
    "gb_graph_free": (C.c_int, [_P]),
    "gb_graph_get_info": (C.c_int, [_P, C.POINTER(GraphInfo)]),
    "gb_graph_copy_csr": (C.c_int, [_P, C.c_int, _P, _P, _P]),
    "gb_graph_csr_len": (C.c_int, [_P, C.c_int, C.POINTER(C.c_uint64)]),
    "gb_graph_stream": (_P, [_P]),
    "gb_graph_last_timing": (C.c_int, [_P, C.POINTER(Timing)]),
    "gb_to_undirected": (C.c_int, [_P, C.c_int, C.POINTER(_P)]),
    "gb_to_undirected_weighted": (C.c_int, [_P, C.c_int, C.POINTER(_P)]),
    "gb_make_degree_ordered": (C.c_int, [_P]),
    "gb_page_rank": (C.c_int, [_P, C.POINTER(PageRankConfig), _P, C.POINTER(C.c_uint64), C.POINTER(C.c_double)]),
    "gb_page_rank_device": (C.c_int, [_P, C.POINTER(PageRankConfig), _P, C.POINTER(C.c_uint64), C.POINTER(C.c_double)]),
    "gb_page_rank_csr_u32": (C.c_int, [C.c_int, C.c_uint32, _P, _P, _P, C.POINTER(PageRankConfig), _P,
                                       C.POINTER(C.c_uint64), C.POINTER(C.c_double)]),
    "gb_digraph_for_page_rank_u32": (C.c_int, [C.c_int, C.c_uint32, _P, _P, _P, C.POINTER(_P)]),
    "gb_wcc": (C.c_int, [_P, C.POINTER(WccConfig), _P]),
    "gb_wcc_device": (C.c_int, [_P, C.POINTER(WccConfig), _P]),
    "gb_wcc_csr_u32": (C.c_int, [C.c_int, C.c_uint32, _P, _P, C.POINTER(WccConfig), _P]),
    "gb_wcc_file_u32": (C.c_int, [C.c_int, C.c_char_p, C.c_int, C.POINTER(WccConfig), C.POINTER(_P)]),
    "gb_components_node_count": (C.c_int, [_P, C.POINTER(C.c_uint32)]),
    "gb_components_copy": (C.c_int, [_P, _P]),
    "gb_components_free": (C.c_int, [_P]),
    "gb_wcc_file_info": (C.c_int, [C.POINTER(WccFileStats)]),
    "gb_wcc_shard_phase": (C.c_int, [_P, C.POINTER(WccConfig), C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32,
                                     C.c_int, _P, _P, _P]),
    "gb_wcc_sample_label": (C.c_int, [_P, C.POINTER(WccConfig), _P, C.POINTER(C.c_uint32), C.POINTER(C.c_int), _P]),
    "gb_sssp": (C.c_int, [_P, C.POINTER(SsspConfig), _P]),
    "gb_sssp_device": (C.c_int, [_P, C.POINTER(SsspConfig), _P]),
    "gb_sssp_csr_u32": (C.c_int, [C.c_int, C.c_uint32, _P, _P, _P, C.POINTER(SsspConfig), _P]),
    "gb_sssp_csr_info": (C.c_int, [C.POINTER(SsspCsrInfo)]),
    "gb_triangle_count": (C.c_int, [_P, C.POINTER(C.c_uint64)]),
    "gb_triangle_count_csr_u32": (C.c_int, [C.c_int, C.c_uint32, _P, _P, C.POINTER(C.c_uint64)]),
    "gb_triangle_count_csr_info": (C.c_int, [C.POINTER(TcCsrInfo)]),
    "gb_in_degree_partition": (C.c_int, [_P, C.c_uint32, _P]),
    "gb_page_rank_plan_info": (C.c_int, [_P, C.POINTER(PrShardStats)]),
    "gb_page_rank_plan_shape": (C.c_int, [_P, C.POINTER(PrPlanShape)]),
    "gb_page_rank_plan_values": (C.c_int, [_P, C.c_int, _P, C.c_uint64]),
    "gb_page_rank_plan_reset": (C.c_int, [_P]),
    "gb_pr_shard_create": (C.c_int, [_P, C.c_uint32, C.c_uint32, C.POINTER(_P)]),
    "gb_pr_shard_info": (C.c_int, [_P, C.POINTER(PrShardStats)]),
    "gb_pr_shard_plan_shape": (C.c_int, [_P, C.POINTER(PrPlanShape)]),
    "gb_pr_shard_plan_values": (C.c_int, [_P, C.c_int, _P, C.c_uint64]),
    "gb_pr_shard_init": (C.c_int, [_P, C.c_float, _P, _P, _P, _P]),
    "gb_pr_shard_step": (C.c_int, [_P, C.c_float, C.c_uint64, _P, _P, _P, C.c_uint32, _P, _P, _P, _P]),
    "gb_pr_shard_sync": (C.c_int, [_P, C.c_uint64, _P, _P, _P, _P, C.c_uint32, _P]),
    "gb_pr_shard_finish": (C.c_int, [_P, _P, _P, _P]),
    "gb_pr_shard_free": (C.c_int, [_P]),
    "gb_comm_init": (C.c_int, [C.c_int, _P, C.POINTER(_P)]),
    "gb_comm_info": (C.c_int, [_P, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "gb_comm_free": (C.c_int, [_P]),
    "gb_page_rank_multi": (C.c_int, [_P, _P, C.POINTER(PageRankConfig), _P, C.POINTER(C.c_uint64),
                                     C.POINTER(C.c_double)]),
    "gb_wcc_csr_multi_u32": (C.c_int, [_P, C.c_uint32, _P, _P, C.POINTER(WccConfig), _P]),
    "gb_page_rank_csr_multi_u32": (C.c_int, [_P, C.c_uint32, _P, _P, _P, C.POINTER(PageRankConfig), _P,
                                             C.POINTER(C.c_uint64), C.POINTER(C.c_double)]),
    "gb_pr_shards_csr_u32": (C.c_int, [_P, C.c_uint32, C.c_uint32, _P, _P, _P, C.POINTER(_P)]),
    "gb_algraph_from_edges_u32": (C.c_int, [C.c_int, C.c_int, _P, _P, _P, C.c_uint64, C.c_uint32, C.c_int, C.c_int,
                                            C.POINTER(_P)]),
    "gb_algraph_from_device_edges_u32": (C.c_int, [C.c_int, C.c_int, _P, _P, _P, C.c_uint64, C.c_uint32, C.c_int,
                                                   C.c_int, _P, C.POINTER(_P)]),
    "gb_algraph_load_u32": (C.c_int, [C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int, C.POINTER(_P)]),
    "gb_algraph_load_info": (C.c_int, [_P, C.POINTER(LoadInfo)]),
    "gb_algraph_add_edges_u32": (C.c_int, [_P, _P, _P, _P, C.c_uint64]),
    "gb_algraph_add_device_edges_u32": (C.c_int, [_P, _P, _P, _P, C.c_uint64, _P]),
    "gb_algraph_last_batch": (C.c_int, [_P, C.POINTER(AlBatchInfo)]),
    "gb_algraph_get_info": (C.c_int, [_P, C.POINTER(GraphInfo)]),
    "gb_algraph_copy_row": (C.c_int, [_P, C.c_int, C.c_uint32, C.c_uint32, _P, _P, C.POINTER(C.c_uint32)]),
    "gb_algraph_copy_csr": (C.c_int, [_P, C.c_int, C.c_uint64, _P, _P, _P, C.POINTER(C.c_uint64)]),
    "gb_algraph_to_graph": (C.c_int, [_P, C.POINTER(_P)]),
    "gb_algraph_free": (C.c_int, [_P]),
}


def load(path: Path = LIB_PATH) -> C.CDLL:
    if not path.exists():
        raise ImportError(
            f"{path} is missing: build it with `python -c 'import __graft_entry__ as e; e.build()'`. "
            "graph_b200 has no CPU fallback.")
    lib = C.CDLL(str(path))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError here = header/library drift
        fn.restype = res
        fn.argtypes = args
    if lib.gb_abi_version() != 1:
        raise ImportError("libgraph_b200.so ABI version mismatch")
    return lib


lib = load()


def check(status: int) -> None:
    if status == GB_OK:
        return
    msg = (lib.gb_last_error() or b"").decode("utf-8", "replace")
    if status in (GB_ERR_INVALID, GB_ERR_UNSUPPORTED):
        raise ValueError(msg)  # graph_mate maps builder errors to ValueError (crates/mate/src/lib.rs:24-28)
    if status == GB_ERR_OOM:
        raise MemoryError(msg)
    raise GraphB200Error(msg)
