/*
 * graph_b200.h — C ABI of libgraph_b200.so
 *
 * The drop-in boundary for the CSR hot path of neo4j-labs/graph (crate `graph`,
 * crates/algos + crates/builder).  The reference has no FFI of its own: its
 * seams are the generic functions in crates/algos/src/{page_rank,wcc,sssp,
 * triangle_count}.rs over the CSR types of crates/builder/src/graph/csr.rs.
 * Each entry point below names the reference item (file:line, relative to the
 * reference checkout) it replaces; INTEGRATION.md shows the `extern "C"` block
 * a maintainer adds on the Rust side.
 *
 * Conventions
 *   - node ids and CSR offsets are uint32_t (the reference's NI = u32:
 *     csr.rs:124 `Csr<NI, NI, EV>` uses NI for offsets too), so m < 2^32.
 *   - every pointer argument is a HOST pointer unless its name starts with
 *     `d_` (device pointer on the graph's device).
 *   - all calls return gb_status; on failure gb_last_error() holds a
 *     thread-local message.  Nothing unwinds or aborts across the ABI.
 *   - a gb_graph is immutable after creation except gb_make_degree_ordered
 *     (exclusive access, like `&mut self` in graph_ops.rs:173).
 *   - there is NO CPU fallback: if no CUDA device is usable every graph
 *     constructor fails with GB_ERR_CUDA.
 */
#ifndef GRAPH_B200_H
#define GRAPH_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GB_ABI_VERSION 1

typedef enum gb_status {
  GB_OK = 0,
  GB_ERR_INVALID = 1,     /* bad argument (null pointer, id out of range, n == 0, ...) */
  GB_ERR_CUDA = 2,        /* CUDA runtime error / no device */
  GB_ERR_OOM = 3,         /* device or host allocation failed */
  GB_ERR_UNSUPPORTED = 4  /* wrong graph kind for the call (e.g. TC on a directed graph) */
} gb_status;

/* crates/builder/src/graph/csr.rs:35-45  `enum CsrLayout` */
typedef enum gb_layout {
  GB_LAYOUT_UNSORTED = 0,     /* default; here: deterministic edge-list order */
  GB_LAYOUT_SORTED = 1,       /* rows ascending, duplicates kept (csr.rs:886-895) */
  GB_LAYOUT_DEDUPLICATED = 2  /* sorted, unique, self-loops removed (csr.rs:897-948) */
} gb_layout;

typedef enum gb_graph_kind {
  GB_KIND_DIRECTED = 0,   /* DirectedCsrGraph<u32>   csr.rs:364-368 */
  GB_KIND_UNDIRECTED = 1  /* UndirectedCsrGraph<u32> csr.rs:658-661 */
} gb_graph_kind;

/* which CSR of a graph an accessor refers to */
typedef enum gb_csr_which {
  GB_CSR_OUT = 0,        /* csr_out  (directed)  */
  GB_CSR_IN = 1,         /* csr_inc  (directed)  */
  GB_CSR_UNDIRECTED = 2  /* csr      (undirected)*/
} gb_csr_which;

/* opaque device-resident twin of DirectedCsrGraph / UndirectedCsrGraph */
typedef struct gb_graph gb_graph;

typedef struct gb_graph_info {
  uint32_t kind;          /* gb_graph_kind */
  uint32_t node_count;    /* Graph::node_count  lib.rs:315-321 */
  uint64_t edge_count;    /* Graph::edge_count: directed = |out targets|; undirected = |targets|/2 (csr.rs:687-689) */
  uint64_t target_count;  /* entries in the out (or undirected) targets array */
  uint32_t has_weights;   /* 1 if the out-CSR carries f32 edge values (Target<u32,f32>, graph/mod.rs:6-10) */
  int32_t device;         /* CUDA device ordinal the arrays live on */
  uint64_t device_bytes;  /* HBM held by this handle */
} gb_graph_info;

/* crates/algos/src/page_rank.rs:14-56  `PageRankConfig` (+ a schedule selector) */
typedef enum gb_pr_mode {
  GB_PR_AUTO = 0,    /* n <= 16384 -> GB_PR_EXACT, else GB_PR_JACOBI */
  GB_PR_EXACT = 1,   /* the reference's sweep as ONE thread runs it: in place, CSR-order f32 sums
                        (page_rank.rs:142-160). Bit-exact with the reference whenever the reference
                        itself is deterministic (n <= CHUNK_SIZE = 16384, page_rank.rs:12). Sequential. */
  GB_PR_JACOBI = 2   /* throughput path: double-buffered sweep (every read sees iteration k), deterministic.
                        CAVEAT for drop-in callers: the reference sweep is in place (Gauss-Seidel-like,
                        and schedule dependent for n > 16384), so with the reference's DEFAULT config
                        (tolerance 1e-4) JACOBI meets the tolerance at a different sweep count and returns
                        ranks ~1e-3 away from an in-place run; both converge to the same fixed point.  Use
                        tolerance 0 + a fixed sweep count, or a tight tolerance, when comparing. */
} gb_pr_mode;

typedef struct gb_page_rank_config {
  uint64_t max_iterations; /* DEFAULT_MAX_ITERATIONS = 20   page_rank.rs:46 */
  double tolerance;        /* DEFAULT_TOLERANCE = 1e-4      page_rank.rs:47 */
  float damping_factor;    /* DEFAULT_DAMPING_FACTOR = 0.85 page_rank.rs:48 */
  uint32_t mode;           /* gb_pr_mode */
} gb_page_rank_config;

/* crates/algos/src/wcc.rs:40-79  `WccConfig` */
typedef struct gb_wcc_config {
  uint64_t chunk_size;      /* 16384 — scheduling only in the reference; ignored on device */
  uint64_t neighbor_rounds; /* 2 */
  uint64_t sampling_size;   /* 1024 */
} gb_wcc_config;

/* crates/algos/src/sssp.rs:18-36  `DeltaSteppingConfig` */
typedef struct gb_sssp_config {
  uint64_t start_node;
  float delta;
} gb_sssp_config;

/* per-call device timing of the last algorithm run on a graph (for bench / result `micros`) */
typedef struct gb_timing {
  double total_ms;       /* CUDA-event time of the whole device section of the call */
  double hot_kernel_ms;  /* summed CUDA-event time of the dominant kernel (only when profiling is on) */
  uint64_t hot_kernel_launches;
  uint64_t kernel_launches; /* all kernels this library launched in the call */
} gb_timing;

/* ---- library ------------------------------------------------------------------------------- */
int gb_abi_version(void);
const char* gb_last_error(void);
/* number of usable CUDA devices (0 when none: every constructor then fails) */
int gb_device_count(void);
/* when on, algorithm calls bracket each launch of their dominant kernel with CUDA events */
void gb_set_profiling(int on);

/* ---- graph lifecycle ----------------------------------------------------------------------- */
/* From already-built host CSR arrays: the device twin of an existing DirectedCsrGraph
 * (csr.rs:364-368: csr_out + csr_inc).  out_w may be NULL (EV = ()).  Arrays are copied. */
gb_status gb_digraph_from_csr_u32(int device, uint32_t node_count,
                                  const uint32_t* out_offsets, const uint32_t* out_targets,
                                  const float* out_weights,
                                  const uint32_t* in_offsets, const uint32_t* in_targets,
                                  gb_graph** graph);
/* Device twin of an UndirectedCsrGraph (csr.rs:658-661); `targets` has offsets[n] entries. */
gb_status gb_graph_from_csr_u32(int device, uint32_t node_count, const uint32_t* offsets,
                                const uint32_t* targets, gb_graph** graph);

/* From an edge list — replaces `Csr::from((&edges, node_count, direction, layout))`
 * (csr.rs:124-221) and the DirectedCsrGraph/UndirectedCsrGraph `From<(E, CsrLayout)>` impls
 * (csr.rs:522-543, :727-760): the CSR is built ON DEVICE (histogram, scan, radix sort).
 * node_count == 0 means max id + 1 (edgelist.rs:84-90).  weights may be NULL.
 * UNSORTED yields the single-thread order of the reference (edge-list order; for undirected
 * graphs the outgoing pass first, then the incoming pass: csr.rs:154-172, :1199-1205). */
gb_status gb_digraph_from_edges_u32(int device, const uint32_t* src, const uint32_t* dst,
                                    const float* weights, uint64_t edge_count,
                                    uint32_t node_count, gb_layout layout, gb_graph** graph);
gb_status gb_graph_from_edges_u32(int device, const uint32_t* src, const uint32_t* dst,
                                  uint64_t edge_count, uint32_t node_count, gb_layout layout,
                                  gb_graph** graph);

/* Synthetic R-MAT / Graph500-style graph generated on device (a,b,c,d = .57,.19,.19,.05,
 * n = 2^scale, m = edge_factor * n, ids scrambled, duplicates and self-loops kept); the same
 * generator exists on the CPU in oracle/ for parity.  The reference reads such inputs from a
 * packed Graph500 file (input/graph500.rs:63-127, node_count = edge_count/16).
 * weights != 0 attaches deterministic uniform (0,1] f32 edge values (for SSSP). */
gb_status gb_digraph_rmat(int device, uint32_t scale, uint32_t edge_factor, uint64_t seed,
                          gb_layout layout, int weights, gb_graph** graph);
gb_status gb_graph_rmat(int device, uint32_t scale, uint32_t edge_factor, uint64_t seed,
                        gb_layout layout, gb_graph** graph);
/* the raw generator: fills host arrays with edges [first, first+count) of that stream */
gb_status gb_rmat_edges(int device, uint32_t scale, uint64_t seed, uint64_t first, uint64_t count,
                        uint32_t* src, uint32_t* dst);

/* ---- input formats (host side, multi-threaded) ------------------------------------------------
 * Graph500 packed 12-byte edges (input/graph500.rs:63-127): src/dst hold len/12 entries;
 * node_count = edge_count / 16 (graph500.rs:74).  Ids above 32 bits are an error. */
gb_status gb_graph500_decode(const void* bytes, uint64_t len, uint32_t* src, uint32_t* dst,
                             uint64_t* edge_count, uint32_t* node_count);
/* edges -> packed records (12 * edge_count bytes): the file the reference's CLI reads with
 * `-f graph500 --use-32-bit` (crates/app/src/runner.rs:104-133); note its node_count = edges/16 rule */
gb_status gb_graph500_encode(const uint32_t* src, const uint32_t* dst, uint64_t edge_count, void* bytes);
/* Text edge list "<src> <dst>[ <f32>]" with \n or \r\n line ends (input/edgelist.rs:181-279).
 * Call with src == NULL to obtain *edge_count, then again with arrays of that size; values may be
 * NULL.  Edges come out in file order. */
gb_status gb_edge_list_parse(const char* text, uint64_t len, uint32_t* src, uint32_t* dst,
                             float* values, uint64_t* edge_count);
/* Binary graph file of SerializeGraphOp (graph_ops.rs:232-238; csr.rs:252-341, :606-656, :817-851; the
 * layout is restated in graph_b200/csrc/binary_format.h): NI "u32", "u64" or "usize", records with or
 * without f32 values (told apart by the file size).  Call with out_offsets == NULL to check the headers and
 * obtain *node_count, *entries (targets per CSR; undirected: 2m) and *has_values; then again with arrays of
 * node_count + 1 offsets and `entries` targets (in_* only for a directed file).  out_values may be NULL (the
 * values are dropped) and must be NULL for a file without values; in-CSR values are never returned.  u64
 * ids are narrowed; ids or offsets >= 2^32, malformed offsets and targets >= node_count are errors. */
gb_status gb_binary_decode(const void* bytes, uint64_t len, gb_graph_kind kind, uint32_t* node_count,
                           uint64_t* entries, int* has_values, uint32_t* out_offsets, uint32_t* out_targets,
                           float* out_values, uint32_t* in_offsets, uint32_t* in_targets);

/* ---- loading files on the device ----------------------------------------------------------------
 * The file is streamed through a ring of pinned buffers (pread on several threads, copy stream, parse
 * kernels); no host edge array exists.  The graph is the one the host readers above followed by
 * gb_[di]graph_from_edges_u32 give, byte for byte, with the same errors and messages.  Text values that
 * the device parser declines (inf, nan, long or exotic spellings) are re-parsed on the host.  Files below
 * 64 MiB are read by the host readers, whose fixed costs are lower; the
 * pinned ring (at most 4 x 64 MiB) is kept for the next load.
 * GB_LOAD_CHUNK_BYTES (environment, read per call) sets the buffer size and selects the device path at
 * any file size, for tests. */
typedef enum gb_file_format {
  GB_FORMAT_GRAPH500 = 0,  /* packed 12-byte records; node_count = edges / 16 */
  GB_FORMAT_EDGE_LIST = 1, /* text "<src> <dst>[ <f32>]"; node_count = max id + 1 */
  GB_FORMAT_BINARY = 2     /* SerializeGraphOp's file (see gb_binary_decode): the CSRs as stored */
} gb_file_format;
/* with_values: read the third column of an edge list as f32 edge values (Graph500 has none).
 * A binary file's rows are kept byte for byte: `layout` is checked and otherwise ignored, as the reference
 * ignores it (csr.rs:650), and the row order is left unknown, as after gb_graph_from_csr_u32.  with_values
 * = 1 needs a file with values; with 0 they are dropped, and so are the in-CSR values (the device keeps
 * none) and an undirected file's values.  The streamed path DMAs u32 sections without values straight into
 * the CSR arrays and narrows / splits the others on the device. */
gb_status gb_digraph_load_u32(int device, const char* path, gb_file_format format, gb_layout layout,
                              int with_values, gb_graph** graph);
gb_status gb_graph_load_u32(int device, const char* path, gb_file_format format, gb_layout layout,
                            gb_graph** graph);
/* SerializeGraphOp::serialize (graph_ops.rs:232-238): writes the graph as a binary file with NI = "u32";
 * a weighted digraph writes Target<u32,f32> records for both CSRs, the in-CSR value of the k-th occurrence
 * of s in in-row t being that of the k-th occurrence of t in out-row s (for every graph built here the
 * value of the same edge; the in-CSR must be the transpose of the out-CSR).  So save(load(f)) is byte-equal
 * to f for files written here, and for a foreign weighted file up to the order of the values among parallel
 * (s, t) edges.  The file is written to a temporary file in the same directory, which is renamed over
 * `path` on success and removed on failure.  GB_ERR_INVALID for a gb_digraph_for_page_rank_u32 twin. */
gb_status gb_graph_serialize(const gb_graph* graph, const char* path);
/* Statistics of the load that created the graph (all zero for graphs made otherwise). */
typedef struct gb_load_info {
  uint64_t file_bytes;     /* size of the file */
  uint64_t chunks;         /* pinned buffers the file was streamed through */
  uint64_t edges;          /* edges read */
  uint64_t fallback_lines; /* lines whose value was re-parsed on the host */
  uint64_t h2d_bytes;      /* bytes copied host -> device */
} gb_load_info;
gb_status gb_graph_load_info(const gb_graph* graph, gb_load_info* info);

/* From DEVICE edge arrays on `device` (not modified, not kept): like gb_[di]graph_from_edges_u32 without the
 * upload.  node_count == 0 means max id + 1, found on the device.  Work already enqueued on `stream`
 * (a cudaStream_t; NULL = the legacy default stream) is waited for before the arrays are read. */
gb_status gb_digraph_from_device_edges_u32(int device, const uint32_t* d_src, const uint32_t* d_dst,
                                           const float* d_weights, uint64_t edge_count, uint32_t node_count,
                                           gb_layout layout, void* stream, gb_graph** graph);
gb_status gb_graph_from_device_edges_u32(int device, const uint32_t* d_src, const uint32_t* d_dst,
                                         uint64_t edge_count, uint32_t node_count, gb_layout layout,
                                         void* stream, gb_graph** graph);
/* Narrows device ids (int32 when id_bytes == 4, int64 when 8) to uint32 on the device; any id outside
 * [0, 2^32) is GB_ERR_INVALID.  Enqueued on `stream`, waited for before returning. */
gb_status gb_ids_to_u32(int device, const void* d_ids, int id_bytes, uint64_t count, uint32_t* d_out,
                        void* stream);

gb_status gb_graph_free(gb_graph* graph);
gb_status gb_graph_get_info(const gb_graph* graph, gb_graph_info* info);
/* copy a CSR back to the host (neighbour views of the host mirror: csr.rs:97-117).
 * offsets: node_count+1 entries; targets: target_count entries; weights may be NULL. */
gb_status gb_graph_copy_csr(const gb_graph* graph, gb_csr_which which, uint32_t* offsets,
                            uint32_t* targets, float* weights);
/* number of entries in the chosen CSR's targets array */
gb_status gb_graph_csr_len(const gb_graph* graph, gb_csr_which which, uint64_t* len);
/* the CUDA stream (cudaStream_t) all work of this graph is issued on */
void* gb_graph_stream(const gb_graph* graph);
gb_status gb_graph_last_timing(const gb_graph* graph, gb_timing* timing);

/* ---- graph ops ----------------------------------------------------------------------------- */
/* ToUndirectedOp::to_undirected (graph_ops.rs:229, csr.rs:391-464) */
gb_status gb_to_undirected(const gb_graph* digraph, gb_layout layout, gb_graph** graph);
/* RelabelByDegreeOp::make_degree_ordered (graph_ops.rs:173,250-252,511-638): new id = rank in
 * (degree, old id) DESCENDING; rows rewritten and re-sorted.  Undirected graphs only. */
gb_status gb_make_degree_ordered(gb_graph* graph);

/* ---- algorithms ---------------------------------------------------------------------------- */
/* page_rank(&graph, config) -> (Vec<f32>, usize, f64)     page_rank.rs:58-111
 * scores: node_count floats, caller-owned. */
gb_status gb_page_rank(const gb_graph* graph, const gb_page_rank_config* config, float* scores,
                       uint64_t* ran_iterations, double* error);
/* same, result left in HBM (d_scores: node_count floats on the graph's device) */
gb_status gb_page_rank_device(const gb_graph* graph, const gb_page_rank_config* config,
                              float* d_scores, uint64_t* ran_iterations, double* error);

/* One-shot form for a caller that holds the CSR on the host and wants no resident twin: exactly
 * what page_rank reads through its trait bounds (page_rank.rs:61: Graph + DirectedDegrees +
 * DirectedNeighbors) — the in-CSR and the out-degrees (given as out offsets).  Uploads
 * 4m + 8(n+1) bytes instead of the full twin's 8m + 8(n+1).  The targets are streamed in row-aligned
 * chunks and the layout build runs underneath the upload (pass page-locked arrays: from pageable memory
 * the copies are synchronous and nothing overlaps; the result is the same). */
gb_status gb_page_rank_csr_u32(int device, uint32_t node_count, const uint32_t* in_offsets,
                               const uint32_t* in_targets, const uint32_t* out_offsets,
                               const gb_page_rank_config* config, float* scores,
                               uint64_t* ran_iterations, double* error);

/* The same upload as a handle: a device twin holding exactly what page_rank reads (in-CSR + out-degrees;
 * there are no out targets, so wcc / sssp / to_undirected on it fail with GB_ERR_INVALID or read an empty
 * out-CSR).  Used by the multi-GPU path, where every rank builds its shard from host arrays. */
gb_status gb_digraph_for_page_rank_u32(int device, uint32_t node_count, const uint32_t* in_offsets,
                                       const uint32_t* in_targets, const uint32_t* out_offsets,
                                       gb_graph** graph);

/* wcc_afforest(&graph, config).to_vec()                    wcc.rs:127-139, afforest.rs:100-114
 * components[v] = root of v = minimum node id of v's weakly connected component. */
gb_status gb_wcc(const gb_graph* graph, const gb_wcc_config* config, uint32_t* components);
gb_status gb_wcc_device(const gb_graph* graph, const gb_wcc_config* config, uint32_t* d_components);

/* wcc_baseline(&graph, config) (wcc.rs:103-123) -- and, since the labels are the same, wcc_afforest(...).to_vec() --
 * from a HOST CSR, with no resident twin.  Reads what wcc_baseline reads: node_count and the out-CSR (any CSR
 * whose rows list the graph's edges gives the same labels; weak connectivity does not depend on the direction).
 * The offsets go first; the targets are streamed in fixed-size edge chunks through a ring of device buffers and
 * every chunk is linked (Afforest::union, afforest.rs:22-39) while the next one is on the bus.  Pass page-locked
 * arrays to get the overlap; from pageable memory the copies are synchronous and the result is the same.
 * components: node_count entries, caller-owned; not written when the call fails.  config is checked and otherwise
 * ignored (the reference's chunk_size / neighbor_rounds / sampling_size change the work, never the labels).
 * targets may be NULL when offsets[node_count] == 0.  GB_WCC_FEED_EDGES (environment, read per call) sets the
 * chunk size in edges (rounded down to a multiple of 4; default 2^22). */
gb_status gb_wcc_csr_u32(int device, uint32_t node_count, const uint32_t* offsets, const uint32_t* targets,
                         const gb_wcc_config* config, uint32_t* components);

/* Multi-GPU WCC (1-D cut by vertex range, one process per GPU; the caller owns the exchange of the
 * parent arrays, e.g. an NCCL all-gather).  The phases of wcc() (wcc.rs:158-183) restricted to the rank's
 * vertices [vertex_begin, vertex_end) over a FULL parent[n] on every rank:
 *   INIT, SAMPLE (own vertices), COMPRESS, exchange + MERGE of every other rank's forest, COMPRESS,
 *   gb_wcc_sample_label on the merged forest (identical on every rank), LINK_REMAINING (own vertices,
 *   skipping the GLOBAL giant component: skipping a vertex is only safe when the other endpoint of each
 *   of its edges is either in the same component already or processed by its own owner — which a
 *   rank-local giant component would not guarantee), COMPRESS, exchange + MERGE, COMPRESS.
 * The link rule is Afforest::union (afforest.rs:22-39) throughout, so the labels are the minimum node id
 * of each component on every rank, bit-equal to gb_wcc. */
typedef enum gb_wcc_phase {
  GB_WCC_INIT = 0,
  GB_WCC_SAMPLE = 1,
  GB_WCC_COMPRESS = 2,
  GB_WCC_MERGE = 3,
  GB_WCC_LINK_REMAINING = 4
} gb_wcc_phase;
gb_status gb_wcc_shard_phase(const gb_graph* graph, const gb_wcc_config* config, uint32_t phase,
                             uint32_t vertex_begin, uint32_t vertex_end, uint32_t skip_label, int use_skip,
                             uint32_t* d_parent, const uint32_t* d_other, void* cuda_stream);
/* most frequent parent[] among config->sampling_size pseudo-random vertices (find_largest_component,
 * wcc.rs:245-271; fixed seed); *found = 0 when sampling_size == 0 */
gb_status gb_wcc_sample_label(const gb_graph* graph, const gb_wcc_config* config, const uint32_t* d_parent,
                              uint32_t* label, int* found, void* cuda_stream);

/* delta_stepping(&graph, config) -> Vec<AtomicF32>          sssp.rs:38-102
 * distances: node_count floats; unreachable = FLT_MAX (sssp.rs:12). */
gb_status gb_sssp(const gb_graph* graph, const gb_sssp_config* config, float* distances);
gb_status gb_sssp_device(const gb_graph* graph, const gb_sssp_config* config, float* d_distances);

/* global_triangle_count(&graph) -> u64                      triangle_count.rs:22-86
 * Any row order, as the reference counts it.  The first call on a graph whose rows are not known to be
 * sorted (an Unsorted build, gb_graph_from_csr_u32) checks them once and caches the answer. */
gb_status gb_triangle_count(const gb_graph* graph, uint64_t* triangles);

/* global_triangle_count (triangle_count.rs:22-86) of a HOST undirected CSR, with no twin kept: the number
 * gb_graph_from_csr_u32 + gb_triangle_count give for the same arrays, with the same checks and messages
 * (on unsorted rows, the reference's list-order number).  Layout rule: offsets has node_count + 1 entries
 * from 0, targets offsets[node_count] (may be NULL when that is 0); the rows are taken as they are, in any
 * order.  Each term of the sum is one entry (u, v <= u) and reads rows u and v only, so the call is causal
 * in row order: the offsets go first, the targets follow in row-aligned chunks of about equal entry counts
 * (a row longer than a chunk gets one of its own), and every chunk is checked (targets < node_count, row
 * order) and counted as soon as its rows have landed, while the next chunks are on the bus.  Chunks count
 * with the sorted-row kernel while every row so far is sorted, and with the list-order kernels from the
 * first chunk with an unsorted row on.  Residency: the terms read earlier rows at random, so unlike
 * gb_wcc_csr_u32's ring the whole CSR (4(n+1) + 4m bytes) is on the device by the end of the call; it is
 * freed before the call returns.  Pass page-locked targets to get the overlap: all chunks then go out at
 * once on a copy stream; from pageable memory the copies are synchronous, one chunk ahead of the count,
 * and the result is the same.  GB_TC_FEED_ENTRIES (environment, read per call) sets the entries per chunk
 * (default ceil(m / 16), at least 2^20; never fewer than m / 4096). */
gb_status gb_triangle_count_csr_u32(int device, uint32_t node_count, const uint32_t* offsets,
                                    const uint32_t* targets, uint64_t* triangles);
/* Statistics of the calling thread's last gb_triangle_count_csr_u32 (all zero after a failed call). */
typedef struct gb_tc_csr_info {
  uint64_t chunks;           /* row-aligned chunks the targets were uploaded and counted in */
  uint64_t chunk_entries;    /* the entry budget of a chunk */
  uint64_t h2d_bytes;        /* bytes copied host -> device: 4(n+1) + 4m */
  uint64_t sorted_chunks;    /* chunks counted by the sorted-row kernel (k_tc) */
  uint64_t list_chunks;      /* chunks counted by the list-order kernels (k_tc_cut + k_tc_list) */
  uint64_t first_list_chunk; /* the first of those; == chunks when every row is sorted */
  uint64_t kernel_launches;  /* checks and counts */
  uint32_t pinned;           /* 1: the targets were page-locked */
  uint32_t reserved;
  double upload_ms;          /* CUDA-event time from the first copy to the last target landing */
  double total_ms;           /* CUDA-event time from the first copy to the end of the last count */
} gb_tc_csr_info;
gb_status gb_triangle_count_csr_info(gb_tc_csr_info* info);

/* ---- PageRank layout statistics / multi-GPU shard (1-D edge-cut by destination) -----------------
 * The JACOBI path renumbers vertices internally (in-degree descending, then out-degree descending)
 * and column-blocks the sweep (graph_b200/csrc/pagerank.cu).  For N GPUs (one process per GPU;
 * torch.distributed / NCCL own the plumbing) the 32-row slices of that internal order are dealt
 * round-robin: rank p owns slices p, p + P, p + 2P, ... — every rank holds the same mix of hub and
 * tail rows, derives its rows from the degree arrays alone and builds the layout of its own rows
 * only.  (The reference's own partitioner, in_degree_partition over the ORIGINAL ids,
 * graph_ops.rs:431-439, is gb_in_degree_partition below; contiguous ranges of the degree-sorted
 * order would give rank 0 all hubs and rank P-1 millions of one-edge rows.)  Rank p owns the
 * out_scores entries of its rows; they are exchanged once per sweep, either by the caller (NCCL
 * all-gather) or by the sweep kernels themselves storing each finished value into the peers' next
 * vectors (fused all-gather: one multimem.st through the NVSwitch, or one store per peer). */
typedef struct gb_pr_shard gb_pr_shard;

typedef struct gb_pr_shard_stats {
  uint32_t rank, world;
  uint32_t active_rows;        /* rows with in-edges, whole graph */
  uint32_t local_rows;         /* of which owned by this shard */
  uint64_t local_edges;        /* in-edges of the local rows */
  uint64_t block_edges;        /* of which gathered from shared-memory column blocks */
  uint32_t block_entries;      /* source-vector entries per column block */
  uint32_t hot_blocks;         /* column blocks that own segments */
  uint64_t segments;           /* (row, block) pairs with a segment */
  uint64_t groups;             /* 4-id groups in all block streams */
  uint32_t chunks, tasks, cut_segments, chunk_groups;
  uint32_t launches_per_sweep;
  uint64_t device_bytes;       /* HBM held by this layout */
} gb_pr_shard_stats;

/* the reference's own partitioner on the ORIGINAL ids: in_degree_partition (graph_ops.rs:431-439,
 * :479-509); ranges has parts+1 entries */
gb_status gb_in_degree_partition(const gb_graph* graph, uint32_t parts, uint32_t* ranges);
/* layout statistics of the single-GPU JACOBI plan (built on first use) */
gb_status gb_page_rank_plan_info(const gb_graph* graph, gb_pr_shard_stats* stats);
/* drops the cached layout (the next JACOBI call rebuilds it, re-reading the GB_PR_* experiment knobs) */
gb_status gb_page_rank_plan_reset(const gb_graph* graph);
/* builds the layout of shard `rank` of `world` on the graph's device */
gb_status gb_pr_shard_create(const gb_graph* graph, uint32_t rank, uint32_t world, gb_pr_shard** shard);
gb_status gb_pr_shard_info(const gb_pr_shard* shard, gb_pr_shard_stats* stats);
/* Diagnostics: the launch shape the layout chose for the sweep kernels (k_pr_cb, k_pr_fixup, k_pr_sell,
 * k_pr_finish), so that tests can tell which variant of each a graph reaches.  Not part of the stable
 * statistics above; fields may be added. */
typedef struct gb_pr_plan_shape {
  uint32_t hot_blocks;         /* column blocks that own segments (KB) */
  uint32_t n_cb;               /* local rows [0, n_cb) own at least one segment */
  uint32_t n_fin;              /* local rows [0, n_fin) are completed by k_pr_finish */
  uint32_t n_fin_warp;         /* of which [0, n_fin_warp) are hub groups (one finish CTA per 32 rows) */
  uint32_t fin_u;              /* 32-row groups per warp iteration of k_pr_finish (2 or 4) */
  uint32_t fin_hub_ctas;       /* finish CTAs reserved for the hub groups (0 = no role split) */
  uint32_t grid_cb, grid_sell, grid_fin;
  uint32_t n_mega;             /* local rows laid out through the sort path of the layout build */
  uint32_t n_fix;              /* chunks whose last segment continues in the next chunk */
  uint32_t fix_in_sell;        /* 1: those parts are added by k_pr_sell, 0: by k_pr_fixup */
  uint32_t dual;               /* always 0 (the sweep's kernels run one after the other on one stream);
                                  kept so that the fields after it keep their offsets */
  uint32_t last_hot_block;     /* largest source block index among the hot blocks (0xFFFFFFFF: none) */
} gb_pr_plan_shape;
gb_status gb_page_rank_plan_shape(const gb_graph* graph, gb_pr_plan_shape* shape);
gb_status gb_pr_shard_plan_shape(const gb_pr_shard* shard, gb_pr_plan_shape* shape);
/* fills the full initial vectors (n floats each, internal order) on this rank: d_x0 = init/outdeg,
 * the constant part of d_x1; d_scores = init for own rows, 0 for the others (rows without in-edges:
 * base on rank 0), so that the ranks' score vectors can be summed into the full one */
gb_status gb_pr_shard_init(const gb_pr_shard* shard, float damping, float* d_x0, float* d_x1,
                           float* d_scores, void* cuda_stream);
/* one sweep (1-based sweep_no) over the shard's rows: reads the full d_x_cur[n], writes the shard's
 * entries of d_x_next and of every peer's next vector — through d_mc_x_next (a multicast mapping of
 * all ranks' next vectors, this rank's included) when it is non-NULL, else through d_peer_x_next[i]
 * (peer-mapped full vectors; peer_count may be 0) — updates the shard's entries of d_scores and stores
 * this shard's share of the sweep error in *d_error.  All work is enqueued on cuda_stream. */
gb_status gb_pr_shard_step(const gb_pr_shard* shard, float damping, uint64_t sweep_no,
                           const float* d_x_cur, float* d_x_next, float* const* d_peer_x_next,
                           uint32_t peer_count, float* d_mc_x_next, float* d_scores, double* d_error,
                           void* cuda_stream);
/* Device-side inter-sweep barrier + error sum of the fused exchange (no collective, no host round trip).
 * Every rank owns a 192-byte control block in peer-mapped memory (zero-initialised; d_self_block is this
 * rank's, d_peer_blocks[q] the mapping of rank q's, entry `rank` ignored).  Enqueued after
 * gb_pr_shard_step: publishes this rank's *d_local_error and its arrival at sweep_no into every rank's
 * block, waits until all ranks have arrived, and stores the sum of the P error shares (added in rank
 * order: identical on every rank) in d_total_error[slot]. */
gb_status gb_pr_shard_sync(const gb_pr_shard* shard, uint64_t sweep_no, const double* d_local_error,
                           void* d_self_block, void* const* d_peer_blocks, double* d_total_error,
                           uint32_t slot, void* cuda_stream);
#define GB_PR_SYNC_BLOCK_BYTES 192
/* internal order -> original ids: d_scores_out[v] = d_scores_internal[new_id[v]] */
gb_status gb_pr_shard_finish(const gb_pr_shard* shard, const float* d_scores_internal,
                             float* d_scores_out, void* cuda_stream);
/* the graph must outlive every other call on its shards; the free may come before or after gb_graph_free */
gb_status gb_pr_shard_free(gb_pr_shard* shard);

/* ---- single-process multi-GPU PageRank ------------------------------------------------------------
 * For a host that owns N devices itself (the reference is one process): no torch, no NCCL.
 * gb_comm_init enables peer access all-to-all among `devices` (NULL = 0..ndev-1).  gb_page_rank_multi
 * takes the SAME graph resident on every device of the communicator (graphs[i] on devices[i]; a
 * gb_digraph_for_page_rank_u32 twin is enough), builds every device's shard, runs the sweeps with the fused
 * exchange (one multimem.st per value when the driver offers multicast objects, else one peer store per
 * device) and the device-side barrier, and returns page_rank's triple (page_rank.rs:58-111).  One host
 * thread drives all devices; inside the sweep loop the host never waits unless tolerance > 0. */
typedef struct gb_comm gb_comm;
gb_status gb_comm_init(int ndev, const int* devices, gb_comm** comm);
gb_status gb_comm_info(const gb_comm* comm, int* ndev, int* multicast);
gb_status gb_comm_free(gb_comm* comm);
gb_status gb_page_rank_multi(gb_comm* comm, const gb_graph* const* graphs, const gb_page_rank_config* config,
                             float* scores, uint64_t* ran_iterations, double* error);
/* page_rank (page_rank.rs:58-111) of a HOST CSR over the devices of a communicator, with no resident twin:
 * the contract, checks, messages and config handling of gb_page_rank_csr_u32 + gb_page_rank_multi (the
 * sharded JACOBI schedule, one rank per device; scores not written when the call fails).  Each device uploads
 * one row-aligned part of the arrays (about 1/ndev of the edges, and 1/ndev of each offset array) over its
 * own link; the offsets are all-gathered over NVLink, and every rank gathers the targets of the rows it
 * owns from the parts (peer reads) into a compact local in-CSR, builds its shard layout from it and frees
 * it.  The ranks are bit-equal to gb_page_rank_multi on the same communicator with a full twin per device.
 * GB_PR_PART_CHUNK_EDGES (environment, read per call; default 2^23) sets the size of the target chunks that
 * the gathers wait for one by one.  Pass page-locked arrays to get the overlap. */
gb_status gb_page_rank_csr_multi_u32(gb_comm* comm, uint32_t node_count, const uint32_t* in_offsets,
                                     const uint32_t* in_targets, const uint32_t* out_offsets,
                                     const gb_page_rank_config* config, float* scores,
                                     uint64_t* ran_iterations, double* error);
/* The shards of that call, for a caller that drives the sweeps itself (gb_pr_shard_init / step / sync /
 * finish).  ranks_per_device = V puts ranks i*V .. i*V+V-1 (of ndev*V <= 8) on devices[i]; shards[r] is rank r.
 * Each shard is identical (plan shape, statistics, device bytes, sweep results) to
 * gb_pr_shard_create(twin, r, ndev*V) on a full twin.  V > 1 runs every multi-part path on one GPU.  The shards
 * hold no graph; free each with gb_pr_shard_free. */
gb_status gb_pr_shards_csr_u32(gb_comm* comm, uint32_t ranks_per_device, uint32_t node_count,
                               const uint32_t* in_offsets, const uint32_t* in_targets,
                               const uint32_t* out_offsets, gb_pr_shard** shards);
/* wcc_baseline(&graph, config) (wcc.rs:103-123) of a HOST out-CSR over the devices of a communicator: the
 * contract, checks, messages and labels of gb_wcc_csr_u32 (the minimum node id of each component; components
 * is not written when the call fails; config is checked and otherwise ignored; targets may be NULL when
 * offsets[node_count] == 0).  The edges are cut into P = ndev x V parts of about m / P edges (cuts at
 * multiples of 4 edges, not at rows); part p runs on devices[p / V], uploads only the offsets of the rows its
 * edges touch, streams its targets over that device's own PCIe link through its own ring of buffers and links
 * them into its own forest.  The P forests then merge in ceil(log2 P) rounds over NVLink (peer reads of the
 * partner's forest), and device 0 copies the labels to the host.  The comm's PageRank buffers are neither used
 * nor changed.  V = 1 unless GB_WCC_MULTI_PARTS (environment, read per call; clamped to 1..64) says otherwise:
 * V > 1 runs several parts per device, which tests every multi-part path on one GPU.  GB_WCC_FEED_EDGES sets
 * the chunk size as for gb_wcc_csr_u32.  Pass page-locked arrays (and components) to get the overlap. */
gb_status gb_wcc_csr_multi_u32(gb_comm* comm, uint32_t node_count, const uint32_t* offsets,
                               const uint32_t* targets, const gb_wcc_config* config, uint32_t* components);

#ifdef __cplusplus
}
#endif
#endif /* GRAPH_B200_H */
