// common.cuh — shared plumbing of libgraph_b200.so (error handling, device buffers, graph handle).
#pragma once
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "../../include/graph_b200.h"
#include "csr_split.h"
#include "dotgraph_line.h"

namespace gb {

// ---- thread-local error message behind gb_last_error() ---------------------------------------
std::string& last_error();
gb_status fail(gb_status st, const char* fmt, ...);

#define GB_CUDA(expr)                                                                          \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      gb_status _s = (_e == cudaErrorMemoryAllocation) ? GB_ERR_OOM : GB_ERR_CUDA;             \
      return gb::fail(_s, "%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
    }                                                                                          \
  } while (0)

#define GB_TRY(expr)                 \
  do {                               \
    gb_status _s = (expr);           \
    if (_s != GB_OK) return _s;      \
  } while (0)

#define GB_REQUIRE(cond, ...)                                   \
  do {                                                          \
    if (!(cond)) return gb::fail(GB_ERR_INVALID, __VA_ARGS__);  \
  } while (0)

// ---- device buffer (RAII) ------------------------------------------------------------------------
// Stream-ordered allocations from the device's default memory pool, whose release threshold is raised
// once so that freed blocks stay cached: the one-shot entry points (gb_page_rank_csr_u32 uploads a CSR,
// builds a layout and frees everything on every call) then pay for their ~9 GB of cudaMalloc/cudaFree
// only the first time.  Semantics stay those of cudaMalloc/cudaFree: alloc returns memory usable on
// any stream at once, release waits for the device before the block goes back to the pool.
inline void devbuf_pool_setup() {
  static thread_local int configured_for = -1;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev == configured_for) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
    unsigned long long keep = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  configured_for = dev;
}
// Inside a DevBufStreamScope every buffer released by this thread is known to have been used on that
// one stream only, so release waits for the stream instead of the device: the layout build can then drop
// its temporaries while a copy stream is still bringing in the rest of the graph.
inline cudaStream_t*& devbuf_scope_slot() {
  static thread_local cudaStream_t* slot = nullptr;
  return slot;
}
struct DevBufStreamScope {
  cudaStream_t stream;
  cudaStream_t* prev;
  explicit DevBufStreamScope(cudaStream_t s) : stream(s), prev(devbuf_scope_slot()) { devbuf_scope_slot() = &stream; }
  ~DevBufStreamScope() { devbuf_scope_slot() = prev; }
  DevBufStreamScope(const DevBufStreamScope&) = delete;
  DevBufStreamScope& operator=(const DevBufStreamScope&) = delete;
};
// The device bytes one call holds: while a DevBufTally is open on a thread, every DevBuf that thread allocates is
// counted in `now` until it is released, and `peak` keeps the most held at once.  A buffer that outlives the call
// leaves the tally first (DevBuf::untally).
struct DevBufTally {
  uint64_t now = 0, peak = 0;
  DevBufTally* prev;
  static DevBufTally*& slot() {
    static thread_local DevBufTally* open = nullptr;
    return open;
  }
  DevBufTally() : prev(slot()) { slot() = this; }
  ~DevBufTally() { slot() = prev; }
  DevBufTally(const DevBufTally&) = delete;
  DevBufTally& operator=(const DevBufTally&) = delete;
};
template <typename T>
struct DevBuf {
  T* p = nullptr;
  size_t n = 0;
  DevBufTally* tally = nullptr;  // counts the block's `held` bytes
  size_t held = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : p(o.p), n(o.n), tally(o.tally), held(o.held) {
    o.p = nullptr; o.n = 0; o.tally = nullptr; o.held = 0;
  }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) {
      release();
      p = o.p; n = o.n; tally = o.tally; held = o.held;
      o.p = nullptr; o.n = 0; o.tally = nullptr; o.held = 0;
    }
    return *this;
  }
  ~DevBuf() { release(); }
  void release() {
    if (p) {
      // like cudaFree: nothing may still be using the block
      if (cudaStream_t* scoped = devbuf_scope_slot()) cudaStreamSynchronize(*scoped);
      else cudaDeviceSynchronize();
      cudaFreeAsync(p, cudaStreamLegacy);
    }
    untally();
    p = nullptr;
    n = 0;
  }
  void untally() {
    if (tally) tally->now -= held;
    tally = nullptr;
    held = 0;
  }
  // allocates count elements (+ pad elements of slack so 128-bit loads may overrun the tail)
  gb_status alloc(size_t count, size_t pad = 0) {
    release();
    size_t bytes = (count + pad) * sizeof(T);
    if (bytes == 0) bytes = sizeof(T);
    devbuf_pool_setup();
    cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&p), bytes, cudaStreamLegacy);
    if (e == cudaSuccess) e = cudaStreamSynchronize(cudaStreamLegacy);  // usable from every stream now
    if (e != cudaSuccess) {
      p = nullptr;
      cudaGetLastError();
      return fail(e == cudaErrorMemoryAllocation ? GB_ERR_OOM : GB_ERR_CUDA,
                  "cudaMallocAsync(%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
    }
    n = count;
    if ((tally = DevBufTally::slot())) {
      held = bytes;
      tally->now += bytes;
      tally->peak = std::max(tally->peak, tally->now);
    }
    return GB_OK;
  }
  size_t bytes() const { return n * sizeof(T); }
};

// Device memory that another device may read or copy from.  cudaDeviceEnablePeerAccess (gb_comm_init) maps
// cudaMalloc memory into the peers, not blocks of the stream-ordered pool DevBuf draws from (a pool is
// reachable from its own device only unless cudaMemPoolSetAccess says otherwise), so a buffer that peers read
// is cudaMalloc'd, on one device as on many; one that no peer reads keeps the pool's cached blocks.
struct PeerBuf {
  uint32_t* p = nullptr;
  uint32_t* shared = nullptr;
  DevBuf<uint32_t> pooled;
  gb_status alloc(size_t count, bool peers, size_t pad = 0) {
    if (!peers) {
      GB_TRY(pooled.alloc(count, pad));
      p = pooled.p;
      return GB_OK;
    }
    const size_t words = count + pad ? count + pad : 1;
    GB_CUDA(cudaMalloc(reinterpret_cast<void**>(&shared), words * sizeof(uint32_t)));
    p = shared;
    return GB_OK;
  }
  void release() {  // on the buffer's device, nothing may still use it
    if (shared) cudaFree(shared);
    shared = p = nullptr;
    pooled.release();
  }
  ~PeerBuf() { release(); }
};

// ---- one device's feed of a slice of a host CSR (graph.cu; csr_split.h cuts the slices) -------------------
// The offsets [r_begin, r_end] of a host CSR, and with them the same rows of a second offsets array when the
// caller has one, go to device dev on the feed's own copy stream, with offsets_in recorded behind them.  The
// targets [e_begin, e_end) follow chunk by chunk, each with an event behind it, either resident (each chunk at
// its place in tgt, one landed event per chunk) or through a ring of R slots (chunk k in slot k mod R, one
// landed and one freed event per slot).  A ring consumer records freed[k mod R] behind its last read of chunk k,
// and must enqueue that record before send(k + R) is called: cudaStreamWaitEvent takes the event's latest
// record at the time of the call, so every wait then refers to a record already enqueued, and a pageable copy,
// which returns only once its stream has drained, blocks the host only until work already enqueued has run.
// A resident feed may carry one f32 value per target (val, asked for with `values`): chunk k's values are
// copied right after its targets, with the same bounds, before landed[k].
// The consumers' streams are the caller's, and must drain before the feed goes.  The id checks are the
// caller's too: WCC and PageRank make their own, and CheckedFeed (below) makes them for a resident feed.
struct CsrFeed {
  int dev = -1;
  uint32_t r_begin = 0, r_end = 0;
  uint64_t e_begin = 0;
  cudaStream_t copy = nullptr;
  cudaEvent_t offsets_in = nullptr;
  PeerBuf off, off2;                      // [r_end - r_begin + 1] each; off2 only with a second offsets array
  PeerBuf tgt;                            // resident: [e_end - e_begin] + 8 zeroed
  DevBuf<float> val;                      // resident with values: [e_end - e_begin]
  std::vector<DevBuf<uint32_t>> ring;     // ring: R slots of `slot` entries + 8 zeroed
  std::vector<cudaEvent_t> landed, freed; // resident: landed[K]; ring: landed[R], freed[R]

  // makes dev current, creates the stream and offsets_in and allocates the offsets (peers: PeerBuf)
  gb_status open(int device, uint32_t rb, uint32_t re, bool peers, bool two_offsets = false);
  gb_status resident(uint64_t eb, uint64_t ee, uint32_t chunks, bool peers, bool values = false);
  gb_status open_ring(uint32_t slots, uint64_t slot);
  // copies off[r_begin .. r_end] (and off2's) and records offsets_in
  gb_status send_offsets(const uint32_t* host_off, const uint32_t* host_off2 = nullptr);
  // chunk k = the targets [e0, e0 + len) of host_tgt (and the same values of host_val, for a feed with values);
  // an empty chunk only records its event
  gb_status send(uint64_t k, const uint32_t* host_tgt, uint64_t e0, uint64_t len, const float* host_val = nullptr);
  // on s, behind offsets_in: bad[0] += the rows v in [r0, r1) with off[v] > off[v + 1], bad[1] the same of off2
  gb_status check_monotone(cudaStream_t s, uint32_t r0, uint32_t r1, unsigned int* bad) const;
  // whether host memory is page-locked: such a copy does not wait for its stream to drain
  static bool pinned(const void* host);
  ~CsrFeed();
};

// ---- a checked, resident upload of a whole host CSR to one device (graph.cu) ---------------------------------
// The triangle count and SSSP of a host CSR (gb_triangle_count_csr_u32, gb_sssp_csr_u32) read chunks of it while
// the rest is on the bus.  open() cuts the targets (and values) into tc_split chunks of tc_chunk_entries(m, knob)
// entries, sends the offsets [0, n] into a resident CsrFeed and queues their monotone check on the check stream.
// issue() sends the next chunk of the send order (sssp_send_order from row `first`; first = 0 sends the chunks in
// row order), and on the check stream behind its landed event counts its targets >= n into h_bad[1 + k], runs
// per_chunk(k) when the caller set one, and records checked[j] (j: the chunk's place in the send order) behind
// it all.  A consumer reads chunk order[j] only once checked[j] has passed and h_bad[1 + order[j]] is 0.
// Page-locked targets (and values) go out all at once; a pageable copy returns only once it is done, so from
// pageable memory the caller issues each chunk when it is ready for it.
// The destructor drains the check stream before the events, the page-locked tally and the feed go.  The
// consumer streams are the caller's, and must drain before it goes: a call keeps it as its first member.
struct CheckedFeed {
  CsrFeed feed;
  CsrChunks ch;
  std::vector<uint32_t> order;  // the send order: order[j] is the j-th chunk sent
  std::function<gb_status(uint32_t k)> per_chunk;  // more of chunk k's checks, enqueued on `check`
  cudaStream_t check = nullptr;
  DevBuf<unsigned int> bad;       // [0] rows whose offsets decrease, [1 + k] targets >= n in chunk k
  unsigned int* h_bad = nullptr;  // page-locked: bad[1 + K]
  cudaEvent_t begin = nullptr, uploaded = nullptr, end = nullptr;  // timed; `end` is recorded by finish()
  cudaEvent_t offsets_checked = nullptr;
  std::vector<cudaEvent_t> checked;  // [j]: behind the checks of the j-th chunk sent
  const uint32_t* tgt = nullptr;
  const float* val = nullptr;
  const char* what = "";  // begins the failure messages ("undirected", "out")
  uint32_t n = 0, K = 0, issued = 0;
  uint64_t chunk_entries = 0, launches = 0;  // launches: the check kernels enqueued
  bool pinned = false;

  // a host CSR of `nodes` rows (require_host_csr has passed) and its values (NULL: none)
  gb_status open(int device, uint32_t nodes, const uint32_t* off, const uint32_t* host_tgt, const float* host_val,
                 uint64_t knob, uint32_t first, const char* name);
  gb_status issue();
  // waits for the monotone check of the offsets: GB_OK, or require_monotone's failure
  gb_status require_offsets();
  // issues every chunk left and waits for their checks: GB_OK, or require_ids's failure on the summed tally
  gb_status check_all();
  // on the consumer stream s: waits for the last chunk to land (so that `end` follows the whole upload), records
  // end, copies `bytes` of the result from dev to host and synchronises s
  gb_status finish(cudaStream_t s, void* host, const void* dev, size_t bytes);
  // the fields gb_tc_csr_info and gb_sssp_csr_stats share, once finish() has returned
  template <typename Info>
  gb_status report(Info* info) const {
    info->chunks = K;
    info->chunk_entries = chunk_entries;
    info->pinned = pinned ? 1 : 0;
    info->h2d_bytes = 4 * ((uint64_t)n + 1) + (val ? 8 : 4) * ch.edge[K];  // edge[K] == m
    info->kernel_launches += launches;
    float up = 0.0f, all = 0.0f;
    GB_CUDA(cudaEventElapsedTime(&up, begin, uploaded));
    GB_CUDA(cudaEventElapsedTime(&all, begin, end));
    info->upload_ms = up;
    info->total_ms = all;
    return GB_OK;
  }
  ~CheckedFeed();
};

// The O(1) host checks of a host CSR, in this order: offsets NULL, offsets[0] == 0, then targets NULL when it
// has entries (not with offsets_only).  Messages begin with `what` ("in", "out", "undirected"; "" for none).
gb_status require_host_csr(uint32_t n, const uint32_t* off, const uint32_t* tgt, const char* what,
                           bool offsets_only = false);
// The verdicts of the device checks on their summed counts: GB_OK when it is 0, else the failure
gb_status require_monotone(const char* what, uint64_t bad_rows);
gb_status require_ids(const char* what, uint64_t bad_targets, uint32_t n);

// an unsigned decimal knob from the environment (experiments); dflt when it is unset or empty
inline uint64_t env_u64(const char* name, uint64_t dflt) {
  const char* e = getenv(name);
  return e && *e ? strtoull(e, nullptr, 10) : dflt;
}

// CUB's two-phase call: call(nullptr, bytes) sizes the temporary storage, call(tmp.p, bytes) runs.  tmp is
// the caller's, so its release (which waits for the stream) stays where the caller puts it; a buffer that
// already holds enough is reused, a new one gets `headroom` times the size asked for.
template <typename Call>
gb_status cub_call(DevBuf<uint8_t>& tmp, Call&& call, size_t headroom = 1) {
  size_t bytes = 0;
  GB_CUDA(call(nullptr, bytes));
  if (!tmp.p || tmp.n < bytes) {
    DevBuf<uint8_t> fresh;
    GB_TRY(fresh.alloc(bytes * headroom));
    tmp = std::move(fresh);  // an old buffer is released once the stream is done with it
  }
  GB_CUDA(call(tmp.p, bytes));
  return GB_OK;
}

// CUB's in-place prefix sums and its radix pair sort over bits [0, end_bit), enqueued on s through cub_call; N, the
// count's type, is CUB's offset type.  For the translation units that include CUB first: an include of CUB emits a
// kernel into its translation unit, so this header does not pull it in.
#ifdef CUB_VERSION
template <typename T, typename N>
gb_status exclusive_sum(cudaStream_t s, DevBuf<uint8_t>& tmp, T* a, N count) {
  return cub_call(tmp, [&](void* t, size_t& tb) { return cub::DeviceScan::ExclusiveSum(t, tb, a, a, count, s); });
}
template <typename T, typename N>
gb_status inclusive_sum(cudaStream_t s, DevBuf<uint8_t>& tmp, T* a, N count) {
  return cub_call(tmp, [&](void* t, size_t& tb) { return cub::DeviceScan::InclusiveSum(t, tb, a, a, count, s); });
}
template <typename K, typename V, typename N>
gb_status sort_pairs(cudaStream_t s, DevBuf<uint8_t>& tmp, cub::DoubleBuffer<K>& k, cub::DoubleBuffer<V>& v, N count,
                     int end_bit) {
  return cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceRadixSort::SortPairs(t, tb, k, v, count, 0, end_bit, s);
  });
}
#endif

// ---- device CSR ----------------------------------------------------------------------------
// offsets[n+1] u32, targets[len] u32 (+8 entries of zeroed slack for 128-bit loads), optional
// SoA weights[len] f32 (the host API exposes the reference's 8-byte AoS Target{u32,f32}).
struct DevCsr {
  DevBuf<uint32_t> off;
  DevBuf<uint32_t> tgt;
  DevBuf<float> w;
  uint64_t len = 0;
  uint64_t bytes() const { return off.bytes() + tgt.bytes() + w.bytes(); }
};

struct PrPlan;  // pr_plan.cuh

// Whether every row of the undirected CSR is in ascending order (an inversion across a row boundary does not
// count).  Sorted and Deduplicated builds and make_degree_ordered write sorted rows; an Unsorted build or a
// caller's CSR is Unknown until gb_triangle_count looks once and caches the answer.
enum class RowOrder : uint8_t { Unknown, Sorted, Unsorted };

}  // namespace gb

// the opaque handle of the C ABI
struct gb_graph {
  int device = 0;
  gb_graph_kind kind = GB_KIND_DIRECTED;
  uint32_t n = 0;
  gb::DevCsr out;  // directed: csr_out; undirected: the single csr
  gb::DevCsr in;   // directed only: csr_inc
  mutable gb::RowOrder row_order = gb::RowOrder::Unknown;  // of `out`; set by the builds, cached by tc.cu
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_begin = nullptr, ev_end = nullptr;
  mutable std::mutex mu;            // algorithms on one handle serialise on its stream
  mutable gb::PrPlan* pr_plan = nullptr;  // lazily built PageRank layout (pagerank.cu)
  mutable gb_timing timing{};
  gb_load_info load{};  // filled by gb_[di]graph_load_u32 (load.cu)
  // NodeValues of a labelled twin (one u32 label per node), NULL otherwise.  Only labels.cu reads them;
  // to_undirected copies them and make_degree_ordered leaves them where they are (graph_ops.rs:511-538).
  gb::DevBuf<uint32_t> labels;
};

namespace gb {
void free_pr_plan(PrPlan* p);
uint64_t pr_plan_bytes(const PrPlan* p);
bool profiling_on();

// RAII: make the graph's device current for the duration of a call
struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
    if (prev != dev) ok = (cudaSetDevice(dev) == cudaSuccess);
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

// owning graph handle: a constructor that fails part-way releases the graph by returning
struct GraphFree {
  void operator()(gb_graph* g) const { gb_graph_free(g); }
};
using GraphPtr = std::unique_ptr<gb_graph, GraphFree>;

// GB_ERR_CUDA when there is no CUDA device, GB_ERR_INVALID when `device` is not one of them
gb_status require_device(int device);
gb_status check_layout(gb_layout layout);

// CSR construction on device (graph.cu)
// rows/cols: device arrays of `count` entries, only read. Builds `csr` with the given layout; n rows.
// w may be null.  It holds one value per entry when w_period is 0; otherwise w_period values that entries j and
// j + w_period share (an undirected build's two passes over one edge list, count = 2 * w_period).  With w_pairs
// entries 2i and 2i + 1 share w[i] instead (an adjacency list's interleaved undirected stream).  keep_self_loops
// makes Deduplicated keep entries whose target is their row, as the adjacency lists do (adj_list.rs:260-263).
gb_status build_csr_device(cudaStream_t s, uint32_t n, const uint32_t* d_rows, const uint32_t* d_cols,
                           const float* d_w, uint64_t count, gb_layout layout, DevCsr* csr, uint64_t w_period = 0,
                           bool keep_self_loops = false, bool w_pairs = false);
// Checks device edge arrays on s: *n == 0 becomes the largest id + 1, otherwise every id must be below *n.
gb_status check_edge_ids(cudaStream_t s, const uint32_t* d_src, const uint32_t* d_dst, uint64_t m, uint32_t* n);
// GB_ERR_INVALID unless p is device (or managed) memory of `device`
gb_status require_device_array(const void* p, int device, const char* what);
// Edge arrays on the device: read from a file (load.cu: Graph500 or text edge list through the pinned-ring
// pipeline, in file order; n is edges / 16 for Graph500 and 0 (max id + 1) for an edge list), or copied from the
// host (upload_edges).
struct EdgeArrays {
  DevBuf<uint32_t> src, dst;
  DevBuf<float> w;
  uint64_t m = 0;
  uint32_t n = 0;
  gb_load_info info{};
};
gb_status load_edge_arrays(int device, const char* path, gb_file_format format, bool with_values, EdgeArrays* out);
// Copies m host edges into out->src, out->dst on stream s, and their values into out->w when w is not NULL (out->w
// is allocated then even for m = 0, which marks a build with values).  Returns once the copies are enqueued.
gb_status upload_edges(cudaStream_t s, const uint32_t* src, const uint32_t* dst, const float* w, uint64_t m,
                       EdgeArrays* out);
// The argument checks of every edge-list constructor, in this order: out, the kind, the edge arrays, the weights
// (with_values only), the layout, the u32 offset limit (2m entries when undirected) and n = 0 without edges.
gb_status check_edge_args(gb_graph_kind kind, const void* src, const void* dst, const void* w, uint64_t m, uint32_t n,
                          gb_layout layout, bool with_values, const void* out);
// Makes stream s wait for the work enqueued on `caller` so far (a caller's producer work comes first).
gb_status wait_on_stream(cudaStream_t s, cudaStream_t caller);
gb_status new_graph(int device, gb_graph_kind kind, uint32_t n, GraphPtr* out);
// Uploads a host CSR on stream s and checks it: require_host_csr on the host, the offsets monotone and the
// targets below n on the device.  offsets_only uploads the offsets alone (degrees); w may be NULL.  Returns
// with s synchronised.
gb_status upload_host_csr(cudaStream_t s, uint32_t n, const uint32_t* off, const uint32_t* tgt, const float* w,
                          DevCsr* csr, const char* what, bool offsets_only = false);
// enqueue on s: *bad += the number of ids in a[0, count) that are >= n
void check_ids_async(cudaStream_t s, const uint32_t* a, uint64_t count, uint32_t n, unsigned int* bad);
// enqueue on s: *bad += the number of rows v < n with off[v] > off[v + 1]
void check_monotone_async(cudaStream_t s, const uint32_t* off, uint32_t n, unsigned int* bad);
// builds a graph from device edge arrays (graph.cu; behind gb_[di]graph_from_device_edges_u32)
gb_status graph_from_device_arrays(int device, gb_graph_kind kind, const uint32_t* d_src, const uint32_t* d_dst,
                                   const float* d_w, uint64_t m, uint32_t n, gb_layout layout, cudaStream_t caller,
                                   gb_graph** out);

// Values for a weighted digraph's in-CSR (graph.cu): the k-th occurrence of s in in-row t gets the value of the
// k-th occurrence of t in out-row s.  Fails when the in-CSR is not the transpose of the out-CSR.  Runs on the
// graph's stream; the caller holds g->mu.
gb_status in_csr_values(const gb_graph* g, DevBuf<float>* in_w);

// ---- DotGraph files (io.cu; grammar in dotgraph_line.h) ----
// The header from the first bytes of the file: its whole first line, or the whole file when it has no '\n'.
gb_status dot_read_header(const char* text, uint64_t len, DotHeader* h);
// The node and edge lines of a whole file in host memory: labels[N], src[M], dst[M].  A NULL labels (or src, and
// with it dst) skips those stores: the lines are still checked.
gb_status dot_read_host(const char* text, uint64_t len, const DotHeader& h, uint32_t* labels, uint32_t* src,
                        uint32_t* dst);
// The failure of a DotGraph read: `code` on 1-based line `line`, or DOT_MISSING with `have` of h.lines lines.
gb_status dot_fail(uint32_t code, uint64_t line, const DotHeader& h, uint64_t have);
// Copies n labels (host or device memory, by `kind`) into g->labels on g's stream and waits for the copy.
gb_status attach_labels(gb_graph* g, const uint32_t* labels, cudaMemcpyKind kind);

// ---- union-find links for the WCC of a graph file (wcc.cu; load.cu decodes the chunks) ----
// Every link hooks the higher root under the lower, so after cc_compress_async parent[v] is the minimum node id of
// v's component, as gb_wcc gives.  All of them enqueue on s.
// parent[v] = v for v in [from, to)
void cc_init_async(cudaStream_t s, uint32_t* parent, uint64_t from, uint64_t to);
// links src[i] with dst[i] for i < count; a pair with an endpoint >= n is not linked, and *bad counts its endpoints
// >= n (the count check_edge_ids makes)
void cc_link_pairs_async(cudaStream_t s, const uint32_t* src, const uint32_t* dst, uint64_t count, uint32_t n,
                         uint32_t* parent, unsigned int* bad);
// links every edge [e0, e0 + len) of a device CSR of n rows whose offsets are checked (off[0] == 0, monotone,
// off[n] == entries): tgt holds those edges' targets with 8 entries of slack; *bad counts the targets >= n
void cc_link_csr_async(cudaStream_t s, const uint32_t* off, uint32_t n, const uint32_t* tgt, uint32_t e0,
                       uint32_t len, uint32_t* parent, unsigned int* bad);
void cc_compress_async(cudaStream_t s, uint32_t* parent, uint32_t n);

// the devices of a communicator, in its order (multi.cu); peer access among them is enabled
const std::vector<int>& comm_devices(const gb_comm* c);

constexpr unsigned H100_SMS = 132;  // streaming multiprocessors of an H100 SXM: sizes the grid-stride grids

inline unsigned grid_for(uint64_t items, unsigned block, unsigned max_blocks = H100_SMS * 16u) {
  uint64_t b = (items + block - 1) / block;
  if (b < 1) b = 1;
  if (b > max_blocks) b = max_blocks;
  return static_cast<unsigned>(b);
}

// bits of the largest id below n (at least 1, at most 32): the width of a field of a packed sort key
inline uint32_t bits_for(uint64_t n) {
  uint32_t b = 1;
  while (b < 32 && (1ull << b) < n) ++b;
  return b;
}

// The library is built without -rdc, so a kernel launched from several translation units lives here; templates,
// so that a translation unit that does not launch one emits nothing.
template <typename T>
__global__ void k_iota(T* __restrict__ a, uint64_t count) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    a[i] = (T)i;
}

template <typename T>
__global__ void k_gather(const T* __restrict__ src, const uint32_t* __restrict__ idx, uint64_t count,
                         T* __restrict__ dst) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    dst[i] = src[idx[i]];
}
}  // namespace gb
