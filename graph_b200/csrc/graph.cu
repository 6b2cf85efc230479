// graph.cu — device-resident twin of the reference's CSR graph types and its construction.
//
//   DirectedCsrGraph{csr_out, csr_inc}   crates/builder/src/graph/csr.rs:364-368
//   UndirectedCsrGraph{csr}              crates/builder/src/graph/csr.rs:658-661
//   Csr::from((&edges, n, direction, layout))   csr.rs:124-221  -> build_csr_device (radix sort)
//   to_undirected                        csr.rs:391-464
//   make_degree_ordered                  crates/builder/src/graph_ops.rs:511-638
//
// The reference builds a CSR with an atomic scatter followed by a per-row sort; here the whole
// build is one device radix sort of packed (row, target) keys, which yields the Sorted layout
// directly, makes Unsorted deterministic (stable sort on the row bits only = edge-list order) and
// turns Deduplicated into a flagged compaction.
#include <cub/cub.cuh>

#include "common.cuh"
#include "rmat.cuh"

namespace gb {

std::string& last_error() {
  static thread_local std::string msg;
  return msg;
}

gb_status fail(gb_status st, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  last_error() = buf;
  return st;
}

static bool g_profiling = false;
bool profiling_on() { return g_profiling; }

static inline uint32_t bits_for(uint32_t n) {
  uint32_t b = 1;
  while (b < 32 && (1ull << b) < n) ++b;
  return b;
}

// ---- kernels -------------------------------------------------------------------------------
__global__ void k_pack_keys(const uint32_t* __restrict__ rows, const uint32_t* __restrict__ cols,
                            uint64_t count, uint32_t bits, uint64_t* __restrict__ keys) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    keys[i] = ((uint64_t)rows[i] << bits) | cols[i];
}

__global__ void k_iota(uint32_t* __restrict__ a, uint64_t count) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    a[i] = (uint32_t)i;
}

// offsets from a row-sorted sequence: the end of each non-empty row's run is marked at
// marks[row + 1]; offsets are the running maximum of the marks (empty rows inherit the previous
// end), so no thread ever walks a gap of empty rows.
template <typename RowFn>
__global__ void k_mark_row_ends(RowFn row_of, uint64_t count, uint32_t* __restrict__ marks) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t r = row_of(i);
    if (i + 1 == count || row_of(i + 1) != r) marks[r + 1] = (uint32_t)(i + 1);
  }
}

struct RowOfKey {
  const uint64_t* keys;
  uint32_t bits;
  __device__ uint32_t operator()(uint64_t i) const { return (uint32_t)(keys[i] >> bits); }
};
struct RowOfArr {
  const uint32_t* rows;
  __device__ uint32_t operator()(uint64_t i) const { return rows[i]; }
};

template <typename RowFn>
static gb_status offsets_from_sorted(cudaStream_t s, RowFn row_of, uint64_t count, uint32_t n,
                                     uint32_t* off) {
  GB_CUDA(cudaMemsetAsync(off, 0, ((size_t)n + 1) * 4, s));
  if (count) k_mark_row_ends<<<grid_for(count, 256), 256, 0, s>>>(row_of, count, off);
  DevBuf<uint8_t> tmp;
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceScan::InclusiveScan(t, tb, off, off, cub::Max(), (int64_t)n + 1, s);
  }));
  GB_CUDA(cudaStreamSynchronize(s));  // tmp is released on return
  return GB_OK;
}

__global__ void k_unpack_targets(const uint64_t* __restrict__ keys, uint64_t count, uint32_t bits,
                                 uint32_t* __restrict__ tgt) {
  uint64_t mask = (bits >= 32) ? 0xFFFFFFFFull : ((1ull << bits) - 1ull);
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    tgt[i] = (uint32_t)(keys[i] & mask);
}

template <typename T>
__global__ void k_gather(const T* __restrict__ src, const uint32_t* __restrict__ idx, uint64_t count,
                         T* __restrict__ dst) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    dst[i] = src[idx[i]];
}

// Deduplicated layout (csr.rs:897-948): keep the first of each run of equal (row,target) keys and
// drop entries whose target is the row itself.
__global__ void k_dedup_flags(const uint64_t* __restrict__ keys, uint64_t count, uint32_t bits,
                              uint8_t* __restrict__ flags) {
  uint64_t mask = (bits >= 32) ? 0xFFFFFFFFull : ((1ull << bits) - 1ull);
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t k = keys[i];
    bool keep = (i == 0 || keys[i - 1] != k) && ((uint32_t)(k >> bits) != (uint32_t)(k & mask));
    flags[i] = keep ? 1 : 0;
  }
}

// expands CSR offsets into one row id per entry: one warp per row (coalesced stores, no searches)
__global__ void k_expand_rows(const uint32_t* __restrict__ off, uint32_t n, uint32_t* __restrict__ rows) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t v = warp; v < n; v += nwarps) {
    const uint32_t b = off[v], e = off[v + 1];
    for (uint32_t i = b + lane; i < e; i += 32) rows[i] = v;
  }
}

__global__ void k_check_ids(const uint32_t* __restrict__ a, uint64_t count, uint32_t n,
                            unsigned int* __restrict__ bad) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    if (a[i] >= n) atomicAdd(bad, 1u);
}

__global__ void k_rmat(uint32_t scale, uint64_t seed, uint64_t first, uint64_t count,
                       uint32_t* __restrict__ src, uint32_t* __restrict__ dst) {
  RmatScramble scr(scale, seed);
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < count;
       k += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t s, t;
    rmat_edge(scale, seed, first + k, scr, &s, &t);
    src[k] = s;
    dst[k] = t;
  }
}

__global__ void k_rmat_weights(uint64_t seed, uint64_t count, float* __restrict__ w) {
  for (uint64_t k = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; k < count;
       k += (uint64_t)gridDim.x * blockDim.x)
    w[k] = rmat_weight(seed, k);
}

// make_degree_ordered helpers
__global__ void k_degree_keys(const uint32_t* __restrict__ off, uint32_t n, uint64_t* __restrict__ keys) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x)
    keys[v] = ((uint64_t)(off[v + 1] - off[v]) << 32) | v;
}
__global__ void k_rank_to_newid(const uint64_t* __restrict__ sorted, uint32_t n,
                                uint32_t* __restrict__ new_id, uint32_t* __restrict__ new_deg) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) {
    uint64_t k = sorted[r];
    new_id[(uint32_t)k] = r;                 // unzip_degrees_and_nodes, graph_ops.rs:564-592
    new_deg[r] = (uint32_t)(k >> 32);
  }
}
__global__ void k_relabel_keys(const uint32_t* __restrict__ rows, const uint32_t* __restrict__ tgt,
                               const uint32_t* __restrict__ new_id, uint64_t count, uint32_t bits,
                               uint64_t* __restrict__ keys) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    keys[i] = ((uint64_t)new_id[rows[i]] << bits) | new_id[tgt[i]];
}

// ---- CSR build -----------------------------------------------------------------------------
gb_status build_csr_device(cudaStream_t s, uint32_t n, const uint32_t* d_rows, const uint32_t* d_cols,
                           const float* d_w, uint64_t count, gb_layout layout, DevCsr* csr) {
  GB_REQUIRE(count < 0xFFFFFFFFull, "CSR with %llu entries does not fit u32 offsets (csr.rs:124)",
             (unsigned long long)count);
  const uint32_t bits = bits_for(n);
  const unsigned blk = 256;
  GB_TRY(csr->off.alloc((size_t)n + 1));
  csr->len = count;
  if (count == 0) {
    GB_CUDA(cudaMemsetAsync(csr->off.p, 0, ((size_t)n + 1) * 4, s));
    GB_TRY(csr->tgt.alloc(0, 8));
    GB_CUDA(cudaMemsetAsync(csr->tgt.p, 0, 8 * 4, s));
    if (d_w) GB_TRY(csr->w.alloc(0, 8));
    return GB_OK;
  }

  if (layout == GB_LAYOUT_UNSORTED) {
    // stable sort on the row id only: within a row the edge-list order survives
    DevBuf<uint32_t> keys_alt, idx, idx_alt, rows_copy;
    GB_TRY(rows_copy.alloc(count));
    GB_TRY(keys_alt.alloc(count));
    GB_TRY(idx.alloc(count));
    GB_TRY(idx_alt.alloc(count));
    GB_CUDA(cudaMemcpyAsync(rows_copy.p, d_rows, count * 4, cudaMemcpyDeviceToDevice, s));
    k_iota<<<grid_for(count, blk), blk, 0, s>>>(idx.p, count);
    cub::DoubleBuffer<uint32_t> kb(rows_copy.p, keys_alt.p);
    cub::DoubleBuffer<uint32_t> vb(idx.p, idx_alt.p);
    DevBuf<uint8_t> tmp;
    GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
      return cub::DeviceRadixSort::SortPairs(t, tb, kb, vb, count, 0, (int)bits, s);
    }));
    GB_TRY(csr->tgt.alloc(count, 8));
    GB_CUDA(cudaMemsetAsync(csr->tgt.p + count, 0, 8 * 4, s));
    k_gather<uint32_t><<<grid_for(count, blk), blk, 0, s>>>(d_cols, vb.Current(), count, csr->tgt.p);
    if (d_w) {
      GB_TRY(csr->w.alloc(count, 8));
      k_gather<float><<<grid_for(count, blk), blk, 0, s>>>(d_w, vb.Current(), count, csr->w.p);
    }
    GB_TRY(offsets_from_sorted(s, RowOfArr{kb.Current()}, count, n, csr->off.p));
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaStreamSynchronize(s));
    return GB_OK;
  }

  // Sorted / Deduplicated: one radix sort of (row << bits | target) keys
  DevBuf<uint64_t> keys, keys_alt;
  GB_TRY(keys.alloc(count));
  GB_TRY(keys_alt.alloc(count));
  k_pack_keys<<<grid_for(count, blk), blk, 0, s>>>(d_rows, d_cols, count, bits, keys.p);
  cub::DoubleBuffer<uint64_t> kb(keys.p, keys_alt.p);
  DevBuf<uint32_t> idx, idx_alt;
  DevBuf<uint8_t> tmp;
  const uint32_t* order = nullptr;
  if (d_w) {
    GB_TRY(idx.alloc(count));
    GB_TRY(idx_alt.alloc(count));
    k_iota<<<grid_for(count, blk), blk, 0, s>>>(idx.p, count);
    cub::DoubleBuffer<uint32_t> vb(idx.p, idx_alt.p);
    GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
      return cub::DeviceRadixSort::SortPairs(t, tb, kb, vb, count, 0, (int)(2 * bits), s);
    }));
    order = vb.Current();
  } else {
    GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
      return cub::DeviceRadixSort::SortKeys(t, tb, kb, count, 0, (int)(2 * bits), s);
    }));
  }
  uint64_t* sorted = kb.Current();
  uint64_t* spare = kb.Alternate();
  uint64_t out_count = count;

  DevBuf<uint32_t> order_c;
  if (layout == GB_LAYOUT_DEDUPLICATED) {
    DevBuf<uint8_t> flags;
    DevBuf<uint64_t> d_num;
    GB_TRY(flags.alloc(count));
    GB_TRY(d_num.alloc(1));
    k_dedup_flags<<<grid_for(count, blk), blk, 0, s>>>(sorted, count, bits, flags.p);
    DevBuf<uint8_t> sel_tmp;
    GB_TRY(cub_call(sel_tmp, [&](void* t, size_t& tb) {
      return cub::DeviceSelect::Flagged(t, tb, sorted, flags.p, spare, d_num.p, (int64_t)count, s);
    }));
    if (order) {
      GB_TRY(order_c.alloc(count));
      // the uint32 selection has its own temporary-storage size: query it (never reuse the uint64 one)
      DevBuf<uint8_t> sel_tmp32;
      GB_TRY(cub_call(sel_tmp32, [&](void* t, size_t& tb) {
        return cub::DeviceSelect::Flagged(t, tb, order, flags.p, order_c.p, d_num.p, (int64_t)count, s);
      }));
      GB_CUDA(cudaStreamSynchronize(s));  // sel_tmp32 is released at the end of this scope
      order = order_c.p;
    }
    GB_CUDA(cudaMemcpyAsync(&out_count, d_num.p, 8, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    sorted = spare;
  }

  csr->len = out_count;
  GB_TRY(csr->tgt.alloc(out_count, 8));
  GB_CUDA(cudaMemsetAsync(csr->tgt.p + out_count, 0, 8 * 4, s));
  if (out_count) {
    k_unpack_targets<<<grid_for(out_count, blk), blk, 0, s>>>(sorted, out_count, bits, csr->tgt.p);
    if (d_w) {
      GB_TRY(csr->w.alloc(out_count, 8));
      k_gather<float><<<grid_for(out_count, blk), blk, 0, s>>>(d_w, order, out_count, csr->w.p);
    }
  } else if (d_w) {
    GB_TRY(csr->w.alloc(0, 8));
  }
  GB_TRY(offsets_from_sorted(s, RowOfKey{sorted, bits}, out_count, n, csr->off.p));
  GB_CUDA(cudaGetLastError());
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

gb_status require_device(int device) {
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0) {
    cudaGetLastError();
    return fail(GB_ERR_CUDA, "no CUDA device available: libgraph_b200 has no CPU fallback");
  }
  GB_REQUIRE(device >= 0 && device < count, "device %d out of range (have %d)", device, count);
  return GB_OK;
}

gb_status check_layout(gb_layout layout) {
  GB_REQUIRE((int)layout >= 0 && (int)layout <= 2, "bad layout %d", (int)layout);
  return GB_OK;
}

gb_status new_graph(int device, gb_graph_kind kind, uint32_t n, GraphPtr* out) {
  GB_TRY(require_device(device));
  GB_CUDA(cudaSetDevice(device));
  GraphPtr g(new (std::nothrow) gb_graph());
  if (!g) return fail(GB_ERR_OOM, "host allocation failed");
  g->device = device;
  g->kind = kind;
  g->n = n;
  cudaError_t e = cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreate(&g->ev_begin);
  if (e == cudaSuccess) e = cudaEventCreate(&g->ev_end);
  if (e != cudaSuccess) return fail(GB_ERR_CUDA, "stream/event creation failed: %s", cudaGetErrorString(e));
  *out = std::move(g);
  return GB_OK;
}

__global__ void k_check_monotone(const uint32_t* __restrict__ off, uint32_t n, unsigned int* __restrict__ bad) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x)
    if (off[v] > off[v + 1]) atomicAdd(bad, 1u);
}

void check_ids_async(cudaStream_t s, const uint32_t* a, uint64_t count, uint32_t n, unsigned int* bad) {
  if (count) k_check_ids<<<grid_for(count, 256), 256, 0, s>>>(a, count, n, bad);
}

void check_monotone_async(cudaStream_t s, const uint32_t* off, uint32_t n, unsigned int* bad) {
  k_check_monotone<<<grid_for(n, 256), 256, 0, s>>>(off, n, bad);
}

// `what` and the space after it, or nothing
#define GB_WHAT(what) (what), (*(what) ? " " : "")

gb_status require_host_csr(uint32_t n, const uint32_t* off, const uint32_t* tgt, const char* what,
                           bool offsets_only) {
  GB_REQUIRE(off != nullptr, "%s%soffsets is NULL", GB_WHAT(what));
  GB_REQUIRE(off[0] == 0, "%s%soffsets[0] must be 0", GB_WHAT(what));
  GB_REQUIRE(offsets_only || off[n] == 0 || tgt != nullptr, "%s%stargets is NULL", GB_WHAT(what));
  return GB_OK;
}

gb_status require_monotone(const char* what, uint64_t bad_rows) {
  if (!bad_rows) return GB_OK;
  return fail(GB_ERR_INVALID, "%s%soffsets are not monotone (%llu rows)", GB_WHAT(what), (unsigned long long)bad_rows);
}

gb_status require_ids(const char* what, uint64_t bad_targets, uint32_t n) {
  if (!bad_targets) return GB_OK;
  return fail(GB_ERR_INVALID, "%s%sCSR holds %llu targets >= node_count %u", GB_WHAT(what),
              (unsigned long long)bad_targets, n);
}

gb_status CsrFeed::open(int device, uint32_t rb, uint32_t re, bool peers, bool two_offsets) {
  dev = device;
  r_begin = rb;
  r_end = re;
  GB_CUDA(cudaSetDevice(dev));
  GB_CUDA(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
  GB_CUDA(cudaEventCreateWithFlags(&offsets_in, cudaEventDisableTiming));
  GB_TRY(off.alloc((size_t)(re - rb) + 1, peers));
  if (two_offsets) GB_TRY(off2.alloc((size_t)(re - rb) + 1, peers));
  return GB_OK;
}

gb_status CsrFeed::resident(uint64_t eb, uint64_t ee, uint32_t chunks, bool peers) {
  e_begin = eb;
  GB_TRY(tgt.alloc(ee - eb, peers, 8));
  GB_CUDA(cudaMemsetAsync(tgt.p + (ee - eb), 0, 8 * 4, copy));
  landed.assign(chunks, nullptr);
  for (cudaEvent_t& ev : landed) GB_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  return GB_OK;
}

gb_status CsrFeed::open_ring(uint32_t slots, uint64_t slot) {
  ring.resize(slots);
  landed.assign(slots, nullptr);
  freed.assign(slots, nullptr);
  for (uint32_t i = 0; i < slots; ++i) {
    GB_TRY(ring[i].alloc(slot, 8));
    GB_CUDA(cudaMemsetAsync(ring[i].p + slot, 0, 8 * 4, copy));
    GB_CUDA(cudaEventCreateWithFlags(&landed[i], cudaEventDisableTiming));
    GB_CUDA(cudaEventCreateWithFlags(&freed[i], cudaEventDisableTiming));
  }
  return GB_OK;
}

gb_status CsrFeed::send_offsets(const uint32_t* host_off, const uint32_t* host_off2) {
  const size_t bytes = ((size_t)(r_end - r_begin) + 1) * 4;
  GB_CUDA(cudaMemcpyAsync(off.p, host_off + r_begin, bytes, cudaMemcpyHostToDevice, copy));
  if (host_off2) GB_CUDA(cudaMemcpyAsync(off2.p, host_off2 + r_begin, bytes, cudaMemcpyHostToDevice, copy));
  GB_CUDA(cudaEventRecord(offsets_in, copy));
  return GB_OK;
}

gb_status CsrFeed::send(uint64_t k, const uint32_t* host_tgt, uint64_t e0, uint64_t len) {
  uint32_t* dst = ring.empty() ? tgt.p + (e0 - e_begin) : ring[k % ring.size()].p;
  if (!ring.empty() && k >= ring.size()) GB_CUDA(cudaStreamWaitEvent(copy, freed[k % ring.size()], 0));
  if (len) GB_CUDA(cudaMemcpyAsync(dst, host_tgt + e0, len * 4, cudaMemcpyHostToDevice, copy));
  GB_CUDA(cudaEventRecord(landed[k % landed.size()], copy));
  return GB_OK;
}

gb_status CsrFeed::check_monotone(cudaStream_t s, uint32_t r0, uint32_t r1, unsigned int* bad) const {
  GB_CUDA(cudaStreamWaitEvent(s, offsets_in, 0));
  check_monotone_async(s, off.p + (r0 - r_begin), r1 - r0, bad);
  if (off2.p) check_monotone_async(s, off2.p + (r0 - r_begin), r1 - r0, bad + 1);
  return GB_OK;
}

bool CsrFeed::pinned(const void* host) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, host) == cudaSuccess) return a.type == cudaMemoryTypeHost;
  cudaGetLastError();
  return false;
}

CsrFeed::~CsrFeed() {
  if (dev < 0) return;
  cudaSetDevice(dev);
  if (copy) cudaStreamSynchronize(copy);
  ring.clear();
  tgt.release();
  off2.release();
  off.release();
  for (const std::vector<cudaEvent_t>* events : {&landed, &freed})
    for (cudaEvent_t ev : *events)
      if (ev) cudaEventDestroy(ev);
  if (offsets_in) cudaEventDestroy(offsets_in);
  if (copy) cudaStreamDestroy(copy);
}

// Only O(1) checks read the host arrays; the O(n + m) ones run on the device after the upload, so that a
// billion-edge twin is not validated by one CPU thread.
gb_status upload_host_csr(cudaStream_t s, uint32_t n, const uint32_t* off, const uint32_t* tgt, const float* w,
                          DevCsr* csr, const char* what, bool offsets_only) {
  GB_TRY(require_host_csr(n, off, tgt, what, offsets_only));
  const uint64_t len = off[n];
  DevBuf<unsigned int> bad;  // [0] targets >= n, [1] rows whose offsets decrease
  GB_TRY(bad.alloc(2));
  GB_CUDA(cudaMemsetAsync(bad.p, 0, 8, s));
  csr->len = len;
  GB_TRY(csr->off.alloc((size_t)n + 1));
  GB_CUDA(cudaMemcpyAsync(csr->off.p, off, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, s));
  check_monotone_async(s, csr->off.p, n, bad.p + 1);
  if (!offsets_only) {
    GB_TRY(csr->tgt.alloc(len, 8));
    if (len) GB_CUDA(cudaMemcpyAsync(csr->tgt.p, tgt, len * 4, cudaMemcpyHostToDevice, s));
    GB_CUDA(cudaMemsetAsync(csr->tgt.p + len, 0, 8 * 4, s));
    if (w) {
      GB_TRY(csr->w.alloc(len, 8));
      if (len) GB_CUDA(cudaMemcpyAsync(csr->w.p, w, len * 4, cudaMemcpyHostToDevice, s));
    }
    check_ids_async(s, csr->tgt.p, len, n, bad.p);
  }
  unsigned int nbad[2] = {0, 0};
  GB_CUDA(cudaMemcpyAsync(nbad, bad.p, 8, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  GB_TRY(require_monotone(what, nbad[1]));
  return require_ids(what, nbad[0], n);
}

// builds a directed or undirected graph's CSRs from DEVICE edge arrays
static gb_status build_graph_csrs(gb_graph* g, const uint32_t* d_src, const uint32_t* d_dst, const float* d_w,
                                  uint64_t m, gb_layout layout) {
  cudaStream_t s = g->stream;
  if (g->kind == GB_KIND_DIRECTED) {
    GB_TRY(build_csr_device(s, g->n, d_src, d_dst, d_w, m, layout, &g->out));
    GB_TRY(build_csr_device(s, g->n, d_dst, d_src, nullptr, m, layout, &g->in));
  } else {
    // one CSR holding both directions: outgoing pass first, then incoming (csr.rs:154-172)
    DevBuf<uint32_t> rows, cols;
    GB_TRY(rows.alloc(2 * m));
    GB_TRY(cols.alloc(2 * m));
    if (m) {
      GB_CUDA(cudaMemcpyAsync(rows.p, d_src, m * 4, cudaMemcpyDeviceToDevice, s));
      GB_CUDA(cudaMemcpyAsync(rows.p + m, d_dst, m * 4, cudaMemcpyDeviceToDevice, s));
      GB_CUDA(cudaMemcpyAsync(cols.p, d_dst, m * 4, cudaMemcpyDeviceToDevice, s));
      GB_CUDA(cudaMemcpyAsync(cols.p + m, d_src, m * 4, cudaMemcpyDeviceToDevice, s));
    }
    GB_TRY(build_csr_device(s, g->n, rows.p, cols.p, nullptr, 2 * m, layout, &g->out));
  }
  // an Unsorted build keeps the edge-list order inside each row, which may or may not be ascending
  g->row_order = (layout == GB_LAYOUT_UNSORTED) ? RowOrder::Unknown : RowOrder::Sorted;
  return GB_OK;
}

__global__ void k_max_ids(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, uint64_t count,
                          unsigned int* __restrict__ mx) {
  uint32_t v = 0;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    v = max(v, max(a[i], b[i]));
  for (int o = 16; o; o >>= 1) v = max(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
  if ((threadIdx.x & 31) == 0) atomicMax(mx, v);
}

// the argument checks of the host and the device edge paths
static gb_status check_edge_args(gb_graph_kind kind, const uint32_t* src, const uint32_t* dst, uint64_t m,
                                 uint32_t n, gb_layout layout, gb_graph** out) {
  GB_REQUIRE(out != nullptr, "graph out-pointer is NULL");
  GB_REQUIRE(m == 0 || (src && dst), "edge arrays are NULL");
  GB_TRY(check_layout(layout));
  uint64_t cap = (kind == GB_KIND_UNDIRECTED) ? 2 * m : m;
  GB_REQUIRE(cap < 0xFFFFFFFFull, "edge count %llu does not fit u32 offsets", (unsigned long long)m);
  GB_REQUIRE(n != 0 || m > 0, "cannot infer node_count from an empty edge list");
  return GB_OK;
}

// Checks device edge arrays on g's stream, then builds g's CSRs from them.  g->n == 0 is inferred as the
// largest id + 1 (Edges::max_node_id + 1, edgelist.rs:84-90); otherwise every id must be below g->n.
static gb_status build_from_edges(gb_graph* g, const uint32_t* d_src, const uint32_t* d_dst, const float* d_w,
                                  uint64_t m, gb_layout layout) {
  cudaStream_t s = g->stream;
  const bool infer = g->n == 0;
  DevBuf<unsigned int> scratch;
  GB_TRY(scratch.alloc(1));
  GB_CUDA(cudaMemsetAsync(scratch.p, 0, 4, s));
  if (infer) {
    k_max_ids<<<grid_for(m, 256), 256, 0, s>>>(d_src, d_dst, m, scratch.p);
  } else {
    check_ids_async(s, d_src, m, g->n, scratch.p);
    check_ids_async(s, d_dst, m, g->n, scratch.p);
  }
  unsigned int h = 0;
  GB_CUDA(cudaMemcpyAsync(&h, scratch.p, 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  GB_CUDA(cudaGetLastError());
  if (infer) {
    GB_REQUIRE(h < 0xFFFFFFFFu, "node id 2^32-1 leaves no room for node_count");
    g->n = h + 1;
  } else {
    GB_REQUIRE(h == 0, "%u edge endpoints are >= node_count %u", h, g->n);
  }
  return build_graph_csrs(g, d_src, d_dst, d_w, m, layout);
}

static gb_status graph_from_host_edges(int device, gb_graph_kind kind, const uint32_t* src,
                                       const uint32_t* dst, const float* w, uint64_t m, uint32_t n,
                                       gb_layout layout, gb_graph** out) {
  GB_TRY(check_edge_args(kind, src, dst, m, n, layout, out));
  GraphPtr g;
  GB_TRY(new_graph(device, kind, n, &g));
  DevBuf<uint32_t> d_src, d_dst;
  DevBuf<float> d_w;
  GB_TRY(d_src.alloc(m));
  GB_TRY(d_dst.alloc(m));
  if (w) GB_TRY(d_w.alloc(m));
  if (m) {
    GB_CUDA(cudaMemcpyAsync(d_src.p, src, m * 4, cudaMemcpyHostToDevice, g->stream));
    GB_CUDA(cudaMemcpyAsync(d_dst.p, dst, m * 4, cudaMemcpyHostToDevice, g->stream));
    if (w) GB_CUDA(cudaMemcpyAsync(d_w.p, w, m * 4, cudaMemcpyHostToDevice, g->stream));
  }
  GB_TRY(build_from_edges(g.get(), d_src.p, d_dst.p, d_w.p, m, layout));
  *out = g.release();
  return GB_OK;
}

static gb_status require_device_array(const void* p, int device, const char* what) {
  cudaPointerAttributes a{};
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return fail(GB_ERR_INVALID, "%s is not a device pointer", what);
  }
  GB_REQUIRE((a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) && a.device == device,
             "%s is not device memory of device %d", what, device);
  return GB_OK;
}

gb_status graph_from_device_arrays(int device, gb_graph_kind kind, const uint32_t* d_src, const uint32_t* d_dst,
                                   const float* d_w, uint64_t m, uint32_t n, gb_layout layout, cudaStream_t caller,
                                   gb_graph** out) {
  GB_TRY(check_edge_args(kind, d_src, d_dst, m, n, layout, out));
  GraphPtr g;
  GB_TRY(new_graph(device, kind, n, &g));
  if (m) {
    GB_TRY(require_device_array(d_src, device, "d_src"));
    GB_TRY(require_device_array(d_dst, device, "d_dst"));
    if (d_w) GB_TRY(require_device_array(d_w, device, "d_weights"));
  }
  // the caller's producer work comes first
  cudaEvent_t ready;
  GB_CUDA(cudaEventCreateWithFlags(&ready, cudaEventDisableTiming));
  cudaError_t e = cudaEventRecord(ready, caller);
  if (e == cudaSuccess) e = cudaStreamWaitEvent(g->stream, ready, 0);
  cudaEventDestroy(ready);
  GB_CUDA(e);
  GB_TRY(build_from_edges(g.get(), d_src, d_dst, d_w, m, layout));
  *out = g.release();
  return GB_OK;
}

__global__ void k_count_diff(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, uint64_t count,
                             unsigned int* __restrict__ bad) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    if (a[i] != b[i]) atomicAdd(bad, 1u);
}

__global__ void k_scatter_values(const float* __restrict__ w, const uint32_t* __restrict__ pos, uint64_t count,
                                 float* __restrict__ out) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x)
    out[pos[i]] = w[i];
}

// Both CSRs are re-sorted by (t, s) with the stable build: the out-CSR's entries, transposed, carry their
// values, and equal keys stay in out-row order; the in-CSR's entries carry their position, and equal keys stay
// in in-row order.  Equal key sequences pair the k-th occurrences, and the values are scattered by position.
gb_status in_csr_values(const gb_graph* g, DevBuf<float>* in_w) {
  cudaStream_t s = g->stream;
  const uint32_t n = g->n;
  const uint64_t m = g->out.len;
  GB_REQUIRE(g->in.len == m && g->in.tgt.p && g->out.w.p, "the graph has no weighted out-CSR and in-CSR pair");
  GB_TRY(in_w->alloc(m, 8));
  if (m == 0) return GB_OK;
  DevBuf<uint32_t> rows, pos;
  GB_TRY(rows.alloc(m));
  GB_TRY(pos.alloc(m));
  const unsigned grid_rows = grid_for((uint64_t)n * 32, 256);
  k_expand_rows<<<grid_rows, 256, 0, s>>>(g->out.off.p, n, rows.p);
  DevCsr tr;  // rows t, targets s, out values
  GB_TRY(build_csr_device(s, n, g->out.tgt.p, rows.p, g->out.w.p, m, GB_LAYOUT_SORTED, &tr));
  k_expand_rows<<<grid_rows, 256, 0, s>>>(g->in.off.p, n, rows.p);
  k_iota<<<grid_for(m, 256), 256, 0, s>>>(pos.p, m);
  DevCsr in;  // rows t, targets s, in-CSR positions (the build moves the 32-bit "values" without reading them)
  GB_TRY(build_csr_device(s, n, rows.p, g->in.tgt.p, reinterpret_cast<const float*>(pos.p), m, GB_LAYOUT_SORTED,
                          &in));
  DevBuf<unsigned int> bad;
  GB_TRY(bad.alloc(1));
  GB_CUDA(cudaMemsetAsync(bad.p, 0, 4, s));
  k_count_diff<<<grid_for((uint64_t)n + 1, 256), 256, 0, s>>>(tr.off.p, in.off.p, (uint64_t)n + 1, bad.p);
  k_count_diff<<<grid_for(m, 256), 256, 0, s>>>(tr.tgt.p, in.tgt.p, m, bad.p);
  k_scatter_values<<<grid_for(m, 256), 256, 0, s>>>(tr.w.p, reinterpret_cast<const uint32_t*>(in.w.p), m, in_w->p);
  GB_CUDA(cudaGetLastError());
  unsigned int h = 0;
  GB_CUDA(cudaMemcpyAsync(&h, bad.p, 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  GB_REQUIRE(h == 0, "the in-CSR is not the transpose of the out-CSR: no in-CSR values can be written");
  return GB_OK;
}

template <typename T>
__global__ void k_ids_to_u32(const T* __restrict__ in, uint64_t count, uint32_t* __restrict__ out,
                             unsigned int* __restrict__ bad) {
  bool b = false;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count;
       i += (uint64_t)gridDim.x * blockDim.x) {
    const long long v = (long long)in[i];
    b |= v < 0 || v > 0xFFFFFFFFll;
    out[i] = (uint32_t)v;
  }
  if (__any_sync(0xFFFFFFFFu, b) && (threadIdx.x & 31) == 0) atomicOr(bad, 1u);
}

static gb_status rmat_graph(int device, gb_graph_kind kind, uint32_t scale, uint32_t edge_factor,
                            uint64_t seed, gb_layout layout, int weights, gb_graph** out) {
  GB_REQUIRE(out != nullptr, "graph out-pointer is NULL");
  GB_REQUIRE(scale >= 1 && scale <= 31, "scale %u out of range [1,31]", scale);
  GB_REQUIRE(edge_factor >= 1, "edge_factor must be >= 1");
  uint64_t m = (uint64_t)edge_factor << scale;
  uint64_t cap = (kind == GB_KIND_UNDIRECTED) ? 2 * m : m;
  GB_REQUIRE(cap < 0xFFFFFFFFull, "2^%u * %u edges do not fit u32 offsets", scale, edge_factor);
  GraphPtr g;
  GB_TRY(new_graph(device, kind, 1u << scale, &g));
  DevBuf<uint32_t> d_src, d_dst;
  DevBuf<float> d_w;
  GB_TRY(d_src.alloc(m));
  GB_TRY(d_dst.alloc(m));
  k_rmat<<<grid_for(m, 256), 256, 0, g->stream>>>(scale, seed, 0, m, d_src.p, d_dst.p);
  if (weights && kind == GB_KIND_DIRECTED) {
    GB_TRY(d_w.alloc(m));
    k_rmat_weights<<<grid_for(m, 256), 256, 0, g->stream>>>(seed, m, d_w.p);
  }
  GB_CUDA(cudaGetLastError());
  GB_TRY(build_graph_csrs(g.get(), d_src.p, d_dst.p, d_w.p, m, layout));
  *out = g.release();
  return GB_OK;
}

}  // namespace gb

using namespace gb;

// ---- C ABI ---------------------------------------------------------------------------------
extern "C" {

int gb_abi_version(void) { return GB_ABI_VERSION; }
const char* gb_last_error(void) { return last_error().c_str(); }
int gb_device_count(void) {
  int c = 0;
  if (cudaGetDeviceCount(&c) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return c;
}
void gb_set_profiling(int on) { gb::g_profiling = on != 0; }

gb_status gb_digraph_from_csr_u32(int device, uint32_t n, const uint32_t* out_off,
                                  const uint32_t* out_tgt, const float* out_w, const uint32_t* in_off,
                                  const uint32_t* in_tgt, gb_graph** graph) {
  GB_REQUIRE(graph != nullptr, "graph out-pointer is NULL");
  GB_REQUIRE(n > 0, "node_count must be > 0");
  GraphPtr g;
  GB_TRY(new_graph(device, GB_KIND_DIRECTED, n, &g));
  GB_TRY(upload_host_csr(g->stream, n, out_off, out_tgt, out_w, &g->out, "out"));
  GB_TRY(upload_host_csr(g->stream, n, in_off, in_tgt, nullptr, &g->in, "in"));
  GB_REQUIRE(g->out.len == g->in.len, "out and in CSR disagree on the edge count");
  *graph = g.release();
  return GB_OK;
}

gb_status gb_graph_from_csr_u32(int device, uint32_t n, const uint32_t* off, const uint32_t* tgt,
                                gb_graph** graph) {
  GB_REQUIRE(graph != nullptr, "graph out-pointer is NULL");
  GB_REQUIRE(n > 0, "node_count must be > 0");
  GraphPtr g;
  GB_TRY(new_graph(device, GB_KIND_UNDIRECTED, n, &g));
  GB_TRY(upload_host_csr(g->stream, n, off, tgt, nullptr, &g->out, "undirected"));
  *graph = g.release();
  return GB_OK;
}

gb_status gb_digraph_from_edges_u32(int device, const uint32_t* src, const uint32_t* dst,
                                    const float* weights, uint64_t m, uint32_t n, gb_layout layout,
                                    gb_graph** graph) {
  return graph_from_host_edges(device, GB_KIND_DIRECTED, src, dst, weights, m, n, layout, graph);
}

gb_status gb_graph_from_edges_u32(int device, const uint32_t* src, const uint32_t* dst, uint64_t m,
                                  uint32_t n, gb_layout layout, gb_graph** graph) {
  return graph_from_host_edges(device, GB_KIND_UNDIRECTED, src, dst, nullptr, m, n, layout, graph);
}

gb_status gb_digraph_from_device_edges_u32(int device, const uint32_t* d_src, const uint32_t* d_dst,
                                           const float* d_weights, uint64_t m, uint32_t n, gb_layout layout,
                                           void* stream, gb_graph** graph) {
  return graph_from_device_arrays(device, GB_KIND_DIRECTED, d_src, d_dst, d_weights, m, n, layout,
                                  static_cast<cudaStream_t>(stream), graph);
}

gb_status gb_graph_from_device_edges_u32(int device, const uint32_t* d_src, const uint32_t* d_dst, uint64_t m,
                                         uint32_t n, gb_layout layout, void* stream, gb_graph** graph) {
  return graph_from_device_arrays(device, GB_KIND_UNDIRECTED, d_src, d_dst, nullptr, m, n, layout,
                                  static_cast<cudaStream_t>(stream), graph);
}

gb_status gb_ids_to_u32(int device, const void* d_ids, int id_bytes, uint64_t count, uint32_t* d_out,
                        void* stream) {
  GB_REQUIRE(id_bytes == 4 || id_bytes == 8, "ids must be 4 or 8 bytes wide, not %d", id_bytes);
  if (count == 0) return GB_OK;
  GB_REQUIRE(d_ids && d_out, "NULL argument");
  GB_TRY(require_device(device));
  DeviceGuard guard(device);
  GB_TRY(require_device_array(d_ids, device, "ids"));
  GB_TRY(require_device_array(d_out, device, "output ids"));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DevBuf<unsigned int> bad;
  GB_TRY(bad.alloc(1));
  GB_CUDA(cudaMemsetAsync(bad.p, 0, 4, s));
  if (id_bytes == 4)
    k_ids_to_u32<int32_t><<<grid_for(count, 256), 256, 0, s>>>(static_cast<const int32_t*>(d_ids), count, d_out, bad.p);
  else
    k_ids_to_u32<int64_t><<<grid_for(count, 256), 256, 0, s>>>(static_cast<const int64_t*>(d_ids), count, d_out, bad.p);
  GB_CUDA(cudaGetLastError());
  unsigned int h = 0;
  GB_CUDA(cudaMemcpyAsync(&h, bad.p, 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  GB_REQUIRE(h == 0, "node ids must be 32-bit unsigned integers");
  return GB_OK;
}

gb_status gb_digraph_rmat(int device, uint32_t scale, uint32_t edge_factor, uint64_t seed,
                          gb_layout layout, int weights, gb_graph** graph) {
  return rmat_graph(device, GB_KIND_DIRECTED, scale, edge_factor, seed, layout, weights, graph);
}
gb_status gb_graph_rmat(int device, uint32_t scale, uint32_t edge_factor, uint64_t seed,
                        gb_layout layout, gb_graph** graph) {
  return rmat_graph(device, GB_KIND_UNDIRECTED, scale, edge_factor, seed, layout, 0, graph);
}

gb_status gb_rmat_edges(int device, uint32_t scale, uint64_t seed, uint64_t first, uint64_t count,
                        uint32_t* src, uint32_t* dst) {
  GB_REQUIRE(scale >= 1 && scale <= 31, "scale %u out of range [1,31]", scale);
  GB_REQUIRE(count == 0 || (src && dst), "output arrays are NULL");
  GB_TRY(require_device(device));
  DeviceGuard guard(device);
  DevBuf<uint32_t> d_src, d_dst;
  GB_TRY(d_src.alloc(count));
  GB_TRY(d_dst.alloc(count));
  if (count) {
    k_rmat<<<grid_for(count, 256), 256>>>(scale, seed, first, count, d_src.p, d_dst.p);
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaMemcpy(src, d_src.p, count * 4, cudaMemcpyDeviceToHost));
    GB_CUDA(cudaMemcpy(dst, d_dst.p, count * 4, cudaMemcpyDeviceToHost));
  }
  return GB_OK;
}

gb_status gb_graph_free(gb_graph* g) {
  if (!g) return GB_OK;
  DeviceGuard guard(g->device);
  if (g->stream) cudaStreamSynchronize(g->stream);
  if (g->pr_plan) free_pr_plan(g->pr_plan);
  g->out = DevCsr();
  g->in = DevCsr();
  if (g->ev_begin) cudaEventDestroy(g->ev_begin);
  if (g->ev_end) cudaEventDestroy(g->ev_end);
  if (g->stream) cudaStreamDestroy(g->stream);
  delete g;
  return GB_OK;
}

gb_status gb_graph_get_info(const gb_graph* g, gb_graph_info* info) {
  GB_REQUIRE(g && info, "NULL argument");
  info->kind = (uint32_t)g->kind;
  info->node_count = g->n;
  info->target_count = g->out.len;
  info->edge_count = (g->kind == GB_KIND_UNDIRECTED) ? g->out.len / 2 : g->out.len;
  info->has_weights = g->out.w.p != nullptr;
  info->device = g->device;
  info->device_bytes = g->out.bytes() + g->in.bytes() + pr_plan_bytes(g->pr_plan);
  return GB_OK;
}

static const DevCsr* pick_csr(const gb_graph* g, gb_csr_which which) {
  if (g->kind == GB_KIND_DIRECTED) {
    if (which == GB_CSR_OUT) return &g->out;
    if (which == GB_CSR_IN) return &g->in;
    return nullptr;
  }
  return which == GB_CSR_UNDIRECTED ? &g->out : nullptr;
}

gb_status gb_graph_csr_len(const gb_graph* g, gb_csr_which which, uint64_t* len) {
  GB_REQUIRE(g && len, "NULL argument");
  const DevCsr* c = pick_csr(g, which);
  if (!c) return fail(GB_ERR_UNSUPPORTED, "graph kind %d has no CSR %d", (int)g->kind, (int)which);
  *len = c->len;
  return GB_OK;
}

gb_status gb_graph_copy_csr(const gb_graph* g, gb_csr_which which, uint32_t* off, uint32_t* tgt,
                            float* w) {
  GB_REQUIRE(g && off, "NULL argument");
  const DevCsr* c = pick_csr(g, which);
  if (!c) return fail(GB_ERR_UNSUPPORTED, "graph kind %d has no CSR %d", (int)g->kind, (int)which);
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  GB_CUDA(cudaMemcpyAsync(off, c->off.p, ((size_t)g->n + 1) * 4, cudaMemcpyDeviceToHost, g->stream));
  if (tgt && c->len) {
    GB_REQUIRE(c->tgt.p != nullptr, "this handle holds no targets for that CSR (page-rank-only twin)");
    GB_CUDA(cudaMemcpyAsync(tgt, c->tgt.p, c->len * 4, cudaMemcpyDeviceToHost, g->stream));
  }
  if (w) {
    GB_REQUIRE(c->w.p != nullptr, "this CSR carries no edge values");
    if (c->len) GB_CUDA(cudaMemcpyAsync(w, c->w.p, c->len * 4, cudaMemcpyDeviceToHost, g->stream));
  }
  GB_CUDA(cudaStreamSynchronize(g->stream));
  return GB_OK;
}

void* gb_graph_stream(const gb_graph* g) { return g ? (void*)g->stream : nullptr; }

gb_status gb_graph_last_timing(const gb_graph* g, gb_timing* t) {
  GB_REQUIRE(g && t, "NULL argument");
  *t = g->timing;
  return GB_OK;
}

// to_undirected: csr.rs:391-464 — every out-edge (u, v) of the directed graph becomes an edge of a
// fresh UndirectedCsrGraph, fed in out-CSR order.
gb_status gb_to_undirected(const gb_graph* dg, gb_layout layout, gb_graph** graph) {
  GB_REQUIRE(dg && graph, "NULL argument");
  if (dg->kind != GB_KIND_DIRECTED) return fail(GB_ERR_UNSUPPORTED, "to_undirected needs a directed graph");
  GB_TRY(check_layout(layout));
  uint64_t m = dg->out.len;
  GB_REQUIRE(m == 0 || dg->out.tgt.p != nullptr, "this handle holds no out targets (page-rank-only twin)");
  GB_REQUIRE(2 * m < 0xFFFFFFFFull, "undirected twin would exceed u32 offsets");
  DeviceGuard guard(dg->device);
  GraphPtr g;
  GB_TRY(new_graph(dg->device, GB_KIND_UNDIRECTED, dg->n, &g));
  std::lock_guard<std::mutex> lock(dg->mu);
  DevBuf<uint32_t> rows;
  GB_TRY(rows.alloc(m));
  if (m) k_expand_rows<<<grid_for((uint64_t)dg->n * 32, 256), 256, 0, g->stream>>>(dg->out.off.p, dg->n, rows.p);
  GB_CUDA(cudaGetLastError());
  GB_TRY(build_graph_csrs(g.get(), rows.p, dg->out.tgt.p, nullptr, m, layout));
  *graph = g.release();
  return GB_OK;
}

// make_degree_ordered: graph_ops.rs:511-638.  (degree, id) pairs sorted descending (:555), so
// ties give the larger old id the smaller new id; rows rewritten and sorted ascending (:629).
gb_status gb_make_degree_ordered(gb_graph* g) {
  GB_REQUIRE(g != nullptr, "NULL graph");
  if (g->kind != GB_KIND_UNDIRECTED)
    return fail(GB_ERR_UNSUPPORTED, "make_degree_ordered is defined for undirected graphs (graph_ops.rs:240-253)");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  cudaStream_t s = g->stream;
  const uint32_t n = g->n;
  const uint64_t len = g->out.len;
  const uint32_t bits = bits_for(n);
  DevBuf<uint64_t> dk, dk_alt;
  GB_TRY(dk.alloc(n));
  GB_TRY(dk_alt.alloc(n));
  k_degree_keys<<<grid_for(n, 256), 256, 0, s>>>(g->out.off.p, n, dk.p);
  cub::DoubleBuffer<uint64_t> db(dk.p, dk_alt.p);
  DevBuf<uint8_t> tmp;
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceRadixSort::SortKeysDescending(t, tb, db, (int)n, 0, 64, s);
  }));
  DevBuf<uint32_t> new_id, new_deg, rows;
  GB_TRY(new_id.alloc(n));
  GB_TRY(new_deg.alloc(n));
  k_rank_to_newid<<<grid_for(n, 256), 256, 0, s>>>(db.Current(), n, new_id.p, new_deg.p);
  DevCsr fresh;
  GB_TRY(fresh.off.alloc((size_t)n + 1));
  GB_TRY(fresh.tgt.alloc(len, 8));
  fresh.len = len;
  GB_CUDA(cudaMemsetAsync(fresh.tgt.p + len, 0, 8 * 4, s));
  if (len) {
    GB_TRY(rows.alloc(len));
    k_expand_rows<<<grid_for((uint64_t)n * 32, 256), 256, 0, s>>>(g->out.off.p, n, rows.p);
    DevBuf<uint64_t> keys, keys_alt;
    GB_TRY(keys.alloc(len));
    GB_TRY(keys_alt.alloc(len));
    k_relabel_keys<<<grid_for(len, 256), 256, 0, s>>>(rows.p, g->out.tgt.p, new_id.p, len, bits, keys.p);
    cub::DoubleBuffer<uint64_t> kb(keys.p, keys_alt.p);
    DevBuf<uint8_t> stmp;
    GB_TRY(cub_call(stmp, [&](void* t, size_t& tb) {
      return cub::DeviceRadixSort::SortKeys(t, tb, kb, len, 0, (int)(2 * bits), s);
    }));
    k_unpack_targets<<<grid_for(len, 256), 256, 0, s>>>(kb.Current(), len, bits, fresh.tgt.p);
    GB_TRY(offsets_from_sorted(s, RowOfKey{kb.Current(), bits}, len, n, fresh.off.p));
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaStreamSynchronize(s));
  } else {
    GB_CUDA(cudaMemsetAsync(fresh.off.p, 0, ((size_t)n + 1) * 4, s));
    GB_CUDA(cudaStreamSynchronize(s));
  }
  g->out = std::move(fresh);  // SwapCsr::swap_csr, csr.rs:120-122
  g->row_order = RowOrder::Sorted;  // the (row, target) keys were sorted above
  return GB_OK;
}

// in_degree_partition: graph_ops.rs:431-439 + greedy_node_map_partition :479-509
gb_status gb_in_degree_partition(const gb_graph* g, uint32_t parts, uint32_t* ranges) {
  GB_REQUIRE(g && ranges, "NULL argument");
  GB_REQUIRE(parts >= 1, "parts must be >= 1");
  if (g->kind != GB_KIND_DIRECTED) return fail(GB_ERR_UNSUPPORTED, "in_degree_partition needs a directed graph");
  DeviceGuard guard(g->device);
  std::vector<uint32_t> off((size_t)g->n + 1);
  {
    std::lock_guard<std::mutex> lock(g->mu);
    GB_CUDA(cudaMemcpyAsync(off.data(), g->in.off.p, off.size() * 4, cudaMemcpyDeviceToHost, g->stream));
    GB_CUDA(cudaStreamSynchronize(g->stream));
  }
  const uint64_t m = g->in.len;
  const uint64_t batch = (m + parts - 1) / parts;  // ceil(m / parts)
  uint32_t count = 0;
  uint64_t acc = 0;
  ranges[0] = 0;
  for (uint32_t v = 0; v < g->n; ++v) {
    acc += off[v + 1] - off[v];
    if ((count < parts - 1 && acc >= batch) || v == g->n - 1) {
      ranges[++count] = v + 1;
      acc = 0;
    }
  }
  for (uint32_t i = count + 1; i <= parts; ++i) ranges[i] = g->n;  // unused trailing ranges are empty
  return GB_OK;
}

}  // extern "C"
