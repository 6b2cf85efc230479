// adj_list.cu — device twins of the reference's adjacency-list graphs, their batched edge insertion and their
// snapshot into an immutable gb_graph.
//
//   AdjacencyList::from((&edges, n, direction, layout))   crates/builder/src/graph/adj_list.rs:216-277
//   DirectedALGraph{al_out, al_inc}                        adj_list.rs:279-450
//   UndirectedALGraph{al}                                  adj_list.rs:452-595
//   add_edge / add_edge_with_value + apply_layout          adj_list.rs:371-404, :524-557, :81-94
//
// Storage.  Each list (out and in, or the one undirected list) keeps per row a 64-bit start, a u32 len and a u32
// cap into a target pool (and a value pool for weighted graphs); the pool hands out [0, bump) to rows and keeps
// [bump, pool) free at its tail.  A fresh list is the CSR build_csr_device makes (start = offset, cap = len) plus
// a free tail.  A batch moves every row it overfills to the tail with max(2 cap, new len) entries; when the tail
// cannot take them the pool is rebuilt compacted, every row keeping its (new) capacity, with as many free entries
// again at the tail.  DESIGN.md §10 gives the cost and byte model.
//
// A batch of k edges leaves exactly the rows k add_edge calls in batch order leave.  Its entries (one per list and
// edge, two per edge for an undirected list, interleaved as add_edge pushes them) are stable-sorted by row, or by
// (row, target) for Sorted and Deduplicated lists, carrying their batch position; Deduplicated drops entries whose
// target the row already holds or an earlier entry of the batch brings.  Unsorted rows get the new entries at
// len + j.  Sorted rows are merged by rank into a scratch run and copied back: new entry j of a row's run goes to
// upper_bound(row, t) + j, existing entry i to i + #(new entries < its target), which puts a new entry after the
// equal ones already there.  Every kernel walks entries, not rows, so a hub row is spread over the whole grid.
#include <cub/cub.cuh>

#include "common.cuh"

namespace gb {

constexpr uint64_t AL_MIN_TAIL = 1ull << 16;      // free tail entries of a fresh or compacted pool, at least
constexpr uint64_t AL_MAX_ENTRIES = 0xFFFFFFFFull;  // a list's entries stay below 2^32 - 1 (u32 snapshot offsets)
constexpr uint64_t AL_MAX_BATCH = 0x7FFFFFFFull;    // list entries of one batch: the run-length encode counts in int

struct AlList {
  DevBuf<uint64_t> start;     // [n]
  DevBuf<uint32_t> len, cap;  // [n]
  DevBuf<uint32_t> tgt;       // [pool] + 8 zeroed
  DevBuf<float> w;            // [pool] for weighted graphs
  uint64_t pool = 0, bump = 0, entries = 0;
  uint64_t bytes() const { return start.bytes() + len.bytes() + cap.bytes() + tgt.bytes() + w.bytes(); }
};

}  // namespace gb

struct gb_algraph {
  int device = 0;
  gb_graph_kind kind = GB_KIND_DIRECTED;
  gb_layout layout = GB_LAYOUT_UNSORTED;
  bool values = false;
  uint32_t n = 0;
  gb::AlList list[2];  // directed: out, in; undirected: list[0]
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_begin = nullptr, ev_end = nullptr, ev_cbegin = nullptr, ev_cend = nullptr;
  mutable std::mutex mu;  // every call on the handle holds it: a batch is atomic for readers
  gb_algraph_batch_info last{};
  uint64_t compactions = 0;
  gb_load_info load{};
  int lists() const { return kind == GB_KIND_DIRECTED ? 2 : 1; }
};

namespace gb {

// ---- kernels --------------------------------------------------------------------------------------------------
#define GB_GRID_LOOP(i, count)                                                     \
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < (count); \
       i += (uint64_t)gridDim.x * blockDim.x)

// the run r < R with prefix[r] <= e < prefix[r + 1] (prefix[0] = 0 <= e < prefix[R])
__device__ __forceinline__ uint32_t run_of(const uint64_t* __restrict__ prefix, uint32_t R, uint64_t e) {
  uint32_t lo = 0, hi = R;
  while (hi - lo > 1) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (prefix[mid] <= e) lo = mid;
    else hi = mid;
  }
  return lo;
}
// #a[i] < t (lower) or #a[i] <= t (upper) of an ascending a[0, len)
template <bool Upper>
__device__ __forceinline__ uint32_t rank_in(const uint32_t* __restrict__ a, uint32_t len, uint32_t t) {
  uint32_t lo = 0, hi = len;
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (Upper ? a[mid] <= t : a[mid] < t) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// edge i -> entries 2i = (s, t) and 2i + 1 = (t, s): add_edge's order on an undirected list (adj_list.rs:234-247)
__global__ void k_al_interleave(const uint32_t* __restrict__ src, const uint32_t* __restrict__ dst, uint64_t m,
                                uint32_t* __restrict__ rows, uint32_t* __restrict__ cols) {
  GB_GRID_LOOP(i, m) {
    const uint32_t s = src[i], t = dst[i];
    rows[2 * i] = s;
    cols[2 * i] = t;
    rows[2 * i + 1] = t;
    cols[2 * i + 1] = s;
  }
}

__global__ void k_al_rows_from_offsets(const uint32_t* __restrict__ off, uint32_t n, uint64_t* __restrict__ start,
                                       uint32_t* __restrict__ len, uint32_t* __restrict__ cap) {
  GB_GRID_LOOP(v, n) {
    const uint32_t b = off[v], e = off[v + 1];
    start[v] = b;
    len[v] = cap[v] = e - b;
  }
}

// the first edge of the batch with an endpoint >= n (~0 when none): the message names the first bad edge
__global__ void k_al_first_bad(const uint32_t* __restrict__ src, const uint32_t* __restrict__ dst, uint64_t count,
                               uint32_t n, unsigned long long* __restrict__ first) {
  GB_GRID_LOOP(i, count)
    if (src[i] >= n || dst[i] >= n) atomicMin(first, (unsigned long long)i);
}

// Entry e of a list's batch stream as a (row << bits | target) key and its position e.  pairs: the undirected
// stream (entry 2i = edge i as is, 2i + 1 = edge i reversed); otherwise entry e is edge e, reversed for an in-list.
__global__ void k_al_batch_keys(const uint32_t* __restrict__ src, const uint32_t* __restrict__ dst, uint64_t count,
                                uint32_t bits, bool reversed, bool pairs, uint64_t* __restrict__ keys,
                                uint32_t* __restrict__ pos) {
  GB_GRID_LOOP(e, count) {
    const uint64_t k = pairs ? e >> 1 : e;
    const bool rev = pairs ? (e & 1) != 0 : reversed;
    const uint32_t s = src[k], t = dst[k];
    keys[e] = rev ? ((uint64_t)t << bits) | s : ((uint64_t)s << bits) | t;
    pos[e] = (uint32_t)e;
  }
}

// Deduplicated: keep the first entry of each (row, target) run of the batch unless the row holds the target
__global__ void k_al_dedup_flags(const uint64_t* __restrict__ keys, uint64_t count, uint32_t bits,
                                 const uint64_t* __restrict__ start, const uint32_t* __restrict__ len,
                                 const uint32_t* __restrict__ tgt, uint8_t* __restrict__ flags) {
  const uint64_t mask = (bits >= 32) ? 0xFFFFFFFFull : ((1ull << bits) - 1ull);
  GB_GRID_LOOP(q, count) {
    const uint64_t k = keys[q];
    bool keep = q == 0 || keys[q - 1] != k;
    if (keep) {
      const uint32_t v = (uint32_t)(k >> bits), t = (uint32_t)(k & mask);
      const uint32_t* row = tgt + start[v];
      const uint32_t L = len[v];
      const uint32_t i = rank_in<false>(row, L, t);
      keep = !(i < L && row[i] == t);
    }
    flags[q] = keep ? 1 : 0;
  }
}

__global__ void k_al_unpack(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ pos, uint64_t count,
                            uint32_t bits, const float* __restrict__ w, uint32_t w_shift, uint32_t* __restrict__ rows,
                            uint32_t* __restrict__ cols, float* __restrict__ vals) {
  const uint64_t mask = (bits >= 32) ? 0xFFFFFFFFull : ((1ull << bits) - 1ull);
  GB_GRID_LOOP(q, count) {
    const uint64_t k = keys[q];
    rows[q] = (uint32_t)(k >> bits);
    cols[q] = (uint32_t)(k & mask);
    if (w) vals[q] = w[pos[q] >> w_shift];
  }
}

// Per run r (row U[r] gets C[r] entries): the values the scans below turn into offsets, element R being 0.
//   run_off <- C, ex_off <- len, sc_off <- new len, tail_off <- new cap of a moved row (else 0),
//   cp_off <- len of a moved row (else 0); rstart = the row's start, rcap = its new cap.
struct AlPlan {
  uint64_t *run_off, *ex_off, *sc_off, *tail_off, *cp_off, *rstart, *dst;
  uint32_t* rcap;
};
__global__ void k_al_plan(const uint32_t* __restrict__ U, const uint32_t* __restrict__ C, uint32_t R,
                          const uint64_t* __restrict__ start, const uint32_t* __restrict__ len,
                          const uint32_t* __restrict__ cap, AlPlan p, unsigned long long* __restrict__ moved) {
  GB_GRID_LOOP(r, (uint64_t)R + 1) {
    if (r == R) {
      p.run_off[R] = p.ex_off[R] = p.sc_off[R] = p.tail_off[R] = p.cp_off[R] = 0;
      continue;
    }
    const uint32_t v = U[r], c = C[r], L = len[v], K = cap[v];
    const uint64_t nl = (uint64_t)L + c;
    const bool move = nl > K;
    unsigned long long ncap = K;
    if (move) {
      ncap = 2ull * K > nl ? 2ull * K : (unsigned long long)nl;
      if (ncap > AL_MAX_ENTRIES) ncap = AL_MAX_ENTRIES;
    }
    p.run_off[r] = c;
    p.ex_off[r] = L;
    p.sc_off[r] = nl;
    p.tail_off[r] = move ? ncap : 0;
    p.cp_off[r] = move ? L : 0;
    p.rstart[r] = start[v];
    p.rcap[r] = (uint32_t)ncap;
    if (move) atomicAdd(moved, 1ull);
  }
}

// where each run's row ends up without a compaction: the tail for a moved row, its place otherwise
__global__ void k_al_dst_tail(AlPlan p, uint32_t R, uint64_t bump) {
  GB_GRID_LOOP(r, R) p.dst[r] = (p.tail_off[r + 1] > p.tail_off[r]) ? bump + p.tail_off[r] : p.rstart[r];
}

// after a compaction every row is in place with its new capacity
__global__ void k_al_dst_start(const uint32_t* __restrict__ U, uint32_t R, const uint64_t* __restrict__ start,
                               AlPlan p) {
  GB_GRID_LOOP(r, R) p.rstart[r] = p.dst[r] = start[U[r]];
}

// caps[v] (u64) = the capacity row v keeps through the compaction; caps[n] = 0 for the scan
__global__ void k_al_widen(const uint32_t* __restrict__ a, uint32_t n, uint64_t* __restrict__ out) {
  GB_GRID_LOOP(v, (uint64_t)n + 1) out[v] = v < n ? a[v] : 0;
}
__global__ void k_al_set_caps(const uint32_t* __restrict__ U, uint32_t R, const uint32_t* __restrict__ rcap,
                              uint64_t* __restrict__ caps) {
  GB_GRID_LOOP(r, R) caps[U[r]] = rcap[r];
}

// Copies runs of entries: entry i of run r goes from src[src_start[r] + i] to dst[dst_start[r] + i], for
// prefix[r] + i < prefix[r + 1].  One thread per entry, so a long run is spread over the grid.
__global__ void k_al_copy_runs(const uint64_t* __restrict__ prefix, uint32_t R, const uint64_t* __restrict__ src_start,
                               const uint64_t* __restrict__ dst_start, uint64_t total, const uint32_t* __restrict__ st,
                               const float* __restrict__ sw, uint32_t* __restrict__ dt, float* __restrict__ dw) {
  GB_GRID_LOOP(e, total) {
    const uint32_t r = run_of(prefix, R, e);
    const uint64_t i = e - prefix[r];
    const uint64_t a = src_start[r] + i, b = dst_start[r] + i;
    dt[b] = st[a];
    if (sw) dw[b] = sw[a];
  }
}

// Unsorted: new entry j of run r goes to the row's len + j (adj_list.rs:87, push)
__global__ void k_al_append(AlPlan p, uint32_t R, const uint32_t* __restrict__ cols, const float* __restrict__ vals,
                            uint64_t count, uint32_t* __restrict__ tgt, float* __restrict__ w) {
  GB_GRID_LOOP(q, count) {
    const uint32_t r = run_of(p.run_off, R, q);
    const uint64_t b = p.dst[r] + (p.ex_off[r + 1] - p.ex_off[r]) + (q - p.run_off[r]);
    tgt[b] = cols[q];
    if (w) w[b] = vals[q];
  }
}

// Sorted / Deduplicated merge by rank into the scratch run sc_off[r] (adj_list.rs:83-91, binary_search + insert)
__global__ void k_al_merge_old(AlPlan p, uint32_t R, uint64_t total, const uint32_t* __restrict__ cols,
                               const uint32_t* __restrict__ tgt, const float* __restrict__ w,
                               uint32_t* __restrict__ st, float* __restrict__ sw) {
  GB_GRID_LOOP(e, total) {
    const uint32_t r = run_of(p.ex_off, R, e);
    const uint64_t i = e - p.ex_off[r];
    const uint64_t a = p.rstart[r] + i;
    const uint32_t t = tgt[a];
    const uint32_t c = (uint32_t)(p.run_off[r + 1] - p.run_off[r]);
    const uint64_t b = p.sc_off[r] + i + rank_in<false>(cols + p.run_off[r], c, t);
    st[b] = t;
    if (w) sw[b] = w[a];
  }
}
__global__ void k_al_merge_new(AlPlan p, uint32_t R, uint64_t count, const uint32_t* __restrict__ cols,
                               const float* __restrict__ vals, const uint32_t* __restrict__ tgt,
                               uint32_t* __restrict__ st, float* __restrict__ sw) {
  GB_GRID_LOOP(q, count) {
    const uint32_t r = run_of(p.run_off, R, q);
    const uint32_t L = (uint32_t)(p.ex_off[r + 1] - p.ex_off[r]);
    const uint32_t t = cols[q];
    const uint64_t b = p.sc_off[r] + rank_in<true>(tgt + p.rstart[r], L, t) + (q - p.run_off[r]);
    st[b] = t;
    if (vals) sw[b] = vals[q];
  }
}

__global__ void k_al_commit(const uint32_t* __restrict__ U, uint32_t R, AlPlan p, uint64_t* __restrict__ start,
                            uint32_t* __restrict__ len, uint32_t* __restrict__ cap) {
  GB_GRID_LOOP(r, R) {
    const uint32_t v = U[r];
    start[v] = p.dst[r];
    len[v] = (uint32_t)(p.sc_off[r + 1] - p.sc_off[r]);
    cap[v] = p.rcap[r];
  }
}

__global__ void k_al_narrow(const uint64_t* __restrict__ a, uint64_t count, uint32_t* __restrict__ out) {
  GB_GRID_LOOP(i, count) out[i] = (uint32_t)a[i];
}

// ---- host side ------------------------------------------------------------------------------------------------
static gb_status d2h(cudaStream_t s, void* host, const void* dev, size_t bytes) {
  GB_CUDA(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

// offsets[v] = sum of len[u < v] as u64 (n + 1 entries); returns the total
static gb_status len_prefix(cudaStream_t s, const AlList& L, uint32_t n, DevBuf<uint64_t>* prefix, uint64_t* total) {
  DevBuf<uint8_t> tmp;
  GB_TRY(prefix->alloc((size_t)n + 1));
  k_al_widen<<<grid_for((uint64_t)n + 1, 256), 256, 0, s>>>(L.len.p, n, prefix->p);
  GB_TRY(exclusive_sum(s, tmp, prefix->p, (int64_t)n + 1));
  GB_TRY(d2h(s, total, prefix->p + n, 8));
  return GB_OK;
}

// the list as a compacted CSR: offsets, targets (+8 zeroed) and, with_values, the values
static gb_status compact_list(cudaStream_t s, const AlList& L, uint32_t n, bool with_values, DevCsr* csr) {
  DevBuf<uint64_t> prefix;
  uint64_t total = 0;
  GB_TRY(len_prefix(s, L, n, &prefix, &total));
  GB_TRY(csr->off.alloc((size_t)n + 1));
  GB_TRY(csr->tgt.alloc(total, 8));
  GB_CUDA(cudaMemsetAsync(csr->tgt.p + total, 0, 8 * 4, s));
  if (with_values) GB_TRY(csr->w.alloc(total, 8));
  csr->len = total;
  k_al_narrow<<<grid_for((uint64_t)n + 1, 256), 256, 0, s>>>(prefix.p, (uint64_t)n + 1, csr->off.p);
  if (total)
    k_al_copy_runs<<<grid_for(total, 256), 256, 0, s>>>(prefix.p, n, L.start.p, prefix.p, total, L.tgt.p,
                                                        with_values ? L.w.p : nullptr, csr->tgt.p, csr->w.p);
  GB_CUDA(cudaGetLastError());
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

// A fresh list from the CSR build: start = offset, cap = len, and a free tail of count / 4 + AL_MIN_TAIL entries
static gb_status list_from_csr(cudaStream_t s, uint32_t n, DevCsr& csr, bool values, AlList* L) {
  const uint64_t count = csr.len;
  L->pool = count + count / 4 + AL_MIN_TAIL;
  L->bump = L->entries = count;
  GB_TRY(L->start.alloc(n));
  GB_TRY(L->len.alloc(n));
  GB_TRY(L->cap.alloc(n));
  GB_TRY(L->tgt.alloc(L->pool, 8));
  GB_CUDA(cudaMemsetAsync(L->tgt.p + L->pool, 0, 8 * 4, s));
  if (count) GB_CUDA(cudaMemcpyAsync(L->tgt.p, csr.tgt.p, count * 4, cudaMemcpyDeviceToDevice, s));
  if (values) {
    GB_TRY(L->w.alloc(L->pool));
    if (count) GB_CUDA(cudaMemcpyAsync(L->w.p, csr.w.p, count * 4, cudaMemcpyDeviceToDevice, s));
  }
  if (n) k_al_rows_from_offsets<<<grid_for(n, 256), 256, 0, s>>>(csr.off.p, n, L->start.p, L->len.p, L->cap.p);
  GB_CUDA(cudaGetLastError());
  GB_CUDA(cudaStreamSynchronize(s));
  csr = DevCsr();  // the CSR's arrays go now: the peak is the build's, not the build's plus the pool's
  return GB_OK;
}

// Checks device edge arrays on g's stream (check_edge_ids, with g->n), then AdjacencyList::from for every list of g
// (adj_list.rs:216-277); d_w is read only when g carries values
static gb_status build_lists(gb_algraph* g, const uint32_t* d_src, const uint32_t* d_dst, const float* d_w,
                             uint64_t m) {
  cudaStream_t s = g->stream;
  const gb_layout lay = g->layout;
  GB_TRY(check_edge_ids(s, d_src, d_dst, m, &g->n));
  if (!g->values) d_w = nullptr;
  if (g->kind == GB_KIND_DIRECTED) {
    DevCsr out, in;
    GB_TRY(build_csr_device(s, g->n, d_src, d_dst, d_w, m, lay, &out, 0, true));
    GB_TRY(list_from_csr(s, g->n, out, g->values, &g->list[0]));
    GB_TRY(build_csr_device(s, g->n, d_dst, d_src, d_w, m, lay, &in, 0, true));
    return list_from_csr(s, g->n, in, g->values, &g->list[1]);
  }
  // the interleaved stream: its stable row sort gives add_edge's order, and equal targets keep it
  DevBuf<uint32_t> rows, cols;
  GB_TRY(rows.alloc(2 * m));
  GB_TRY(cols.alloc(2 * m));
  if (m) k_al_interleave<<<grid_for(m, 256), 256, 0, s>>>(d_src, d_dst, m, rows.p, cols.p);
  GB_CUDA(cudaGetLastError());
  DevCsr csr;
  GB_TRY(build_csr_device(s, g->n, rows.p, cols.p, d_w, 2 * m, lay, &csr, 0, true, true));
  return list_from_csr(s, g->n, csr, g->values, &g->list[0]);
}

using AlPtr = std::unique_ptr<gb_algraph, void (*)(gb_algraph*)>;
static void al_free(gb_algraph* g) { gb_algraph_free(g); }

static gb_status new_algraph(int device, gb_graph_kind kind, gb_layout layout, bool values, uint32_t n, AlPtr* out) {
  GB_TRY(require_device(device));
  GB_CUDA(cudaSetDevice(device));
  AlPtr g(new (std::nothrow) gb_algraph(), al_free);
  if (!g) return fail(GB_ERR_OOM, "host allocation failed");
  g->device = device;
  g->kind = kind;
  g->layout = layout;
  g->values = values;
  g->n = n;
  cudaError_t e = cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking);
  for (cudaEvent_t* ev : {&g->ev_begin, &g->ev_end, &g->ev_cbegin, &g->ev_cend})
    if (e == cudaSuccess) e = cudaEventCreate(ev);
  if (e != cudaSuccess) return fail(GB_ERR_CUDA, "stream/event creation failed: %s", cudaGetErrorString(e));
  *out = std::move(g);
  return GB_OK;
}

// builds an adjacency-list graph from device edge arrays, after work enqueued on `caller`
static gb_status algraph_from_device(int device, gb_graph_kind kind, const uint32_t* d_src, const uint32_t* d_dst,
                                     const float* d_w, uint64_t m, uint32_t n, gb_layout layout, bool values,
                                     cudaStream_t caller, gb_algraph** out) {
  AlPtr g(nullptr, al_free);
  GB_TRY(new_algraph(device, kind, layout, values, n, &g));
  DevBufStreamScope scope(g->stream);
  GB_TRY(wait_on_stream(g->stream, caller));
  GB_TRY(build_lists(g.get(), d_src, d_dst, d_w, m));
  *out = g.release();
  return GB_OK;
}

// One list's share of a batch, in two steps so that a batch is all or nothing across a digraph's two lists:
// prepare_list reads the list and allocates everything the batch needs (sorted entries, runs, plan, merge scratch,
// a compacted pool), apply_list then changes the list and allocates nothing.  Every list is prepared before any is
// applied, so a failed allocation leaves the graph as it was.
struct AlStep {
  DevBuf<uint64_t> keys, keys_alt, arr, caps, live;
  DevBuf<uint32_t> pos, pos_alt, rows, cols, U, C, rcap, sc_t, nt;
  DevBuf<float> vals, sc_w, nw;
  AlPlan p{};
  uint64_t Bk = 0, ex_total = 0, sc_total = 0, tail_total = 0, cp_total = 0, cap_total = 0, live_total = 0, pool = 0;
  uint32_t R = 0;
  bool compact = false;
};

static gb_status prepare_list(gb_algraph* g, const AlList& L, const uint32_t* d_src, const uint32_t* d_dst,
                              const float* d_w, uint64_t b, bool reversed, AlStep& st, gb_algraph_batch_info* info) {
  cudaStream_t s = g->stream;
  const uint32_t n = g->n, bits = bits_for(n);
  const bool pairs = g->kind == GB_KIND_UNDIRECTED;
  const bool sorted = g->layout != GB_LAYOUT_UNSORTED;
  const uint64_t B = pairs ? 2 * b : b;
  const unsigned blk = 256;
  DevBuf<uint64_t>& keys = st.keys;
  DevBuf<uint64_t>& keys_alt = st.keys_alt;
  DevBuf<uint32_t>& pos = st.pos;
  DevBuf<uint32_t>& pos_alt = st.pos_alt;

  // 1. the batch's entries, stable-sorted by row (Unsorted) or by (row, target), with their stream positions
  GB_TRY(keys.alloc(B));
  GB_TRY(keys_alt.alloc(B));
  GB_TRY(pos.alloc(B));
  GB_TRY(pos_alt.alloc(B));
  k_al_batch_keys<<<grid_for(B, blk), blk, 0, s>>>(d_src, d_dst, B, bits, reversed, pairs, keys.p, pos.p);
  cub::DoubleBuffer<uint64_t> kb(keys.p, keys_alt.p);
  cub::DoubleBuffer<uint32_t> pb(pos.p, pos_alt.p);
  DevBuf<uint8_t> tmp;
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceRadixSort::SortPairs(t, tb, kb, pb, (int64_t)B, sorted ? 0 : (int)bits, (int)(2 * bits), s);
  }));
  uint64_t* skeys = kb.Current();
  uint32_t* spos = pb.Current();
  uint64_t& Bk = st.Bk;  // entries kept
  Bk = B;

  // 2. Deduplicated: drop targets the row holds or an earlier entry of the batch brings (the first value wins)
  DevBuf<uint64_t> d_num;
  GB_TRY(d_num.alloc(1));
  if (g->layout == GB_LAYOUT_DEDUPLICATED) {
    DevBuf<uint8_t> flags;
    GB_TRY(flags.alloc(B));
    k_al_dedup_flags<<<grid_for(B, blk), blk, 0, s>>>(skeys, B, bits, L.start.p, L.len.p, L.tgt.p, flags.p);
    DevBuf<uint8_t> t64, t32;
    GB_TRY(cub_call(t64, [&](void* t, size_t& tb) {
      return cub::DeviceSelect::Flagged(t, tb, skeys, flags.p, kb.Alternate(), d_num.p, (int64_t)B, s);
    }));
    GB_TRY(cub_call(t32, [&](void* t, size_t& tb) {
      return cub::DeviceSelect::Flagged(t, tb, spos, flags.p, pb.Alternate(), d_num.p, (int64_t)B, s);
    }));
    GB_TRY(d2h(s, &Bk, d_num.p, 8));
    skeys = kb.Alternate();
    spos = pb.Alternate();
  }
  info->inserted += Bk;
  if (Bk == 0) return GB_OK;

  DevBuf<uint32_t>& rows = st.rows;
  DevBuf<uint32_t>& cols = st.cols;
  DevBuf<float>& vals = st.vals;
  GB_TRY(rows.alloc(Bk));
  GB_TRY(cols.alloc(Bk));
  if (d_w) GB_TRY(vals.alloc(Bk));
  k_al_unpack<<<grid_for(Bk, blk), blk, 0, s>>>(skeys, spos, Bk, bits, d_w, pairs ? 1 : 0, rows.p, cols.p, vals.p);

  // 3. runs: the touched rows and how many entries each gets
  DevBuf<uint32_t>& U = st.U;
  DevBuf<uint32_t>& C = st.C;
  GB_TRY(U.alloc(Bk));
  GB_TRY(C.alloc(Bk));
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceRunLengthEncode::Encode(t, tb, rows.p, U.p, C.p, d_num.p, (int)Bk, s);
  }));
  uint64_t R64 = 0;
  GB_TRY(d2h(s, &R64, d_num.p, 8));
  const uint32_t R = st.R = (uint32_t)R64;

  // 4. plan: new lengths and capacities, the scans, and the totals
  DevBuf<uint64_t>& arr = st.arr;  // run_off, ex_off, sc_off, tail_off, cp_off (R + 1 each), rstart, dst (R each)
  DevBuf<uint32_t>& rcap = st.rcap;
  DevBuf<unsigned long long> moved;
  GB_TRY(arr.alloc(7 * ((size_t)R + 1)));
  GB_TRY(rcap.alloc(R));
  GB_TRY(moved.alloc(1));
  GB_CUDA(cudaMemsetAsync(moved.p, 0, 8, s));
  AlPlan& p = st.p;
  uint64_t* a = arr.p;
  const size_t R1 = (size_t)R + 1;
  p.run_off = a;
  p.ex_off = a + R1;
  p.sc_off = a + 2 * R1;
  p.tail_off = a + 3 * R1;
  p.cp_off = a + 4 * R1;
  p.rstart = a + 5 * R1;
  p.dst = a + 6 * R1;
  p.rcap = rcap.p;
  k_al_plan<<<grid_for(R1, blk), blk, 0, s>>>(U.p, C.p, R, L.start.p, L.len.p, L.cap.p, p, moved.p);
  for (uint64_t* x : {p.run_off, p.ex_off, p.sc_off, p.tail_off, p.cp_off})
    GB_TRY(exclusive_sum(s, tmp, x, (int64_t)R1));
  uint64_t &ex_total = st.ex_total, &sc_total = st.sc_total, &tail_total = st.tail_total, &cp_total = st.cp_total;
  unsigned long long nmoved = 0;
  GB_CUDA(cudaMemcpyAsync(&ex_total, p.ex_off + R, 8, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaMemcpyAsync(&sc_total, p.sc_off + R, 8, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaMemcpyAsync(&tail_total, p.tail_off + R, 8, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaMemcpyAsync(&cp_total, p.cp_off + R, 8, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaMemcpyAsync(&nmoved, moved.p, 8, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  info->touched_rows += R;
  info->relocated_rows += nmoved;

  // scratch of the merge
  if (sorted) {
    GB_TRY(st.sc_t.alloc(sc_total));
    if (d_w) GB_TRY(st.sc_w.alloc(sc_total));
  }

  // a compacted pool when the tail cannot take the rows that move: every row keeps its (new) capacity
  st.compact = L.bump + tail_total > L.pool;
  if (st.compact) {
    GB_TRY(st.caps.alloc((size_t)n + 1));
    k_al_widen<<<grid_for((uint64_t)n + 1, blk), blk, 0, s>>>(L.cap.p, n, st.caps.p);
    k_al_set_caps<<<grid_for(R, blk), blk, 0, s>>>(U.p, R, p.rcap, st.caps.p);
    GB_TRY(exclusive_sum(s, tmp, st.caps.p, (int64_t)n + 1));
    GB_TRY(d2h(s, &st.cap_total, st.caps.p + n, 8));
    GB_TRY(len_prefix(s, L, n, &st.live, &st.live_total));
    st.pool = 2 * st.cap_total + AL_MIN_TAIL;
    GB_TRY(st.nt.alloc(st.pool, 8));
    if (L.w.p) GB_TRY(st.nw.alloc(st.pool));
  }
  GB_CUDA(cudaGetLastError());
  return GB_OK;
}

static gb_status apply_list(gb_algraph* g, AlList& L, AlStep& st, gb_algraph_batch_info* info) {
  if (st.Bk == 0) return GB_OK;
  cudaStream_t s = g->stream;
  const uint32_t n = g->n;
  const bool sorted = g->layout != GB_LAYOUT_UNSORTED;
  const bool with_w = L.w.p != nullptr;
  const unsigned blk = 256;
  const uint32_t R = st.R;
  const uint64_t Bk = st.Bk, ex_total = st.ex_total, sc_total = st.sc_total, cp_total = st.cp_total;
  AlPlan& p = st.p;
  uint32_t* U = st.U.p;

  // 5. place the rows: moved rows at the tail, or every row in the compacted pool
  if (!st.compact) {
    k_al_dst_tail<<<grid_for(R, blk), blk, 0, s>>>(p, R, L.bump);
    if (!sorted && cp_total)  // an Unsorted row that moves takes its entries along; a Sorted one is merged below
      k_al_copy_runs<<<grid_for(cp_total, blk), blk, 0, s>>>(p.cp_off, R, p.rstart, p.dst, cp_total, L.tgt.p,
                                                              L.w.p, L.tgt.p, L.w.p);
    L.bump += st.tail_total;
  } else {
    GB_CUDA(cudaEventRecord(g->ev_cbegin, s));
    GB_CUDA(cudaMemsetAsync(st.nt.p + st.pool, 0, 8 * 4, s));
    if (st.live_total)
      k_al_copy_runs<<<grid_for(st.live_total, blk), blk, 0, s>>>(st.live.p, n, L.start.p, st.caps.p, st.live_total,
                                                                   L.tgt.p, L.w.p, st.nt.p, st.nw.p);
    GB_CUDA(cudaMemcpyAsync(L.start.p, st.caps.p, (size_t)n * 8, cudaMemcpyDeviceToDevice, s));
    k_al_dst_start<<<grid_for(R, blk), blk, 0, s>>>(U, R, L.start.p, p);
    GB_CUDA(cudaEventRecord(g->ev_cend, s));
    L.tgt = std::move(st.nt);  // the old pools are released once the stream is done with them
    L.w = std::move(st.nw);
    L.pool = st.pool;
    L.bump = st.cap_total;
    GB_CUDA(cudaEventSynchronize(g->ev_cend));
    float ms = 0.0f;
    GB_CUDA(cudaEventElapsedTime(&ms, g->ev_cbegin, g->ev_cend));
    info->compactions += 1;
    info->compaction_ms += ms;
  }
  uint32_t* cols = st.cols.p;
  float* vals = with_w ? st.vals.p : nullptr;
  uint32_t* sc_t = st.sc_t.p;
  float* sc_w = st.sc_w.p;

  // 6. write the entries
  if (!sorted) {
    k_al_append<<<grid_for(Bk, blk), blk, 0, s>>>(p, R, cols, vals, Bk, L.tgt.p, L.w.p);
  } else {
    if (ex_total)
      k_al_merge_old<<<grid_for(ex_total, blk), blk, 0, s>>>(p, R, ex_total, cols, L.tgt.p, L.w.p, sc_t, sc_w);
    k_al_merge_new<<<grid_for(Bk, blk), blk, 0, s>>>(p, R, Bk, cols, vals, L.tgt.p, sc_t, sc_w);
    k_al_copy_runs<<<grid_for(sc_total, blk), blk, 0, s>>>(p.sc_off, R, p.sc_off, p.dst, sc_total, sc_t, sc_w,
                                                            L.tgt.p, L.w.p);
  }
  k_al_commit<<<grid_for(R, blk), blk, 0, s>>>(U, R, p, L.start.p, L.len.p, L.cap.p);
  GB_CUDA(cudaGetLastError());
  GB_CUDA(cudaStreamSynchronize(s));
  L.entries += Bk;
  return GB_OK;
}

// add_edges on device arrays: the checks, then every list; g->mu is held
static gb_status add_edges_locked(gb_algraph* g, const uint32_t* d_src, const uint32_t* d_dst, const float* d_w,
                                  uint64_t b) {
  cudaStream_t s = g->stream;
  gb_algraph_batch_info info{};
  info.edges = b;
  GB_CUDA(cudaEventRecord(g->ev_begin, s));
  if (b) {
    DevBuf<unsigned long long> first;
    GB_TRY(first.alloc(1));
    GB_CUDA(cudaMemsetAsync(first.p, 0xFF, 8, s));
    k_al_first_bad<<<grid_for(b, 256), 256, 0, s>>>(d_src, d_dst, b, g->n, first.p);
    GB_CUDA(cudaGetLastError());
    unsigned long long k = 0;
    GB_TRY(d2h(s, &k, first.p, 8));
    if (k != ~0ull) {
      uint32_t e[2] = {0, 0};
      GB_CUDA(cudaMemcpyAsync(&e[0], d_src + k, 4, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaMemcpyAsync(&e[1], d_dst + k, 4, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
      const uint32_t missing = e[0] >= g->n ? e[0] : e[1];  // check_bounds(source) first (adj_list.rs:383-384)
      return fail(GB_ERR_INVALID, "node \"%u\" does not exist in the graph (edge %llu of the batch, %u -> %u; "
                  "node_count %u): no edge of the batch was added", missing, k, e[0], e[1], g->n);
    }
    AlStep step[2];
    for (int i = 0; i < g->lists(); ++i)
      GB_TRY(prepare_list(g, g->list[i], d_src, d_dst, g->values ? d_w : nullptr, b, i == 1, step[i], &info));
    for (int i = 0; i < g->lists(); ++i) GB_TRY(apply_list(g, g->list[i], step[i], &info));
  }
  GB_CUDA(cudaEventRecord(g->ev_end, s));
  GB_CUDA(cudaEventSynchronize(g->ev_end));
  float ms = 0.0f;
  GB_CUDA(cudaEventElapsedTime(&ms, g->ev_begin, g->ev_end));
  info.total_ms = ms;
  g->compactions += info.compactions;
  info.total_compactions = g->compactions;
  for (int i = 0; i < g->lists(); ++i) {
    info.pool_entries += g->list[i].pool;
    info.pool_used += g->list[i].bump;
  }
  g->last = info;
  return GB_OK;
}

// the arithmetic checks of a batch, before anything is read or allocated
static gb_status check_batch(const gb_algraph* g, const void* src, const void* dst, const void* w, uint64_t b) {
  GB_REQUIRE(b == 0 || (src && dst), "edge arrays are NULL");
  GB_REQUIRE(b == 0 || !g->values || w, "the graph carries edge values: weights is NULL");
  const uint64_t have = g->list[0].entries;
  const uint64_t add = g->kind == GB_KIND_UNDIRECTED ? 2 * b : b;
  GB_REQUIRE(b < AL_MAX_ENTRIES && add < AL_MAX_ENTRIES - have,
             "a batch of %llu edges would bring the list to %llu entries: a list holds fewer than 2^32 - 1; no edge "
             "of the batch was added", (unsigned long long)b, (unsigned long long)(have + add));
  GB_REQUIRE(add <= AL_MAX_BATCH, "a batch of %llu edges holds more than 2^31 - 1 list entries: split it; no edge of "
             "the batch was added", (unsigned long long)b);
  return GB_OK;
}

static gb_status pick_list(const gb_algraph* g, gb_csr_which which, const AlList** L) {
  if (g->kind == GB_KIND_DIRECTED && (which == GB_CSR_OUT || which == GB_CSR_IN)) {
    *L = &g->list[which == GB_CSR_OUT ? 0 : 1];
    return GB_OK;
  }
  if (g->kind == GB_KIND_UNDIRECTED && which == GB_CSR_UNDIRECTED) {
    *L = &g->list[0];
    return GB_OK;
  }
  return fail(GB_ERR_UNSUPPORTED, "graph kind %d has no list %d", (int)g->kind, (int)which);
}

}  // namespace gb

using namespace gb;

extern "C" {

gb_status gb_algraph_from_edges_u32(int device, gb_graph_kind kind, const uint32_t* src, const uint32_t* dst,
                                    const float* weights, uint64_t edge_count, uint32_t node_count, gb_layout layout,
                                    int with_values, gb_algraph** graph) {
  GB_TRY(check_edge_args(kind, src, dst, weights, edge_count, node_count, layout, with_values != 0, graph));
  GB_TRY(require_device(device));
  DeviceGuard guard(device);
  AlPtr g(nullptr, al_free);
  GB_TRY(new_algraph(device, kind, layout, with_values != 0, node_count, &g));
  DevBufStreamScope scope(g->stream);
  EdgeArrays e;
  GB_TRY(upload_edges(g->stream, src, dst, with_values ? weights : nullptr, edge_count, &e));
  GB_TRY(build_lists(g.get(), e.src.p, e.dst.p, e.w.p, edge_count));
  *graph = g.release();
  return GB_OK;
}

gb_status gb_algraph_from_device_edges_u32(int device, gb_graph_kind kind, const uint32_t* d_src,
                                           const uint32_t* d_dst, const float* d_weights, uint64_t edge_count,
                                           uint32_t node_count, gb_layout layout, int with_values, void* stream,
                                           gb_algraph** graph) {
  GB_TRY(check_edge_args(kind, d_src, d_dst, d_weights, edge_count, node_count, layout, with_values != 0, graph));
  GB_TRY(require_device(device));
  DeviceGuard guard(device);
  if (edge_count) {
    GB_TRY(require_device_array(d_src, device, "d_src"));
    GB_TRY(require_device_array(d_dst, device, "d_dst"));
    if (with_values) GB_TRY(require_device_array(d_weights, device, "d_weights"));
  }
  return algraph_from_device(device, kind, d_src, d_dst, d_weights, edge_count, node_count, layout, with_values != 0,
                             static_cast<cudaStream_t>(stream), graph);
}

gb_status gb_algraph_load_u32(int device, gb_graph_kind kind, const char* path, gb_file_format format,
                              gb_layout layout, int with_values, gb_algraph** graph) {
  GB_REQUIRE(graph != nullptr, "graph out-pointer is NULL");
  GB_REQUIRE(kind == GB_KIND_DIRECTED || kind == GB_KIND_UNDIRECTED, "bad graph kind %d", (int)kind);
  GB_TRY(check_layout(layout));
  EdgeArrays e;
  GB_TRY(load_edge_arrays(device, path, format, with_values != 0, &e));
  DeviceGuard guard(device);
  GB_TRY(check_edge_args(kind, e.src.p, e.dst.p, e.w.p, e.m, e.n, layout, with_values != 0, graph));
  GB_TRY(algraph_from_device(device, kind, e.src.p, e.dst.p, e.w.p, e.m, e.n, layout, with_values != 0, nullptr,
                             graph));
  (*graph)->load = e.info;
  return GB_OK;
}

gb_status gb_algraph_add_edges_u32(gb_algraph* g, const uint32_t* src, const uint32_t* dst, const float* weights,
                                   uint64_t edge_count) {
  GB_REQUIRE(g != nullptr, "NULL graph");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  GB_TRY(check_batch(g, src, dst, weights, edge_count));
  DevBufStreamScope scope(g->stream);
  EdgeArrays e;
  if (edge_count) GB_TRY(upload_edges(g->stream, src, dst, g->values ? weights : nullptr, edge_count, &e));
  return add_edges_locked(g, e.src.p, e.dst.p, e.w.p, edge_count);
}

gb_status gb_algraph_add_device_edges_u32(gb_algraph* g, const uint32_t* d_src, const uint32_t* d_dst,
                                          const float* d_weights, uint64_t edge_count, void* stream) {
  GB_REQUIRE(g != nullptr, "NULL graph");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  GB_TRY(check_batch(g, d_src, d_dst, d_weights, edge_count));
  if (edge_count) {
    GB_TRY(require_device_array(d_src, g->device, "d_src"));
    GB_TRY(require_device_array(d_dst, g->device, "d_dst"));
    if (g->values) GB_TRY(require_device_array(d_weights, g->device, "d_weights"));
  }
  DevBufStreamScope scope(g->stream);
  GB_TRY(wait_on_stream(g->stream, static_cast<cudaStream_t>(stream)));
  return add_edges_locked(g, d_src, d_dst, d_weights, edge_count);
}

gb_status gb_algraph_get_info(const gb_algraph* g, gb_graph_info* info) {
  GB_REQUIRE(g && info, "NULL argument");
  std::lock_guard<std::mutex> lock(g->mu);
  info->kind = (uint32_t)g->kind;
  info->node_count = g->n;
  info->target_count = g->list[0].entries;
  info->edge_count = g->kind == GB_KIND_UNDIRECTED ? g->list[0].entries / 2 : g->list[0].entries;
  info->has_weights = g->values ? 1 : 0;
  info->device = g->device;
  info->device_bytes = g->list[0].bytes() + g->list[1].bytes();
  return GB_OK;
}

gb_status gb_algraph_last_batch(const gb_algraph* g, gb_algraph_batch_info* info) {
  GB_REQUIRE(g && info, "NULL argument");
  std::lock_guard<std::mutex> lock(g->mu);
  *info = g->last;
  return GB_OK;
}

gb_status gb_algraph_copy_row(const gb_algraph* g, gb_csr_which which, uint32_t node, uint32_t capacity,
                              uint32_t* targets, float* values, uint32_t* len) {
  GB_REQUIRE(g && len, "NULL argument");
  const AlList* L = nullptr;
  GB_TRY(pick_list(g, which, &L));
  GB_REQUIRE(node < g->n, "node %u out of range for a graph with %u nodes", node, g->n);
  GB_REQUIRE(!values || g->values, "the graph carries no edge values");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  uint64_t start = 0;
  GB_CUDA(cudaMemcpyAsync(len, L->len.p + node, 4, cudaMemcpyDeviceToHost, g->stream));
  GB_CUDA(cudaMemcpyAsync(&start, L->start.p + node, 8, cudaMemcpyDeviceToHost, g->stream));
  GB_CUDA(cudaStreamSynchronize(g->stream));
  const uint32_t k = *len < capacity ? *len : capacity;
  if (k && targets) GB_CUDA(cudaMemcpyAsync(targets, L->tgt.p + start, (size_t)k * 4, cudaMemcpyDeviceToHost, g->stream));
  if (k && values) GB_CUDA(cudaMemcpyAsync(values, L->w.p + start, (size_t)k * 4, cudaMemcpyDeviceToHost, g->stream));
  GB_CUDA(cudaStreamSynchronize(g->stream));
  return GB_OK;
}

gb_status gb_algraph_copy_csr(const gb_algraph* g, gb_csr_which which, uint64_t capacity, uint32_t* offsets,
                              uint32_t* targets, float* values, uint64_t* count) {
  GB_REQUIRE(g && offsets && count, "NULL argument");
  const AlList* L = nullptr;
  GB_TRY(pick_list(g, which, &L));
  GB_REQUIRE(!values || g->values, "the graph carries no edge values");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  DevBufStreamScope scope(g->stream);
  DevCsr csr;
  GB_TRY(compact_list(g->stream, *L, g->n, values != nullptr, &csr));
  *count = csr.len;
  GB_CUDA(cudaMemcpyAsync(offsets, csr.off.p, ((size_t)g->n + 1) * 4, cudaMemcpyDeviceToHost, g->stream));
  const bool fits = csr.len <= capacity;  // a batch may have landed since the caller sized its arrays
  if (fits && targets && csr.len)
    GB_CUDA(cudaMemcpyAsync(targets, csr.tgt.p, csr.len * 4, cudaMemcpyDeviceToHost, g->stream));
  if (fits && values && csr.len)
    GB_CUDA(cudaMemcpyAsync(values, csr.w.p, csr.len * 4, cudaMemcpyDeviceToHost, g->stream));
  GB_CUDA(cudaStreamSynchronize(g->stream));
  return GB_OK;
}

gb_status gb_algraph_to_graph(const gb_algraph* al, gb_graph** graph) {
  GB_REQUIRE(al && graph, "NULL argument");
  DeviceGuard guard(al->device);
  GraphPtr g;
  GB_TRY(new_graph(al->device, al->kind, al->n, &g));
  std::lock_guard<std::mutex> lock(al->mu);
  DevBufStreamScope scope(g->stream);
  GB_CUDA(cudaEventRecord(g->ev_begin, g->stream));
  GB_TRY(compact_list(g->stream, al->list[0], al->n, al->values, &g->out));
  if (al->kind == GB_KIND_DIRECTED) GB_TRY(compact_list(g->stream, al->list[1], al->n, false, &g->in));
  GB_CUDA(cudaEventRecord(g->ev_end, g->stream));
  GB_CUDA(cudaEventSynchronize(g->ev_end));
  float ms = 0.0f;
  GB_CUDA(cudaEventElapsedTime(&ms, g->ev_begin, g->ev_end));
  g->timing = gb_timing{};
  g->timing.total_ms = ms;
  g->row_order = al->layout == GB_LAYOUT_UNSORTED ? RowOrder::Unknown : RowOrder::Sorted;
  *graph = g.release();
  return GB_OK;
}

gb_status gb_algraph_load_info(const gb_algraph* g, gb_load_info* info) {
  GB_REQUIRE(g && info, "NULL argument");
  *info = g->load;
  return GB_OK;
}

gb_status gb_algraph_free(gb_algraph* g) {
  if (!g) return GB_OK;
  DeviceGuard guard(g->device);
  if (g->stream) cudaStreamSynchronize(g->stream);
  for (AlList& L : g->list) L = AlList();
  for (cudaEvent_t e : {g->ev_begin, g->ev_end, g->ev_cbegin, g->ev_cend})
    if (e) cudaEventDestroy(e);
  if (g->stream) cudaStreamDestroy(g->stream);
  delete g;
  return GB_OK;
}

}  // extern "C"
