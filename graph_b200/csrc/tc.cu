// tc.cu — global triangle count on the undirected device CSR.
//
// Replaces crates/algos/src/triangle_count.rs:22-86 (`global_triangle_count`).  The reference walks
//   for u: for v in N(u), stop at v > u: for w in N(v), stop at w > v: advance a put-back cursor over
//   N(u) while *cursor < w; count if *cursor == w
// in list order, whatever the order of the rows.  On sorted rows that evaluates
//   T = sum_u sum_{v-occurrence in N(u), v<=u} sum_{w-occurrence in N(v), w<=v} [w in set(N(u))]
// (duplicate v and w occurrences multiply, duplicate x in N(u) do not; self loops take part) —
// SURVEY.md A.5.  On unsorted rows the stops and the cursor give a different number, and the reference
// returns that number; Layout::Unsorted is the default layout, so it is the common case, not an error.
//
// The row order picks one of two paths.  Sorted and Deduplicated builds and make_degree_ordered write
// sorted rows (gb_graph::row_order); for any other CSR the first call runs k_tc_rows_unsorted once, which
// looks for a descent inside a row (one across a row boundary does not count), and caches the answer.
//   sorted rows   — k_tc, one launch: the sum above, edge-parallel.  One CSR entry (u, v) with v <= u per
//                   work item; both lists are cut to values <= v by binary search, and the cheaper one is
//                   walked while the other is searched.  Walks of at most TC_SHORT entries stay in one
//                   lane, longer ones go to the whole warp in steps of 32.
//   unsorted rows — k_tc_cut + k_tc_list, the reference loop restated: cut[u] is the first index of row
//                   u whose target is > u, and one thread per entry i < cut[u] walks N(v)[.. cut[v]) in
//                   list order with the put-back cursor over N(u).  A path for correctness: its work is
//                   O(deg u + deg v) per entry in one thread, and no benchmark runs it.
//
// Compulsory bytes per run: 8m + 4(n+1) (the undirected CSR once); the kernel is bound by the
// dependent lookups (latency / L2), not by HBM.
//
// One-shot count of a host CSR (gb_triangle_count_csr_u32).  Each term of the sum is one entry (u, v <= u)
// and reads N(u) and N(v) only, on both paths, so the entries of the rows [r0, r1) can be counted once the
// rows 0 .. r1 - 1 are on the device: the stream is causal in row order.  A CheckedFeed (common.cuh) sends the
// offsets first and the targets in row order after them, straight into their final place in one targets[m]
// array, because the terms read earlier rows at random: unlike the WCC ring, the whole CSR ends up resident.
// Once chunk k has landed, the feed's check stream runs the id check and k_tc_rows_unsorted over its rows only,
// and the host counts its entries with k_tc while every chunk so far had sorted rows, and with k_tc_cut +
// k_tc_list from the first unsorted chunk on, for the rest of the call (k_tc's searches in N(v) are wrong once
// an earlier row v is unsorted; on sorted rows u and v the two give the same term).  All chunks add into one
// device total, read back once.
#include "common.cuh"

namespace gb {

constexpr uint32_t TC_SHORT = 16;

__device__ __forceinline__ uint32_t tc_lower_bound(const uint32_t* __restrict__ a, uint32_t lo, uint32_t hi,
                                                   uint32_t x) {
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(a + mid) < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}
__device__ __forceinline__ uint32_t tc_upper_bound(const uint32_t* __restrict__ a, uint32_t lo, uint32_t hi,
                                                   uint32_t x) {
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(a + mid) <= x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// The entries [e_begin, e_end) of the rows [row_begin, row_end) (off[row_begin] == e_begin, off[row_end] ==
// e_end): the whole CSR is 0, n, 0, len.  Rows below row_begin are read as N(v) only.
__global__ void __launch_bounds__(256) k_tc(const uint32_t* __restrict__ off, const uint32_t* __restrict__ tgt,
                                            uint32_t row_begin, uint32_t row_end, uint64_t e_begin, uint64_t e_end,
                                            unsigned long long* total) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  unsigned long long count = 0;
  for (uint64_t base = e_begin + warp * 32; base < e_end; base += nwarps * 32) {
    const uint64_t i = base + lane;
    uint32_t u = 0, v = 0, ub = 0, ue = 0, vb = 0, ve = 0;
    bool live = false;
    if (i < e_end) {
      // row of entry i: last u with off[u] <= i
      uint32_t lo = row_begin, hi = row_end;
      while (hi - lo > 1) {
        const uint32_t mid = lo + ((hi - lo) >> 1);
        if (__ldg(off + mid) <= i) lo = mid; else hi = mid;
      }
      u = lo;
      v = __ldg(tgt + i);
      if (v <= u) {  // triangle_count.rs:49-51
        ub = __ldg(off + u);
        ue = __ldg(off + u + 1);
        vb = __ldg(off + v);
        ve = tc_upper_bound(tgt, vb, __ldg(off + v + 1), v);  // w <= v only, :56-58
        // matches can only be values <= v: restrict the search window in N(u) once
        ue = tc_upper_bound(tgt, ub, ue, v);
        live = ve > vb && ue > ub;
      }
    }
    // The sum over w-occurrences of N(v) found in set(N(u)) equals the sum over DISTINCT x of N(u) of
    // x's multiplicity in N(v); walk whichever list makes the lookups cheaper.
    bool by_u = false;
    if (live) {
      const uint32_t lv = ve - vb, lu = ue - ub;
      by_u = (uint64_t)lu * (32 - __clz(lv)) < (uint64_t)lv * (32 - __clz(lu));
    }
    const uint32_t walk_b = by_u ? ub : vb, walk_e = by_u ? ue : ve;
    const uint32_t find_b = by_u ? vb : ub, find_e = by_u ? ve : ue;
    const bool is_short = live && (walk_e - walk_b) <= TC_SHORT;
    if (is_short) {
      uint32_t prev = 0xFFFFFFFFu;
      for (uint32_t j = walk_b; j < walk_e; ++j) {
        const uint32_t w = __ldg(tgt + j);
        if (by_u) {
          if (w != prev) {
            const uint32_t lo = tc_lower_bound(tgt, find_b, find_e, w);
            count += tc_upper_bound(tgt, lo, find_e, w) - lo;
          }
          prev = w;
        } else {
          const uint32_t p = tc_lower_bound(tgt, find_b, find_e, w);
          count += (p < find_e && __ldg(tgt + p) == w) ? 1u : 0u;
        }
      }
    }
    unsigned long_mask = __ballot_sync(0xFFFFFFFFu, live && !is_short);
    while (long_mask) {
      const int owner = __ffs(long_mask) - 1;
      long_mask &= long_mask - 1;
      const uint32_t owb = __shfl_sync(0xFFFFFFFFu, walk_b, owner), owe = __shfl_sync(0xFFFFFFFFu, walk_e, owner);
      const uint32_t ofb = __shfl_sync(0xFFFFFFFFu, find_b, owner), ofe = __shfl_sync(0xFFFFFFFFu, find_e, owner);
      const bool oby_u = __shfl_sync(0xFFFFFFFFu, (int)by_u, owner) != 0;
      for (uint32_t j = owb + lane; j < owe; j += 32) {
        const uint32_t w = __ldg(tgt + j);
        if (oby_u) {
          if (j == owb || __ldg(tgt + j - 1) != w) {  // first occurrence of x in N(u)
            const uint32_t lo = tc_lower_bound(tgt, ofb, ofe, w);
            count += tc_upper_bound(tgt, lo, ofe, w) - lo;
          }
        } else {
          const uint32_t p = tc_lower_bound(tgt, ofb, ofe, w);
          count += (p < ofe && __ldg(tgt + p) == w) ? 1u : 0u;
        }
      }
    }
  }
  for (int o = 16; o > 0; o >>= 1) count += __shfl_xor_sync(0xFFFFFFFFu, count, o);
  if (lane == 0 && count) atomicAdd(total, count);
}

// *found = 1 when some row of [row_begin, row_end) (entries [e_begin, e_end), as for k_tc) holds
// tgt[i-1] > tgt[i]; a descent at an entry that begins a row does not count
__global__ void __launch_bounds__(256) k_tc_rows_unsorted(const uint32_t* __restrict__ off,
                                                          const uint32_t* __restrict__ tgt, uint32_t row_begin,
                                                          uint32_t row_end, uint64_t e_begin, uint64_t e_end,
                                                          unsigned long long* found) {
  for (uint64_t i = e_begin + 1 + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < e_end;
       i += (uint64_t)gridDim.x * blockDim.x) {
    if (__ldg(tgt + i - 1) <= __ldg(tgt + i)) continue;
    // a row begins at entry i iff some off[u] == i; p == row_end means i lies inside row row_end-1
    // (off[row_end] = e_end > i)
    const uint32_t p = tc_lower_bound(off, row_begin, row_end, (uint32_t)i);
    if (p == row_end || __ldg(off + p) != i) *found = 1ull;
  }
}

// cut[u] = the first index of row u whose target is > u, else off[u + 1]: where the reference stops its
// walk of N(u) (triangle_count.rs:49-51) and, for u in the role of v, its walk of N(v) (:56-58).
// One warp per row of [row_begin, row_end).
__global__ void __launch_bounds__(256) k_tc_cut(const uint32_t* __restrict__ off, const uint32_t* __restrict__ tgt,
                                                uint32_t row_begin, uint32_t row_end, uint32_t* __restrict__ cut) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warp = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint64_t nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t u = row_begin + warp; u < row_end; u += nwarps) {
    const uint64_t b = __ldg(off + u), e = __ldg(off + u + 1);
    uint64_t c = e;
    for (uint64_t j0 = b; j0 < e; j0 += 32) {
      const uint64_t j = j0 + lane;
      const unsigned hit = __ballot_sync(0xFFFFFFFFu, j < e && __ldg(tgt + j) > u);
      if (hit) {
        c = j0 + __ffs(hit) - 1;
        break;
      }
    }
    if (lane == 0) cut[u] = (uint32_t)c;
  }
}

// One thread per entry i of row u with i < cut[u] (so v = tgt[i] <= u): the reference's loop for that
// v-occurrence, in list order — a fresh cursor over all of N(u), advanced while *cursor < w, stops once
// it runs out (oracle.c tc_vertex).  Entries [e_begin, e_end) of the rows [row_begin, row_end), as for k_tc;
// cut[] must hold every row up to row_end - 1.
__global__ void __launch_bounds__(256) k_tc_list(const uint32_t* __restrict__ off, const uint32_t* __restrict__ tgt,
                                                 const uint32_t* __restrict__ cut, uint32_t row_begin,
                                                 uint32_t row_end, uint64_t e_begin, uint64_t e_end,
                                                 unsigned long long* total) {
  unsigned long long count = 0;
  for (uint64_t i = e_begin + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < e_end;
       i += (uint64_t)gridDim.x * blockDim.x) {
    // row of entry i: last u with off[u] <= i
    uint32_t lo = row_begin, hi = row_end;
    while (hi - lo > 1) {
      const uint32_t mid = lo + ((hi - lo) >> 1);
      if (__ldg(off + mid) <= i) lo = mid; else hi = mid;
    }
    const uint32_t u = lo;
    if (i >= __ldg(cut + u)) continue;
    const uint32_t v = __ldg(tgt + i);
    uint32_t it = __ldg(off + u);
    const uint32_t ue = __ldg(off + u + 1), ve = __ldg(cut + v);
    for (uint32_t j = __ldg(off + v); j < ve; ++j) {
      const uint32_t w = __ldg(tgt + j);
      while (it < ue && __ldg(tgt + it) < w) ++it;
      if (it == ue) break;  // later w find nothing either
      count += __ldg(tgt + it) == w ? 1u : 0u;
    }
  }
  for (int o = 16; o > 0; o >>= 1) count += __shfl_xor_sync(0xFFFFFFFFu, count, o);
  if ((threadIdx.x & 31) == 0 && count) atomicAdd(total, count);
}

// ---- one-shot count of a host CSR (gb_triangle_count_csr_u32) ----------------------------------------------
// k_tc launches of consecutive chunks go round-robin to this many streams: a chunk's count ends in a tail of
// a few heavy warps (hub rows), and the next chunks' blocks fill the SMs meanwhile
constexpr uint32_t TC_COUNT_LANES = 4;

thread_local gb_tc_csr_info tc_csr_last{};  // behind gb_triangle_count_csr_info

// Everything one call holds.  The destructor drains the consumer streams, and the check stream that writes
// h_found, before anything they use goes: the pinned flags, the events, the device buffers (members) and the
// feed (the first member).
struct TcCall {
  CheckedFeed feed;  // the offsets [0, n] and the resident targets, sent in row order
  DevBuf<uint32_t> cut;
  DevBuf<unsigned long long> found, total;  // found[k]: chunk k has a descent inside a row
  unsigned long long* h_found = nullptr;    // page-locked: found[K], then the total
  cudaStream_t count = nullptr;             // the list-order path, and the join
  cudaStream_t lanes[TC_COUNT_LANES] = {};  // the k_tc launches
  cudaEvent_t lane_done[TC_COUNT_LANES] = {};

  gb_status create(uint32_t K) {
    GB_CUDA(cudaStreamCreateWithFlags(&count, cudaStreamNonBlocking));
    for (uint32_t i = 0; i < TC_COUNT_LANES; ++i) {
      GB_CUDA(cudaStreamCreateWithFlags(&lanes[i], cudaStreamNonBlocking));
      GB_CUDA(cudaEventCreateWithFlags(&lane_done[i], cudaEventDisableTiming));
    }
    GB_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&h_found), ((size_t)K + 1) * 8, cudaHostAllocDefault));
    GB_TRY(found.alloc(K));
    return total.alloc(1);
  }
  ~TcCall() {
    for (cudaStream_t s : {feed.check, count})
      if (s) cudaStreamSynchronize(s);
    for (uint32_t i = 0; i < TC_COUNT_LANES; ++i) {
      if (lanes[i]) cudaStreamSynchronize(lanes[i]), cudaStreamDestroy(lanes[i]);
      if (lane_done[i]) cudaEventDestroy(lane_done[i]);
    }
    if (count) cudaStreamDestroy(count);
    if (h_found) cudaFreeHost(h_found);
  }
};

// The checks and messages are those of gb_graph_from_csr_u32 (upload_host_csr) for the same arrays.
static gb_status tc_csr(int device, uint32_t n, const uint32_t* off, const uint32_t* tgt, uint64_t* triangles) {
  tc_csr_last = gb_tc_csr_info{};
  GB_REQUIRE(triangles != nullptr, "triangles is NULL");
  GB_REQUIRE(n > 0, "node_count must be > 0");
  GB_TRY(require_device(device));
  GB_TRY(require_host_csr(n, off, tgt, "undirected"));
  DeviceGuard guard(device);
  GB_CUDA(cudaSetDevice(device));
  TcCall t;
  CheckedFeed& f = t.feed;
  GB_TRY(f.open(device, n, off, tgt, nullptr, env_u64("GB_TC_FEED_ENTRIES", 0), 0, "undirected"));
  const uint32_t K = f.K;
  GB_TRY(t.create(K));
  gb_tc_csr_info info{};
  info.first_list_chunk = K;
  GB_CUDA(cudaMemsetAsync(t.found.p, 0, (size_t)K * 8, f.check));
  // on the check stream: every count launch, on a lane or on t.count, waits for a checked[] event recorded there
  GB_CUDA(cudaMemsetAsync(t.total.p, 0, 8, f.check));
  const uint32_t *d_off = f.feed.off.p, *d_tgt = f.feed.tgt.p;
  // chunk k's row-order flag, checked with its ids
  f.per_chunk = [&](uint32_t k) -> gb_status {
    const uint64_t e0 = f.ch.edge[k], e1 = f.ch.edge[k + 1];
    if (e1 - e0 >= 2) {
      k_tc_rows_unsorted<<<grid_for(e1 - e0, 256, H100_SMS * 32u), 256, 0, f.check>>>(
          d_off, d_tgt, f.ch.row[k], f.ch.row[k + 1], e0, e1, t.found.p + k);
      info.kernel_launches += 1;
    }
    GB_CUDA(cudaMemcpyAsync(t.h_found + k, t.found.p + k, 8, cudaMemcpyDeviceToHost, f.check));
    return GB_OK;
  };
  // from pageable memory one chunk is kept on the bus ahead of the one being counted
  const uint32_t ahead = f.pinned ? K : 1;
  while (f.issued < ahead) GB_TRY(f.issue());
  // the offsets are monotone before anything indexes with them
  GB_TRY(f.require_offsets());
  bool list = false;  // from the first chunk with an unsorted row on, every chunk takes k_tc_cut + k_tc_list
  for (uint32_t k = 0; k < K; ++k) {
    if (f.issued < K) GB_TRY(f.issue());  // the next chunk is on the bus while this one is checked and counted
    GB_CUDA(cudaEventSynchronize(f.checked[k]));
    if (f.h_bad[1 + k]) return f.check_all();  // nothing of this chunk is counted
    const uint64_t e0 = f.ch.edge[k], e1 = f.ch.edge[k + 1];
    const uint32_t r0 = f.ch.row[k], r1 = f.ch.row[k + 1];
    if (e1 == e0) continue;
    const unsigned grid = grid_for(e1 - e0, 256, H100_SMS * 32u);
    list = list || t.h_found[k];
    if (!list) {  // k_tc reads only landed rows: the chunks count side by side
      cudaStream_t lane = t.lanes[info.sorted_chunks % TC_COUNT_LANES];
      GB_CUDA(cudaStreamWaitEvent(lane, f.checked[k], 0));
      k_tc<<<grid, 256, 0, lane>>>(d_off, d_tgt, r0, r1, e0, e1, t.total.p);
      info.sorted_chunks += 1;
      info.kernel_launches += 1;
    } else {  // k_tc_list reads cut[v] for every v <= u: the cuts and counts go in row order on one stream
      GB_CUDA(cudaStreamWaitEvent(t.count, f.checked[k], 0));
      const uint32_t c0 = info.list_chunks ? r0 : 0;  // the first list chunk cuts every row so far
      if (!info.list_chunks) {
        info.first_list_chunk = k;
        GB_TRY(t.cut.alloc(n));
      }
      k_tc_cut<<<grid_for((uint64_t)(r1 - c0) * 32, 256, H100_SMS * 32u), 256, 0, t.count>>>(d_off, d_tgt, c0, r1,
                                                                                             t.cut.p);
      k_tc_list<<<grid, 256, 0, t.count>>>(d_off, d_tgt, t.cut.p, r0, r1, e0, e1, t.total.p);
      info.list_chunks += 1;
      info.kernel_launches += 2;
    }
    GB_CUDA(cudaGetLastError());
  }
  for (uint32_t i = 0; i < TC_COUNT_LANES; ++i) {
    GB_CUDA(cudaEventRecord(t.lane_done[i], t.lanes[i]));
    GB_CUDA(cudaStreamWaitEvent(t.count, t.lane_done[i], 0));
  }
  GB_TRY(f.finish(t.count, t.h_found + K, t.total.p, 8));
  GB_TRY(f.report(&info));
  *triangles = t.h_found[K];
  tc_csr_last = info;
  return GB_OK;
}

}  // namespace gb

extern "C" gb_status gb_triangle_count(const gb_graph* g, uint64_t* triangles) {
  using namespace gb;
  GB_REQUIRE(g && triangles, "NULL argument");
  if (g->kind != GB_KIND_UNDIRECTED)
    return fail(GB_ERR_UNSUPPORTED, "global_triangle_count needs an undirected graph (triangle_count.rs:25)");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  cudaStream_t s = g->stream;
  const DevCsr& c = g->out;
  DevBuf<unsigned long long> total;  // [0] the count, [1] the row-order flag
  DevBuf<uint32_t> cut;
  GB_TRY(total.alloc(2));
  g->timing = gb_timing{};
  GB_CUDA(cudaEventRecord(g->ev_begin, s));
  GB_CUDA(cudaMemsetAsync(total.p, 0, 16, s));
  const unsigned grid = grid_for(c.len, 256, H100_SMS * 32u);
  if (c.len && g->row_order == RowOrder::Unknown) {  // once per CSR
    k_tc_rows_unsorted<<<grid, 256, 0, s>>>(c.off.p, c.tgt.p, 0, g->n, 0, c.len, total.p + 1);
    g->timing.kernel_launches += 1;
    GB_CUDA(cudaGetLastError());
    unsigned long long found = 0;
    GB_CUDA(cudaMemcpyAsync(&found, total.p + 1, 8, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    g->row_order = found ? RowOrder::Unsorted : RowOrder::Sorted;
  }
  if (c.len && g->row_order == RowOrder::Sorted) {
    k_tc<<<grid, 256, 0, s>>>(c.off.p, c.tgt.p, 0, g->n, 0, c.len, total.p);
    g->timing.kernel_launches += 1;
  } else if (c.len) {
    GB_TRY(cut.alloc(g->n));
    k_tc_cut<<<grid_for((uint64_t)g->n * 32, 256, H100_SMS * 32u), 256, 0, s>>>(c.off.p, c.tgt.p, 0, g->n,
                                                                             cut.p);
    k_tc_list<<<grid, 256, 0, s>>>(c.off.p, c.tgt.p, cut.p, 0, g->n, 0, c.len, total.p);
    g->timing.kernel_launches += 2;
  }
  GB_CUDA(cudaGetLastError());
  GB_CUDA(cudaEventRecord(g->ev_end, s));
  unsigned long long h = 0;
  GB_CUDA(cudaMemcpyAsync(&h, total.p, 8, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  float ms = 0.0f;
  GB_CUDA(cudaEventElapsedTime(&ms, g->ev_begin, g->ev_end));
  g->timing.total_ms = ms;
  *triangles = h;
  return GB_OK;
}

extern "C" gb_status gb_triangle_count_csr_u32(int device, uint32_t node_count, const uint32_t* offsets,
                                               const uint32_t* targets, uint64_t* triangles) {
  return gb::tc_csr(device, node_count, offsets, targets, triangles);
}

extern "C" gb_status gb_triangle_count_csr_info(gb_tc_csr_info* info) {
  GB_REQUIRE(info != nullptr, "info is NULL");
  *info = gb::tc_csr_last;
  return GB_OK;
}
