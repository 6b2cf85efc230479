// sssp.cu — single-source shortest paths (delta-stepping) on the weighted device out-CSR.
//
// Replaces crates/algos/src/sssp.rs:38-204 (`delta_stepping`, `relax_edges`, the bin loop).
// The reference relaxes with a CAS-min on AtomicF32 and files improved targets into bins of width
// delta.  Here distances are non-negative f32 bit patterns, which order like u32, so the CAS loop
// of sssp.rs:184-202 becomes one atomicMin; improved targets go to a NEAR queue (distance below the
// current bucket's upper bound) or a FAR pile, the device analogue of the thread-local bins.
// Because f32 `+` is monotone and weights are >= 0 the fixed point dist[t] = min fl(dist[u] + w) is
// unique, so results are bit-exact with the reference for every schedule and every delta.
//
// Algorithmic bytes per run: 8m + 4(n+1) + 8n (weighted out-CSR once, distances read + write).
//
// One-shot SSSP of a host out-CSR (gb_sssp_csr_u32).  A CheckedFeed (common.cuh) sends the offsets first and
// checks them; the targets and their f32 values follow in its chunks, sent from the chunk that holds the start on
// and wrapping round (sssp_send_order), into one resident CSR.  A chunk is available once its id check has
// passed, and the available rows are then one cyclic interval from the start's chunk (SsspRows).  The bucket
// loop is the twin's, with one change in k_sssp_relax<true>: a queue entry whose row is not available yet is
// not relaxed but PARKED, once per vertex, in a parked list; between passes the host raises the available bound
// and k_sssp_unpark moves the parked vertices whose rows are now present into the near queue.  When only parked
// vertices are left the host blocks on the next chunk.
// Parking breaks what the stale filter (`du < lower`) relies on: that a vertex below the current bucket was
// relaxed with its final distance while its bucket drained.  A parked vertex relaxed late can improve a vertex
// of a drained bucket to a distance below `lower`, and that vertex must be relaxed again.  So from the first park
// on the relax passes take lower = 0 and drop nothing: every strict improvement is then relaxed once its row is
// present, and the loop still ends at the unique fixed point above (SURVEY.md A.4), bit-equal to the twin.
#include <algorithm>
#include <cfloat>

#include "common.cuh"
#include "sssp_bucket.h"

namespace gb {

struct SsspQueues {
  uint32_t* near_in;
  uint32_t* near_out;
  uint32_t* far;
  uint32_t* far_out;
  uint32_t* counts;  // [0] near_out count, [1] far count, [2] far_out count, [3] near_in count
};

__global__ void k_sssp_init(uint32_t* __restrict__ dist, uint32_t n, uint32_t start) {
  for (uint64_t v = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; v < n; v += (uint64_t)gridDim.x * blockDim.x)
    dist[v] = (v == start) ? 0u : __float_as_uint(FLT_MAX);  // INF = f32::MAX, sssp.rs:12
}

// relax_edges, sssp.rs:170-204, for every vertex of the near queue.  One lane per queue entry; short
// adjacency lists are relaxed by their own lane, long ones by the whole warp.
// queue slot reservation, aggregated over the lanes that are appending right now: one atomicAdd per
// group of converged lanes instead of one per successful relaxation (a single hot counter otherwise
// serialises every append of the pass)
// Lanes are grouped BY COUNTER (match_any on the pointer): callers append to different queues from
// sibling branches, and nothing guarantees that the active mask holds lanes of one branch only.
__device__ __forceinline__ uint32_t sssp_reserve(uint32_t* counter) {
  const unsigned active = __activemask();
  const unsigned peers = __match_any_sync(active, (unsigned long long)counter);
  const int leader = __ffs(peers) - 1;
  const uint32_t lane = threadIdx.x & 31;
  uint32_t base = 0;
  if ((int)lane == leader) base = atomicAdd(counter, (uint32_t)__popc(peers));
  base = __shfl_sync(peers, base, leader);
  return base + __popc(peers & ((1u << lane) - 1u));
}

// A vertex whose distance improves several times in one pass (or several times while it waits in the far
// pile) is queued once: near_stamp[t] holds the last pass in which t was appended to the near queue, and
// in_pile[t] is 1 while t has an entry in the far pile (set by the append here, cleared by k_sssp_split_far
// when the entry leaves the pile).  The pile never holds a vertex twice, however many buckets pass while t
// waits in it, and every queue is bounded by n whatever delta is.
struct SsspStamps {
  uint32_t* near_stamp;
  uint32_t* in_pile;
  uint32_t pass;
};

// The rows a relax pass may read: `span` rows from row `first` on, modulo n (the chunks sent and checked so
// far, gb_sssp_csr_u32).  parked[u] is 1 while u has an entry in the parked list, so that the list holds a
// vertex once, as in_pile does for the far pile; counts[4] is the list's length.  The twin's instantiation
// of k_sssp_relax does not read it.
struct SsspRows {
  uint32_t first, span, n;
  uint32_t* parked;
  __device__ __forceinline__ bool present(uint32_t u) const {
    return (u >= first ? u - first : u + (n - first)) < span;
  }
};

__device__ __forceinline__ void sssp_relax_edge(const uint32_t* __restrict__ tgt, const float* __restrict__ w,
                                                uint32_t* dist, uint32_t i, float du, float upper,
                                                uint32_t* __restrict__ near_out, uint32_t* __restrict__ far,
                                                uint32_t* counts, uint32_t cap, const SsspStamps& st) {
  const uint32_t t = tgt[i];
  const float nd = __fadd_rn(du, w[i]);
  const uint32_t nb = __float_as_uint(nd);
  const uint32_t old = atomicMin(dist + t, nb);  // the CAS-min loop of sssp.rs:184-202
  if (nb < old) {
    if (nd < upper) {
      if (atomicMax(st.near_stamp + t, st.pass) < st.pass) {
        const uint32_t pos = sssp_reserve(counts + 0);
        if (pos < cap) near_out[pos] = t;
      }
    } else {
      if (atomicExch(st.in_pile + t, 1u) == 0u) {
        const uint32_t pos = sssp_reserve(counts + 1);
        if (pos < cap) far[pos] = t;
      }
    }
  }
}

// kPark: an entry whose row is not in `rows` is appended to park_list (once per vertex) instead of relaxed
template <bool kPark>
__global__ void k_sssp_relax(const uint32_t* __restrict__ off, const uint32_t* __restrict__ tgt,
                             const float* __restrict__ w, uint32_t* dist, const uint32_t* __restrict__ queue,
                             uint32_t count, float lower, float upper, uint32_t* __restrict__ near_out,
                             uint32_t* __restrict__ far, uint32_t* counts, uint32_t cap, const SsspStamps st,
                             const SsspRows rows, uint32_t* __restrict__ park_list) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t nthreads = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t qb = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) & ~31ull; qb < count; qb += nthreads) {
    const uint64_t q = qb + lane;
    uint32_t b = 0, e = 0;
    float du = 0.0f;
    bool live = q < count;
    if (live) {
      const uint32_t u = queue[q];
      du = __uint_as_float(*((volatile uint32_t*)(dist + u)));
      live = !(du < lower);  // stale entry: settled in an earlier bucket (sssp.rs:126)
      if (kPark && live && !rows.present(u)) {
        if (atomicExch(rows.parked + u, 1u) == 0u) {
          const uint32_t pos = sssp_reserve(counts + 4);
          if (pos < cap) park_list[pos] = u;
        }
        live = false;
      }
      if (live) {
        b = off[u];
        e = off[u + 1];
        live = e > b;
      }
    }
    const bool small = live && (e - b) <= 8;
    if (small)
      for (uint32_t i = b; i < e; ++i) sssp_relax_edge(tgt, w, dist, i, du, upper, near_out, far, counts, cap, st);
    unsigned mask = __ballot_sync(0xFFFFFFFFu, live && !small);
    while (mask) {
      const int owner = __ffs(mask) - 1;
      mask &= mask - 1;
      const uint32_t ob = __shfl_sync(0xFFFFFFFFu, b, owner), oe = __shfl_sync(0xFFFFFFFFu, e, owner);
      const float odu = __shfl_sync(0xFFFFFFFFu, du, owner);
      for (uint32_t i = ob + lane; i < oe; i += 32)
        sssp_relax_edge(tgt, w, dist, i, odu, upper, near_out, far, counts, cap, st);
    }
  }
}

// The parked vertices whose rows are now in `rows` leave the list (clearing their flag) for the near queue,
// appended after its counts[0] entries and stamped with the pass that filled it, so that a vertex already
// queued there is not queued twice; the rest are carried to parked_out (counts[5]).
__global__ void k_sssp_unpark(const uint32_t* __restrict__ parked, uint32_t count, const SsspRows rows,
                              uint32_t* __restrict__ near_out, uint32_t* __restrict__ parked_out, uint32_t* counts,
                              uint32_t cap, const SsspStamps st) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t u = parked[i];
    if (rows.present(u)) {
      rows.parked[u] = 0u;
      if (atomicMax(st.near_stamp + u, st.pass) < st.pass) {
        const uint32_t pos = sssp_reserve(counts + 0);
        if (pos < cap) near_out[pos] = u;
      }
    } else {
      const uint32_t pos = sssp_reserve(counts + 5);
      if (pos < cap) parked_out[pos] = u;
    }
  }
}

// splits the far pile at the new bucket bound; entries whose distance dropped below `lower` were
// settled already and are discarded.  An entry that leaves the pile clears in_pile; one that stays keeps it,
// so k_sssp_relax does not append the vertex a second time while it waits (a vertex improved in k buckets
// while it stayed far used to have k entries).  Carried entries cost no write.
__global__ void k_sssp_split_far(const uint32_t* __restrict__ dist, const uint32_t* __restrict__ far_in,
                                 uint32_t count, float lower, float upper, uint32_t* __restrict__ near_out,
                                 uint32_t* __restrict__ far_out, uint32_t* counts, uint32_t cap,
                                 uint32_t* __restrict__ in_pile) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t t = far_in[i];
    const float d = __uint_as_float(dist[t]);
    if (d < upper) in_pile[t] = 0u;
    if (d < lower) continue;
    if (d < upper) {
      uint32_t pos = sssp_reserve(counts + 0);
      if (pos < cap) near_out[pos] = t;
    } else {
      uint32_t pos = sssp_reserve(counts + 2);
      if (pos < cap) far_out[pos] = t;
    }
  }
}

__global__ void k_sssp_min_far(const uint32_t* __restrict__ dist, const uint32_t* __restrict__ far,
                               uint32_t count, float lower, uint32_t* min_bits) {
  uint32_t best = 0xFFFFFFFFu;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t d = dist[far[i]];
    if (__uint_as_float(d) >= lower && d < best) best = d;
  }
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, o));
  if ((threadIdx.x & 31) == 0 && best != 0xFFFFFFFFu) atomicMin(min_bits, best);
}

// ---- the one-shot call's chunks (gb_sssp_csr_u32) ---------------------------------------------------------------
thread_local gb_sssp_csr_stats sssp_csr_last{};  // behind gb_sssp_csr_info

// Everything one call holds besides its work buffers.  Chunks go out in the feed's send order; `avail` of them (a
// prefix of that order) have passed their checks and may be read by the compute stream, which waits on the last
// one's `checked` event.  The destructor drains the compute stream before the feed (the first member) goes.
struct SsspCsrCall {
  CheckedFeed feed;  // the offsets [0, n], the resident targets and values, sent from the start's chunk on
  cudaStream_t compute = nullptr;
  uint32_t avail = 0;
  uint64_t step = 0;  // GB_SSSP_FEED_STEP: the j-th chunk goes out after j * step passes, and is waited for
  gb_sssp_csr_stats info{};

  ~SsspCsrCall() {
    if (compute) cudaStreamSynchronize(compute), cudaStreamDestroy(compute);
  }
  // once a relax pass is launched: from pageable memory the copies are synchronous, one chunk per pass
  gb_status after_launch() {
    info.passes += 1;
    if (avail < feed.K) info.passes_before_last_landed += 1;
    if (!feed.pinned && !step && feed.issued < feed.K) GB_TRY(feed.issue());
    return GB_OK;
  }
  // Raises avail over the chunks whose checks have passed, without waiting, unless the step rule sends and
  // waits for chunks or `block` asks for one more chunk at least.  A chunk that failed stops the call.
  gb_status poll(bool block, bool* raised) {
    const uint32_t was = avail, K = feed.K;
    if (step)
      while (feed.issued < K && feed.issued * step <= info.passes) GB_TRY(feed.issue());
    if (block && avail == feed.issued) {
      if (feed.issued == K) return fail(GB_ERR_CUDA, "sssp: parked vertices with every chunk available");
      GB_TRY(feed.issue());
    }
    while (avail < feed.issued) {
      if (step || (block && avail == was)) {
        GB_CUDA(cudaEventSynchronize(feed.checked[avail]));
      } else {
        const cudaError_t e = cudaEventQuery(feed.checked[avail]);
        if (e == cudaErrorNotReady) break;
        GB_CUDA(e);
      }
      if (feed.h_bad[1 + feed.order[avail]]) return feed.check_all();
      ++avail;
    }
    *raised = avail > was;
    if (*raised) GB_CUDA(cudaStreamWaitEvent(compute, feed.checked[avail - 1], 0));
    return GB_OK;
  }
  SsspRows rows(uint32_t* parked) const {
    const uint32_t n = feed.n, first = feed.ch.row[feed.order[0]];
    uint32_t span = avail ? n : 0u;
    if (avail && avail < feed.K) {
      const uint32_t stop = feed.ch.row[feed.order[avail]];  // the first row not yet available
      span = stop > first ? stop - first : stop + (n - first);
    }
    return SsspRows{first, span, n, parked};
  }
};

// ---- the bucket loop ----------------------------------------------------------------------------------------
// The device buffers of one run; the parked list and flags only with a feed
struct SsspWork {
  DevBuf<uint32_t> qa, qb, fa, fb, counts, minb, near_stamp, in_pile;
  DevBuf<uint32_t> pa, pb, parked;
};

// Delta-stepping from `start` over the out-CSR (off, tgt, w) on stream s, into dist.  Without a feed every row is
// present (gb_sssp); with one (gb_sssp_csr_u32) the rows are those of feed->rows() and the loop parks, unparks
// and waits for chunks as the header of this file says.
static gb_status sssp_loop(cudaStream_t s, uint32_t n, const uint32_t* off, const uint32_t* tgt, const float* w,
                           uint32_t* dist, uint32_t start, float delta, SsspWork& wk, SsspCsrCall* feed,
                           uint64_t* launches) {
  const unsigned blk = 256;
  const uint32_t cap = n;
  SsspStamps st{wk.near_stamp.p, wk.in_pile.p, 0u};
  uint32_t* counts = wk.counts.p;
  k_sssp_init<<<grid_for(n, blk), blk, 0, s>>>(dist, n, start);
  GB_CUDA(cudaMemcpyAsync(wk.qa.p, &start, 4, cudaMemcpyHostToDevice, s));
  *launches += 1;
  uint32_t* near_in = wk.qa.p;
  uint32_t* near_out = wk.qb.p;
  uint32_t* far = wk.fa.p;
  uint32_t* far_out = wk.fb.p;
  uint32_t near_count = 1, far_count = 0, parked_count = 0;
  float lower = 0.0f, upper = delta;  // the current bucket (sssp_bucket.h)
  uint32_t h_counts[6];
  SsspRows rows = feed ? feed->rows(wk.parked.p) : SsspRows{0u, n, n, nullptr};
  bool any_parked = false;  // from the first park on, no pass drops an entry by `du < lower`
  // the parked vertices whose rows are present now go to the near queue, after its near_count entries
  auto unpark = [&]() -> gb_status {
    rows = feed->rows(wk.parked.p);
    const uint32_t set[6] = {near_count, far_count, 0u, 0u, parked_count, 0u};
    GB_CUDA(cudaMemcpyAsync(counts, set, 24, cudaMemcpyHostToDevice, s));
    k_sssp_unpark<<<grid_for(parked_count, blk), blk, 0, s>>>(wk.pa.p, parked_count, rows, near_in, wk.pb.p, counts,
                                                              cap, st);
    *launches += 1;
    GB_CUDA(cudaMemcpyAsync(h_counts, counts, 24, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    if (h_counts[0] > cap || h_counts[5] > cap) return fail(GB_ERR_OOM, "sssp work queue overflow");
    near_count = h_counts[0];
    parked_count = h_counts[5];
    std::swap(wk.pa.p, wk.pb.p);
    feed->info.unpark_rounds += 1;
    return GB_OK;
  };
  for (;;) {
    // drain the near queue of this bucket
    while (near_count > 0) {
      st.pass += 1;
      if (!feed) {
        const uint32_t zero2[2] = {0u, far_count};
        GB_CUDA(cudaMemcpyAsync(counts, zero2, 8, cudaMemcpyHostToDevice, s));
        k_sssp_relax<false><<<grid_for((uint64_t)near_count, blk), blk, 0, s>>>(
            off, tgt, w, dist, near_in, near_count, lower, upper, near_out, far, counts, cap, st, rows, nullptr);
      } else {
        const uint32_t zero5[5] = {0u, far_count, 0u, 0u, parked_count};
        GB_CUDA(cudaMemcpyAsync(counts, zero5, 20, cudaMemcpyHostToDevice, s));
        k_sssp_relax<true><<<grid_for((uint64_t)near_count, blk), blk, 0, s>>>(
            off, tgt, w, dist, near_in, near_count, any_parked ? 0.0f : lower, upper, near_out, far, counts, cap, st,
            rows, wk.pa.p);
        GB_TRY(feed->after_launch());
      }
      *launches += 1;
      GB_CUDA(cudaMemcpyAsync(h_counts, counts, feed ? 20 : 8, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
      if (h_counts[0] > cap || h_counts[1] > cap) return fail(GB_ERR_OOM, "sssp work queue overflow");
      near_count = h_counts[0];
      far_count = h_counts[1];
      std::swap(near_in, near_out);
      if (feed) {
        if (h_counts[4] > cap) return fail(GB_ERR_OOM, "sssp work queue overflow");
        feed->info.parked += h_counts[4] - parked_count;
        parked_count = h_counts[4];
        any_parked = any_parked || parked_count > 0;
        bool raised = false;
        GB_TRY(feed->poll(false, &raised));
        if (raised) rows = feed->rows(wk.parked.p);
        if (raised && parked_count > 0) GB_TRY(unpark());
      }
    }
    if (far_count > 0) {
      // next non-empty bucket: the smallest live distance in the far pile decides (min_non_empty_bin,
      // sssp.rs:159-168)
      const uint32_t inf = 0xFFFFFFFFu;
      GB_CUDA(cudaMemcpyAsync(wk.minb.p, &inf, 4, cudaMemcpyHostToDevice, s));
      k_sssp_min_far<<<grid_for(far_count, blk), blk, 0, s>>>(dist, far, far_count, upper, wk.minb.p);
      uint32_t h_min = inf;
      GB_CUDA(cudaMemcpyAsync(&h_min, wk.minb.p, 4, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
      *launches += 1;
      if (h_min != inf) {
        float dmin;
        memcpy(&dmin, &h_min, 4);
        const SsspBucket next = sssp_next_bucket(dmin, delta, upper);
        lower = next.lower;
        upper = next.upper;
        const uint32_t zero3[3] = {0u, 0u, 0u};
        GB_CUDA(cudaMemcpyAsync(counts, zero3, 12, cudaMemcpyHostToDevice, s));
        // anything below lower in the pile was settled (its distance was final when its bucket drained)
        k_sssp_split_far<<<grid_for(far_count, blk), blk, 0, s>>>(dist, far, far_count, 0.0f, upper, near_in,
                                                                 far_out, counts, cap, st.in_pile);
        *launches += 1;
        GB_CUDA(cudaMemcpyAsync(h_counts, counts, 12, cudaMemcpyDeviceToHost, s));
        GB_CUDA(cudaStreamSynchronize(s));
        near_count = h_counts[0];
        far_count = h_counts[2];
        std::swap(far, far_out);
        continue;
      }
      // everything left in the pile is stale: each of its vertices was improved below the pile's bucket since,
      // and was queued near then
      far_count = 0;
    }
    if (!feed || parked_count == 0) break;
    // only parked vertices are left: wait for the next chunk
    bool raised = false;
    GB_TRY(feed->poll(true, &raised));
    GB_TRY(unpark());
  }
  GB_CUDA(cudaGetLastError());
  return GB_OK;
}

static gb_status sssp_impl(const gb_graph* g, const gb_sssp_config* cfg, float* d_dist, float* h_dist) {
  GB_REQUIRE(g && cfg, "NULL argument");
  if (g->kind != GB_KIND_DIRECTED) return fail(GB_ERR_UNSUPPORTED, "sssp needs a directed graph");
  if (!g->out.w.p)
    return fail(GB_ERR_UNSUPPORTED, "sssp needs f32 edge values (DirectedNeighborsWithValues<NI, f32>, sssp.rs:41)");
  GB_REQUIRE(cfg->start_node < g->n, "start_node %llu out of range (n = %u)",
             (unsigned long long)cfg->start_node, g->n);
  GB_REQUIRE(cfg->delta > 0.0f && cfg->delta < FLT_MAX, "delta must be a positive finite f32");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  cudaStream_t s = g->stream;
  const uint32_t n = g->n;
  DevBuf<float> tmp;
  if (!d_dist) {
    GB_TRY(tmp.alloc(n));
    d_dist = tmp.p;
  }
  uint32_t* dist = reinterpret_cast<uint32_t*>(d_dist);
  // a vertex is appended at most once per pass to the near queue (near stamps), and the far pile holds it
  // at most once (in_pile): n bounds every queue for every delta (the overflow check in the loop is an
  // internal-error guard only)
  const uint32_t cap = n;
  SsspWork wk;
  GB_TRY(wk.near_stamp.alloc(n));
  GB_TRY(wk.in_pile.alloc(n));
  GB_CUDA(cudaMemsetAsync(wk.near_stamp.p, 0, (size_t)n * 4, s));
  GB_CUDA(cudaMemsetAsync(wk.in_pile.p, 0, (size_t)n * 4, s));
  GB_TRY(wk.qa.alloc(cap));
  GB_TRY(wk.qb.alloc(cap));
  GB_TRY(wk.fa.alloc(cap));
  GB_TRY(wk.fb.alloc(cap));
  GB_TRY(wk.counts.alloc(4));
  GB_TRY(wk.minb.alloc(1));
  g->timing = gb_timing{};
  GB_CUDA(cudaEventRecord(g->ev_begin, s));
  GB_TRY(sssp_loop(s, n, g->out.off.p, g->out.tgt.p, g->out.w.p, dist, (uint32_t)cfg->start_node, cfg->delta, wk,
                   nullptr, &g->timing.kernel_launches));
  GB_CUDA(cudaEventRecord(g->ev_end, s));
  if (h_dist) GB_CUDA(cudaMemcpyAsync(h_dist, d_dist, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  float ms = 0.0f;
  GB_CUDA(cudaEventElapsedTime(&ms, g->ev_begin, g->ev_end));
  g->timing.total_ms = ms;
  return GB_OK;
}

// ---- one-shot SSSP of a host out-CSR (gb_sssp_csr_u32) ----------------------------------------------------------
// The checks and messages are those of gb_digraph_from_csr_u32 + gb_sssp for the same out-CSR, in the order of
// the header: the O(1) host checks, the values, the config, then the device checks of the offsets and targets.
static gb_status sssp_csr(int device, uint32_t n, const uint32_t* off, const uint32_t* tgt, const float* w,
                          const gb_sssp_config* cfg, float* distances) {
  sssp_csr_last = gb_sssp_csr_stats{};
  GB_REQUIRE(distances != nullptr, "distances is NULL");
  GB_REQUIRE(cfg != nullptr, "config is NULL");
  GB_REQUIRE(n > 0, "node_count must be > 0");
  GB_TRY(require_device(device));
  GB_TRY(require_host_csr(n, off, tgt, "out"));
  const uint64_t m = off[n];
  if (m > 0 && !w)
    return fail(GB_ERR_UNSUPPORTED, "sssp needs f32 edge values (DirectedNeighborsWithValues<NI, f32>, sssp.rs:41)");
  GB_REQUIRE(cfg->start_node < n, "start_node %llu out of range (n = %u)", (unsigned long long)cfg->start_node, n);
  GB_REQUIRE(cfg->delta > 0.0f && cfg->delta < FLT_MAX, "delta must be a positive finite f32");
  DeviceGuard guard(device);
  GB_CUDA(cudaSetDevice(device));
  const uint32_t start = (uint32_t)cfg->start_node;
  SsspCsrCall t;
  CheckedFeed& f = t.feed;
  t.step = env_u64("GB_SSSP_FEED_STEP", 0);
  GB_CUDA(cudaStreamCreateWithFlags(&t.compute, cudaStreamNonBlocking));
  SsspWork wk;
  DevBuf<float> dist;
  GB_TRY(dist.alloc(n));
  for (DevBuf<uint32_t>* b : {&wk.qa, &wk.qb, &wk.fa, &wk.fb, &wk.pa, &wk.pb}) GB_TRY(b->alloc(n));
  for (DevBuf<uint32_t>* b : {&wk.near_stamp, &wk.in_pile, &wk.parked}) {
    GB_TRY(b->alloc(n));
    GB_CUDA(cudaMemsetAsync(b->p, 0, (size_t)n * 4, t.compute));
  }
  GB_TRY(wk.counts.alloc(6));
  GB_TRY(wk.minb.alloc(1));
  GB_TRY(f.open(device, n, off, tgt, w, env_u64("GB_SSSP_FEED_ENTRIES", 0), start, "out"));
  gb_sssp_csr_stats& info = t.info;
  info.start_chunk = f.order[0];
  // from pageable memory one chunk goes out while each pass runs (after_launch); the step rule holds page-locked
  // chunks back as well
  const uint32_t ahead = f.pinned && !t.step ? f.K : 1;
  while (f.issued < ahead) GB_TRY(f.issue());
  // the offsets are monotone before anything indexes with them
  GB_TRY(f.require_offsets());
  GB_CUDA(cudaStreamWaitEvent(t.compute, f.offsets_checked, 0));
  bool raised = false;
  GB_TRY(t.poll(true, &raised));  // the start's chunk
  uint64_t launches = 0;
  GB_TRY(sssp_loop(t.compute, n, f.feed.off.p, f.feed.tgt.p, f.feed.val.p, reinterpret_cast<uint32_t*>(dist.p),
                   start, cfg->delta, wk, &t, &launches));
  // the distances are final; a chunk the loop never read still fails the call as the twin's upload would
  GB_TRY(f.check_all());
  info.kernel_launches += launches;
  GB_TRY(f.finish(t.compute, distances, dist.p, (size_t)n * 4));
  GB_TRY(f.report(&info));
  sssp_csr_last = info;
  return GB_OK;
}

}  // namespace gb

extern "C" {
gb_status gb_sssp(const gb_graph* graph, const gb_sssp_config* config, float* distances) {
  GB_REQUIRE(distances != nullptr, "distances is NULL");
  return gb::sssp_impl(graph, config, nullptr, distances);
}
gb_status gb_sssp_device(const gb_graph* graph, const gb_sssp_config* config, float* d_distances) {
  GB_REQUIRE(d_distances != nullptr, "d_distances is NULL");
  return gb::sssp_impl(graph, config, d_distances, nullptr);
}
gb_status gb_sssp_csr_u32(int device, uint32_t node_count, const uint32_t* offsets, const uint32_t* targets,
                          const float* weights, const gb_sssp_config* config, float* distances) {
  return gb::sssp_csr(device, node_count, offsets, targets, weights, config, distances);
}
gb_status gb_sssp_csr_info(gb_sssp_csr_stats* info) {
  GB_REQUIRE(info != nullptr, "info is NULL");
  *info = gb::sssp_csr_last;
  return GB_OK;
}
}
