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
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x)
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

__global__ void k_sssp_relax(const uint32_t* __restrict__ off, const uint32_t* __restrict__ tgt,
                             const float* __restrict__ w, uint32_t* dist, const uint32_t* __restrict__ queue,
                             uint32_t count, float lower, float upper, uint32_t* __restrict__ near_out,
                             uint32_t* __restrict__ far, uint32_t* counts, uint32_t cap, const SsspStamps st) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t nthreads = gridDim.x * blockDim.x;
  for (uint32_t qb = (blockIdx.x * blockDim.x + threadIdx.x) & ~31u; qb < count; qb += nthreads) {
    const uint32_t q = qb + lane;
    uint32_t b = 0, e = 0;
    float du = 0.0f;
    bool live = q < count;
    if (live) {
      const uint32_t u = queue[q];
      du = __uint_as_float(*((volatile uint32_t*)(dist + u)));
      live = !(du < lower);  // stale entry: settled in an earlier bucket (sssp.rs:126)
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

// splits the far pile at the new bucket bound; entries whose distance dropped below `lower` were
// settled already and are discarded.  An entry that leaves the pile clears in_pile; one that stays keeps it,
// so k_sssp_relax does not append the vertex a second time while it waits (a vertex improved in k buckets
// while it stayed far used to have k entries).  Carried entries cost no write.
__global__ void k_sssp_split_far(const uint32_t* __restrict__ dist, const uint32_t* __restrict__ far_in,
                                 uint32_t count, float lower, float upper, uint32_t* __restrict__ near_out,
                                 uint32_t* __restrict__ far_out, uint32_t* counts, uint32_t cap,
                                 uint32_t* __restrict__ in_pile) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
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
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
    const uint32_t d = dist[far[i]];
    if (__uint_as_float(d) >= lower && d < best) best = d;
  }
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, o));
  if ((threadIdx.x & 31) == 0 && best != 0xFFFFFFFFu) atomicMin(min_bits, best);
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
  const uint64_t m = g->out.len;
  DevBuf<float> tmp;
  if (!d_dist) {
    GB_TRY(tmp.alloc(n));
    d_dist = tmp.p;
  }
  uint32_t* dist = reinterpret_cast<uint32_t*>(d_dist);
  // a vertex is appended at most once per pass to the near queue (near stamps), and the far pile holds it
  // at most once (in_pile): n bounds every queue for every delta (the overflow check below is an
  // internal-error guard only)
  (void)m;
  const uint32_t cap = n;
  DevBuf<uint32_t> qa, qb, fa, fb, counts, minb, near_stamp, in_pile;
  GB_TRY(near_stamp.alloc(n));
  GB_TRY(in_pile.alloc(n));
  GB_CUDA(cudaMemsetAsync(near_stamp.p, 0, (size_t)n * 4, s));
  GB_CUDA(cudaMemsetAsync(in_pile.p, 0, (size_t)n * 4, s));
  SsspStamps st{near_stamp.p, in_pile.p, 0u};
  GB_TRY(qa.alloc(cap));
  GB_TRY(qb.alloc(cap));
  GB_TRY(fa.alloc(cap));
  GB_TRY(fb.alloc(cap));
  GB_TRY(counts.alloc(4));
  GB_TRY(minb.alloc(1));
  g->timing = gb_timing{};
  GB_CUDA(cudaEventRecord(g->ev_begin, s));
  const unsigned blk = 256;
  k_sssp_init<<<grid_for(n, blk), blk, 0, s>>>(dist, n, (uint32_t)cfg->start_node);
  const uint32_t start = (uint32_t)cfg->start_node;
  GB_CUDA(cudaMemcpyAsync(qa.p, &start, 4, cudaMemcpyHostToDevice, s));
  g->timing.kernel_launches += 1;
  uint32_t* near_in = qa.p;
  uint32_t* near_out = qb.p;
  uint32_t* far = fa.p;
  uint32_t* far_out = fb.p;
  uint32_t near_count = 1, far_count = 0;
  const float delta = cfg->delta;
  float lower = 0.0f, upper = delta;  // the current bucket (sssp_bucket.h)
  uint32_t h_counts[4];
  for (;;) {
    // drain the near queue of this bucket
    while (near_count > 0) {
      const uint32_t zero2[2] = {0u, far_count};
      GB_CUDA(cudaMemcpyAsync(counts.p, zero2, 8, cudaMemcpyHostToDevice, s));
      st.pass += 1;
      k_sssp_relax<<<grid_for((uint64_t)near_count, blk), blk, 0, s>>>(
          g->out.off.p, g->out.tgt.p, g->out.w.p, dist, near_in, near_count, lower, upper, near_out, far,
          counts.p, cap, st);
      g->timing.kernel_launches += 1;
      GB_CUDA(cudaMemcpyAsync(h_counts, counts.p, 8, cudaMemcpyDeviceToHost, s));
      GB_CUDA(cudaStreamSynchronize(s));
      if (h_counts[0] > cap || h_counts[1] > cap) return fail(GB_ERR_OOM, "sssp work queue overflow");
      near_count = h_counts[0];
      far_count = h_counts[1];
      std::swap(near_in, near_out);
    }
    if (far_count == 0) break;
    // next non-empty bucket: the smallest live distance in the far pile decides (min_non_empty_bin,
    // sssp.rs:159-168)
    const uint32_t inf = 0xFFFFFFFFu;
    GB_CUDA(cudaMemcpyAsync(minb.p, &inf, 4, cudaMemcpyHostToDevice, s));
    k_sssp_min_far<<<grid_for(far_count, blk), blk, 0, s>>>(dist, far, far_count, upper, minb.p);
    uint32_t h_min = inf;
    GB_CUDA(cudaMemcpyAsync(&h_min, minb.p, 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    g->timing.kernel_launches += 1;
    if (h_min == inf) break;  // everything left in the pile is stale
    float dmin;
    memcpy(&dmin, &h_min, 4);
    const SsspBucket next = sssp_next_bucket(dmin, delta, upper);
    lower = next.lower;
    upper = next.upper;
    const uint32_t zero3[3] = {0u, 0u, 0u};
    GB_CUDA(cudaMemcpyAsync(counts.p, zero3, 12, cudaMemcpyHostToDevice, s));
    // anything below lower in the pile was settled (its distance was final when its bucket drained)
    k_sssp_split_far<<<grid_for(far_count, blk), blk, 0, s>>>(dist, far, far_count, 0.0f, upper, near_in, far_out,
                                                             counts.p, cap, st.in_pile);
    g->timing.kernel_launches += 1;
    GB_CUDA(cudaMemcpyAsync(h_counts, counts.p, 12, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    near_count = h_counts[0];
    far_count = h_counts[2];
    std::swap(far, far_out);
  }
  GB_CUDA(cudaGetLastError());
  GB_CUDA(cudaEventRecord(g->ev_end, s));
  if (h_dist) GB_CUDA(cudaMemcpyAsync(h_dist, d_dist, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  float ms = 0.0f;
  GB_CUDA(cudaEventElapsedTime(&ms, g->ev_begin, g->ev_end));
  g->timing.total_ms = ms;
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
}
