// wcc.cu — weakly connected components (Afforest) on the device CSR pair.
//
// Replaces crates/algos/src/wcc.rs:127-139,158-301 (`wcc_afforest`, `sample_subgraph`,
// `find_largest_component`, `link_remaining`) and crates/algos/src/afforest.rs:22-56,100-114
// (`Afforest::union/compress/to_vec`).  Same five phases, same link rule (hook the higher root
// under the lower with a CAS), so parent[x] <= x holds throughout and after the final compress
// every entry is the minimum node id of its component — the value `to_vec()` returns.
//
// Algorithmic bytes per run: 8m + 16n + 8 (both CSRs once, parent read + write); the sampling
// phase lets most vertices skip their edge lists, so effective GB/s can exceed the HBM peak.
#include <algorithm>
#include <cstdlib>
#include <memory>
#include <vector>

#include "common.cuh"
#include "csr_split.h"

namespace gb {

__device__ __forceinline__ uint32_t ld_parent(const uint32_t* p, uint32_t i) {
  return *((const volatile uint32_t*)(p + i));
}

// Afforest::union, afforest.rs:22-39
__device__ __forceinline__ void af_link(uint32_t* parent, uint32_t u, uint32_t v) {
  uint32_t p1 = ld_parent(parent, u);
  uint32_t p2 = ld_parent(parent, v);
  while (p1 != p2) {
    const uint32_t high = p1 > p2 ? p1 : p2;
    const uint32_t low = p1 + p2 - high;
    const uint32_t p_high = ld_parent(parent, high);
    if (p_high == low) break;
    if (p_high == high && atomicCAS(parent + high, high, low) == high) break;
    p1 = ld_parent(parent, ld_parent(parent, high));
    p2 = ld_parent(parent, low);
  }
}

__global__ void k_cc_init(uint32_t* __restrict__ parent, uint32_t n) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) parent[v] = v;
}

// sample_subgraph, wcc.rs:186-204: link u with its first `rounds` out-neighbours
__global__ void k_cc_sample(const uint32_t* __restrict__ off, const uint32_t* __restrict__ tgt, uint32_t vb,
                            uint32_t n, uint32_t rounds, uint32_t* parent) {
  for (uint32_t u = vb + blockIdx.x * blockDim.x + threadIdx.x; u < n; u += gridDim.x * blockDim.x) {
    const uint32_t b = off[u], e = off[u + 1];
    const uint32_t lim = (e - b < rounds) ? e : b + rounds;  // out_neighbors(u).take(neighbor_rounds)
    for (uint32_t i = b; i < lim; ++i) af_link(parent, u, tgt[i]);
  }
}

// Afforest::compress, afforest.rs:50-56
__global__ void k_cc_compress(uint32_t* parent, uint32_t n) {
  for (uint32_t x = blockIdx.x * blockDim.x + threadIdx.x; x < n; x += gridDim.x * blockDim.x) {
    uint32_t p = ld_parent(parent, x);
    uint32_t pp = ld_parent(parent, p);
    while (p != pp) {
      parent[x] = pp;
      p = pp;
      pp = ld_parent(parent, p);
    }
  }
}

__global__ void k_cc_sample_labels(const uint32_t* __restrict__ parent, uint32_t n, uint32_t count,
                                   uint64_t seed, uint32_t* __restrict__ out) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) {
    uint64_t z = seed + 0x9E3779B97F4A7C15ull * (i + 1);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    out[i] = parent[(uint32_t)(z % n)];
  }
}

// the root of x; every non-root on the way is pointed at its grandparent (path halving).  The writes race
// only with writes of other ancestors, and a CAS only ever changes a root, so parent[y] <= y and every tree
// stay as they were
__device__ __forceinline__ uint32_t find_halving(uint32_t* parent, uint32_t x) {
  uint32_t p = ld_parent(parent, x);
  while (true) {
    const uint32_t gp = ld_parent(parent, p);
    if (gp == p) return p;
    parent[x] = gp;
    x = gp;
    p = ld_parent(parent, x);
  }
}

// Afforest::union's rule (hook the higher root under the lower with a CAS) on roots found with path halving.
// af_link walks parent chains without shortening them; edges linked all at once in id order (a path) build
// chains as long as the chunk, which only path halving keeps cheap to walk and to compress.  k_cc_link_remaining
// links with it too: its lanes hook the vertices of an unsampled path into a chain as deep as the path while
// the warp of a hub on that path walks the chain once per entry of its lists
__device__ __forceinline__ void link_halving(uint32_t* parent, uint32_t u, uint32_t v) {
  uint32_t a = find_halving(parent, u), b = find_halving(parent, v);
  while (a != b) {
    const uint32_t high = a > b ? a : b;
    const uint32_t low = a + b - high;
    const uint32_t prev = atomicCAS(parent + high, high, low);
    if (prev == high) return;
    a = find_halving(parent, prev);  // high was hooked meanwhile
    b = find_halving(parent, low);
  }
}

// link_remaining, wcc.rs:274-301: one warp per vertex outside the sampled giant component.  A vertex is
// skipped only while parent[v] == skip, so it is already joined to the giant; once skip is hooked under a
// lower root a halving find may point a giant vertex past it, and that vertex then links its lists again
__global__ void k_cc_link_remaining(const uint32_t* __restrict__ out_off, const uint32_t* __restrict__ out_tgt,
                                    const uint32_t* __restrict__ in_off, const uint32_t* __restrict__ in_tgt,
                                    uint32_t vb, uint32_t n, uint32_t rounds, uint32_t skip, int use_skip,
                                    uint32_t* parent) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  // lanes first test 32 consecutive vertices, then the warp serves the survivors one by one
  for (uint32_t base = vb + warp * 32; base < n; base += nwarps * 32) {
    const uint32_t mine = base + lane;
    bool live = mine < n;
    uint32_t ob = 0, oe = 0, ib = 0, ie = 0;
    if (live) {
      // offsets are read lane-parallel (coalesced); vertices without remaining edges (all isolated
      // vertices, ~half of an R-MAT graph) never enter the warp-serial part
      ob = out_off[mine];
      oe = out_off[mine + 1];
      ib = in_off[mine];
      ie = in_off[mine + 1];
      ob = (oe - ob > rounds) ? ob + rounds : oe;
      live = (oe > ob) || (ie > ib);
    }
    if (live && use_skip) live = ld_parent(parent, mine) != skip;
    // short lists are linked by their own lane; long ones are served by the whole warp
    const uint32_t work = (oe - ob) + (ie - ib);
    const bool small = live && work <= 8;
    if (small) {
      for (uint32_t i = ob; i < oe; ++i) link_halving(parent, mine, out_tgt[i]);
      for (uint32_t i = ib; i < ie; ++i) link_halving(parent, mine, in_tgt[i]);
    }
    unsigned mask = __ballot_sync(0xFFFFFFFFu, live && !small);
    while (mask) {
      const int owner = __ffs(mask) - 1;
      mask &= mask - 1;
      const uint32_t u = base + owner;
      const uint32_t b0 = __shfl_sync(0xFFFFFFFFu, ob, owner), e0 = __shfl_sync(0xFFFFFFFFu, oe, owner);
      const uint32_t b1 = __shfl_sync(0xFFFFFFFFu, ib, owner), e1 = __shfl_sync(0xFFFFFFFFu, ie, owner);
      for (uint32_t i = b0 + lane; i < e0; i += 32) link_halving(parent, u, out_tgt[i]);
      for (uint32_t i = b1 + lane; i < e1; i += 32) link_halving(parent, u, in_tgt[i]);
    }
  }
}

// the most frequent label among `sampling_size` pseudo-random vertices (fixed seed: every rank of a
// sharded run that holds the same parent array picks the same label)
static gb_status most_frequent_label(cudaStream_t s, const uint32_t* d_parent, uint32_t n, uint64_t sampling_size,
                                     uint32_t* label, int* found) {
  *label = 0;
  *found = 0;
  const uint32_t samples = (uint32_t)std::min<uint64_t>(sampling_size, 1u << 20);
  if (samples == 0 || n == 0) return GB_OK;
  DevBuf<uint32_t> d_samp;
  GB_TRY(d_samp.alloc(samples));
  k_cc_sample_labels<<<grid_for(samples, 256), 256, 0, s>>>(d_parent, n, samples, 0x5DEECE66Dull, d_samp.p);
  std::vector<uint32_t> h(samples);
  GB_CUDA(cudaMemcpyAsync(h.data(), d_samp.p, (size_t)samples * 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  std::sort(h.begin(), h.end());
  uint32_t best_cnt = 0, run = 0;
  for (uint32_t i = 0; i < samples; ++i) {
    run = (i > 0 && h[i] == h[i - 1]) ? run + 1 : 1;
    if (run > best_cnt) {
      best_cnt = run;
      *label = h[i];
    }
  }
  *found = 1;
  return GB_OK;
}

// union of two forests over the same vertex set: every tree edge (v, other[v]) of the other forest is
// linked into parent[] with the Afforest rule, so parent[] ends up connecting what either forest connected
__global__ void k_cc_merge(uint32_t* parent, const uint32_t* __restrict__ other, uint32_t n) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    const uint32_t o = other[v];
    if (o != v) af_link(parent, v, o);
  }
}

// ---- one-shot WCC of a host out-CSR (gb_wcc_csr_u32): wcc_baseline, wcc.rs:103-123 ----------------------
constexpr uint32_t LINK_TILE = 128;  // edges per warp step of k_cc_link_edges: one uint4 of targets per lane

// the row r in [lo, hi) with off[r] <= e < off[r + 1], given off[lo] <= e < off[hi]
__device__ __forceinline__ uint32_t row_search(const uint32_t* __restrict__ off, uint32_t lo, uint32_t hi, uint32_t e) {
  while (hi - lo > 1) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (off[mid] <= e) lo = mid;
    else hi = mid;
  }
  return lo;
}

// the same search by a whole warp: 31 probes per step cut [lo, hi) 32-fold, so a row among 2^24 is found
// in five dependent loads
__device__ __forceinline__ uint32_t warp_row_search(const uint32_t* __restrict__ off, uint32_t lo, uint32_t hi,
                                                    uint32_t e, uint32_t lane) {
  while (hi - lo > 1) {
    const uint32_t p = lo + (uint32_t)(((uint64_t)(hi - lo) * (lane + 1)) >> 5);  // lane 31 would probe hi
    const unsigned le = __ballot_sync(0xFFFFFFFFu, lane < 31 && off[p] <= e);   // a prefix of the lanes
    const int c = __popc(le);
    const uint32_t below = __shfl_sync(0xFFFFFFFFu, p, c > 0 ? c - 1 : 0);
    const uint32_t above = __shfl_sync(0xFFFFFFFFu, p, c < 31 ? c : 0);
    if (c > 0) lo = below;
    if (c < 31) hi = above;
  }
  return lo;
}

// Links every edge of one chunk: tgt holds the targets of the edges [e0, e0 + len) of the CSR (e0 a multiple
// of 4, 8 entries of slack behind len), and off the device offsets of its rows [row_base, row_base + rows]
// (the whole CSR: row_base 0, rows n), with off[0] <= e0 and e0 + len <= off[rows].  Edge-parallel: warp
// step t takes the 128 edges from e0 + 128t, finds the row of the first one with a warp search over all
// those offsets and an upper bound for the last one with 32 galloping probes, and each lane then places its
// 4 edges by binary search inside that window.  A hub row split over chunks and warps, or a run of empty
// rows, costs a search of logarithmic depth, never a walk.  Targets >= n are counted in *bad and not linked.
__global__ void __launch_bounds__(256) k_cc_link_edges(const uint32_t* __restrict__ off, uint32_t rows,
                                                       uint32_t row_base, const uint32_t* __restrict__ tgt,
                                                       uint32_t e0, uint32_t len, uint32_t n, uint32_t* parent,
                                                       unsigned int* bad) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t tiles = (len + LINK_TILE - 1) / LINK_TILE;
  unsigned int nbad = 0;
  for (uint32_t t = warp; t < tiles; t += nwarps) {
    const uint32_t b = t * LINK_TILE;  // chunk-local
    const uint32_t g0 = e0 + b, glast = g0 + min(LINK_TILE, len - b) - 1;
    const uint32_t r0 = warp_row_search(off, 0, rows, g0, lane);
    // hi: the first of r0 + 1, r0 + 2, r0 + 4, ... whose row starts after the tile (off[rows] > glast)
    const uint64_t step = (uint64_t)r0 + (1ull << lane);
    const uint32_t probe = step < rows ? (uint32_t)step : rows;
    const unsigned past = __ballot_sync(0xFFFFFFFFu, off[probe] > glast);
    const uint32_t hi = past ? __shfl_sync(0xFFFFFFFFu, probe, __ffs(past) - 1) : rows;
    const uint32_t l0 = b + 4 * lane;
    if (l0 < len) {
      const uint4 v4 = *reinterpret_cast<const uint4*>(tgt + l0);
      const uint32_t v[4] = {v4.x, v4.y, v4.z, v4.w};
      uint32_t r = row_search(off, r0, hi, e0 + l0);
#pragma unroll
      for (uint32_t j = 0; j < 4; ++j) {
        if (l0 + j >= len) break;
        const uint32_t e = e0 + l0 + j;
        if (j && off[r + 1] <= e) r = row_search(off, r + 1, hi, e);
        if (v[j] < n) link_halving(parent, row_base + r, v[j]);
        else ++nbad;
      }
    }
  }
  nbad = __reduce_add_sync(0xFFFFFFFFu, nbad);
  if (lane == 0 && nbad) atomicAdd(bad, nbad);
}

// union of another part's forest into this one (gb_wcc_csr_multi_u32): other is that part's compressed
// parent[], a peer device's memory or this device's, read once and coalesced.  The links halve paths as the
// edge links do, for the same reason: a forest can hold chains as long as the graph's paths
__global__ void k_cc_merge_halving(uint32_t* parent, const uint32_t* __restrict__ other, uint32_t n) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    const uint32_t o = other[v];
    if (o != v) link_halving(parent, v, o);
  }
}

static gb_status wcc_impl(const gb_graph* g, const gb_wcc_config* cfg, uint32_t* d_comp, uint32_t* h_comp) {
  GB_REQUIRE(g && cfg, "NULL argument");
  if (g->kind != GB_KIND_DIRECTED)
    return fail(GB_ERR_UNSUPPORTED, "wcc needs a directed graph (wcc.rs:130: DirectedNeighbors)");
  GB_REQUIRE(g->out.len == 0 || g->out.tgt.p != nullptr, "this handle holds no out targets (page-rank-only twin)");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  cudaStream_t s = g->stream;
  const uint32_t n = g->n;
  DevBuf<uint32_t> tmp;
  if (!d_comp) {
    GB_TRY(tmp.alloc(n));
    d_comp = tmp.p;
  }
  g->timing = gb_timing{};
  GB_CUDA(cudaEventRecord(g->ev_begin, s));
  const unsigned blk = 256;
  const unsigned grid = grid_for(n, blk);
  const uint32_t rounds = (uint32_t)std::min<uint64_t>(cfg->neighbor_rounds, 0xFFFFFFFFull);
  k_cc_init<<<grid, blk, 0, s>>>(d_comp, n);
  // sample_subgraph, wcc.rs:186-204: every vertex links its first `neighbor_rounds` out-neighbours
  const uint32_t sample_rounds = rounds;
  if (sample_rounds) k_cc_sample<<<grid, blk, 0, s>>>(g->out.off.p, g->out.tgt.p, 0, n, sample_rounds, d_comp);
  k_cc_compress<<<grid, blk, 0, s>>>(d_comp, n);
  g->timing.kernel_launches += 2 + (sample_rounds ? 1 : 0);
  // find_largest_component, wcc.rs:245-271 (which component is skipped never changes the result)
  uint32_t skip = 0;
  int use_skip = 0;
  GB_TRY(most_frequent_label(s, d_comp, n, cfg->sampling_size, &skip, &use_skip));
  if (use_skip) g->timing.kernel_launches += 1;
  k_cc_link_remaining<<<grid_for((uint64_t)n, blk), blk, 0, s>>>(g->out.off.p, g->out.tgt.p, g->in.off.p,
                                                               g->in.tgt.p, 0, n, sample_rounds, skip, use_skip,
                                                               d_comp);
  k_cc_compress<<<grid, blk, 0, s>>>(d_comp, n);
  g->timing.kernel_launches += 2;
  GB_CUDA(cudaGetLastError());
  GB_CUDA(cudaEventRecord(g->ev_end, s));
  if (h_comp) GB_CUDA(cudaMemcpyAsync(h_comp, d_comp, (size_t)n * 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  float ms = 0.0f;
  GB_CUDA(cudaEventElapsedTime(&ms, g->ev_begin, g->ev_end));
  g->timing.total_ms = ms;
  return GB_OK;
}

// The targets of gb_wcc_csr_u32 cross the bus in chunks of C edges through a ring of WCC_FEED_RING device
// buffers; chunk k is the edges [kC, min((k + 1)C, m)), whatever rows it cuts.
constexpr uint32_t WCC_FEED_RING = 3;
constexpr uint64_t WCC_FEED_EDGES = 1u << 22;  // C: 16 MiB per buffer (DESIGN.md §5)
constexpr uint32_t WCC_MULTI_MAX_PARTS = 64;   // GB_WCC_MULTI_PARTS is clamped to [1, 64] parts per device

// One part of a one-shot WCC (csr_split.h): the edges [e_begin, e_end) stream through the ring of the part's
// feed in chunks of C edges (chunk k is [e_begin + kC, min(e_begin + (k + 1)C, e_end)), whatever rows it cuts)
// and are linked on the part's link stream into its own forest parent[n], which the other parts read when
// there are several.
struct WccPart {
  WccPartRange range{};
  uint64_t C = 4, K = 0;  // chunk size in edges, chunks
  unsigned int nbad[2] = {0, 0};
  CsrFeed feed;  // the offsets and the ring; destroyed last
  cudaStream_t link = nullptr;
  cudaEvent_t forest_done = nullptr;  // recorded behind the part's finished forest, for the part that merges it
  PeerBuf forest;  // parent[n]
  DevBuf<unsigned int> bad;  // [0] rows whose offsets decrease, [1] targets >= n
  uint64_t e0(uint64_t k) const { return range.e_begin + k * C; }
  uint64_t len(uint64_t k) const { return std::min<uint64_t>(C, range.e_end - e0(k)); }
  ~WccPart() {
    if (feed.dev >= 0) cudaSetDevice(feed.dev);  // the members are released on the part's device
    if (forest_done) cudaEventDestroy(forest_done);
    if (link) cudaStreamDestroy(link);
  }
};

// Every part's link stream drains before any part goes: a merge reads its partner's parent[].
struct WccParts {
  std::vector<std::unique_ptr<WccPart>> v;
  ~WccParts() {
    for (auto& q : v)
      if (q->link) cudaStreamSynchronize(q->link);
  }
};

// Union of every out-edge (wcc_baseline), linked chunk by chunk as the targets land: union-find does not
// depend on the order of the links, and hooking the higher root under the lower keeps parent[x] <= x, so
// after the final compress every label is the minimum node id of its component, as gb_wcc gives.  The
// finds halve the paths they walk, so no compress is needed between chunks (DESIGN.md §5).
// The edges are cut into devs.size() * per_dev parts (wcc_split), part p on devs[p / per_dev], each with
// its own streams, ring and forest.  One part is gb_wcc_csr_u32.  With more, the forests merge in
// ceil(log2 P) tree rounds: in round s = 1, 2, 4, ... part p (p mod 2s == 0) links the forest of part p + s
// into its own through a peer pointer and compresses, and part 0 ends with the union of all edges.
static gb_status wcc_csr_parts(const std::vector<int>& devs, uint32_t per_dev, uint32_t n, const uint32_t* off,
                               const uint32_t* tgt, uint32_t* comp) {
  GB_TRY(require_host_csr(n, off, tgt, ""));
  const uint32_t P = (uint32_t)devs.size() * per_dev;
  const std::vector<WccPartRange> split = wcc_split(off, n, P);
  DeviceGuard guard(devs[0]);
  // C: a multiple of 4 edges (chunk starts stay 16-byte aligned for the uint4 loads), no more than a part needs
  const uint64_t C = std::min<uint64_t>(std::max<uint64_t>(env_u64("GB_WCC_FEED_EDGES", WCC_FEED_EDGES), 4), 1u << 28);
  WccParts parts;
  // every part's offsets and first copies are enqueued before the host waits for any check: all buses stay busy
  for (uint32_t p = 0; p < P; ++p) {
    parts.v.emplace_back(new (std::nothrow) WccPart());
    GB_REQUIRE(parts.v.back() != nullptr, "host allocation failed");
    WccPart& q = *parts.v.back();
    q.range = split[p];
    const uint64_t len = q.range.e_end - q.range.e_begin;
    q.C = std::min<uint64_t>(C, (len + 3)) & ~3ull;
    if (q.C == 0) q.C = 4;
    q.K = (len + q.C - 1) / q.C;
    GB_TRY(q.feed.open(devs[p / per_dev], q.range.r_begin, q.range.r_end, false));
    GB_CUDA(cudaStreamCreateWithFlags(&q.link, cudaStreamNonBlocking));
    GB_CUDA(cudaEventCreateWithFlags(&q.forest_done, cudaEventDisableTiming));
    GB_TRY(q.forest.alloc(n, P > 1));
    GB_TRY(q.bad.alloc(2));
    const uint32_t R = (uint32_t)std::min<uint64_t>(WCC_FEED_RING, q.K);
    GB_TRY(q.feed.open_ring(R, q.C));
    GB_TRY(q.feed.send_offsets(off));
    for (uint32_t k = 0; k < R; ++k) GB_TRY(q.feed.send(k, tgt, q.e0(k), q.len(k)));
  }
  // offsets: monotone, checked before anything indexes with them.  The slices tile [0, n], so the rows each
  // part checks cover every row once, whatever the host array holds
  for (auto& qp : parts.v) {
    WccPart& q = *qp;
    GB_CUDA(cudaSetDevice(q.feed.dev));
    GB_CUDA(cudaMemsetAsync(q.bad.p, 0, 8, q.link));
    GB_TRY(q.feed.check_monotone(q.link, q.range.check_begin, q.range.r_end, q.bad.p));
    GB_CUDA(cudaMemcpyAsync(q.nbad, q.bad.p, 4, cudaMemcpyDeviceToHost, q.link));
  }
  unsigned int nbad = 0;
  for (auto& q : parts.v) {
    GB_CUDA(cudaStreamSynchronize(q->link));
    nbad += q->nbad[0];
  }
  GB_TRY(require_monotone("", nbad));
  const unsigned blk = 256;
  const unsigned grid = grid_for(n, blk);
  uint64_t chunks = 0;
  for (auto& q : parts.v) {
    GB_CUDA(cudaSetDevice(q->feed.dev));
    k_cc_init<<<grid, blk, 0, q->link>>>(q->forest.p, n);
    chunks = std::max(chunks, q->K);
  }
  for (uint64_t k = 0; k < chunks; ++k) {
    for (auto& qp : parts.v) {
      WccPart& q = *qp;
      if (k >= q.K) continue;
      GB_CUDA(cudaSetDevice(q.feed.dev));
      const uint64_t R = q.feed.ring.size();
      if (k >= R) GB_TRY(q.feed.send(k, tgt, q.e0(k), q.len(k)));
      GB_CUDA(cudaStreamWaitEvent(q.link, q.feed.landed[k % R], 0));
      k_cc_link_edges<<<grid_for(q.len(k), LINK_TILE * (blk / 32)), blk, 0, q.link>>>(
          q.feed.off.p, q.range.r_end - q.range.r_begin, q.range.r_begin, q.feed.ring[k % R].p, (uint32_t)q.e0(k),
          (uint32_t)q.len(k), n, q.forest.p, q.bad.p + 1);
      GB_CUDA(cudaEventRecord(q.feed.freed[k % R], q.link));
    }
  }
  for (auto& q : parts.v) {
    GB_CUDA(cudaSetDevice(q->feed.dev));
    k_cc_compress<<<grid, blk, 0, q->link>>>(q->forest.p, n);
  }
  // a partner p + s never merges again after round s, so its forest is final when its event is recorded
  for (uint32_t s = 1; s < P; s *= 2) {
    for (uint32_t p = 0; p + s < P; p += 2 * s) {
      WccPart &a = *parts.v[p], &b = *parts.v[p + s];
      GB_CUDA(cudaSetDevice(b.feed.dev));
      GB_CUDA(cudaEventRecord(b.forest_done, b.link));
      GB_CUDA(cudaSetDevice(a.feed.dev));
      GB_CUDA(cudaStreamWaitEvent(a.link, b.forest_done, 0));
      k_cc_merge_halving<<<grid, blk, 0, a.link>>>(a.forest.p, b.forest.p, n);
      k_cc_compress<<<grid, blk, 0, a.link>>>(a.forest.p, n);
    }
  }
  GB_CUDA(cudaGetLastError());
  for (auto& q : parts.v) {
    GB_CUDA(cudaSetDevice(q->feed.dev));
    GB_CUDA(cudaMemcpyAsync(q->nbad + 1, q->bad.p + 1, 4, cudaMemcpyDeviceToHost, q->link));
  }
  nbad = 0;
  for (auto& q : parts.v) {
    GB_CUDA(cudaStreamSynchronize(q->link));
    nbad += q->nbad[1];
  }
  GB_TRY(require_ids("", nbad, n));
  WccPart& root = *parts.v[0];
  GB_CUDA(cudaSetDevice(root.feed.dev));
  GB_CUDA(cudaMemcpyAsync(comp, root.forest.p, (size_t)n * 4, cudaMemcpyDeviceToHost, root.link));
  GB_CUDA(cudaStreamSynchronize(root.link));
  return GB_OK;
}

}  // namespace gb

extern "C" {
gb_status gb_wcc(const gb_graph* graph, const gb_wcc_config* config, uint32_t* components) {
  GB_REQUIRE(components != nullptr, "components is NULL");
  return gb::wcc_impl(graph, config, nullptr, components);
}
gb_status gb_wcc_device(const gb_graph* graph, const gb_wcc_config* config, uint32_t* d_components) {
  GB_REQUIRE(d_components != nullptr, "d_components is NULL");
  return gb::wcc_impl(graph, config, d_components, nullptr);
}
gb_status gb_wcc_csr_u32(int device, uint32_t node_count, const uint32_t* offsets, const uint32_t* targets,
                         const gb_wcc_config* config, uint32_t* components) {
  GB_REQUIRE(components != nullptr, "components is NULL");
  GB_REQUIRE(config != nullptr, "config is NULL");  // chunk_size / neighbor_rounds / sampling_size: labels unchanged
  GB_REQUIRE(node_count > 0, "node_count must be > 0");
  GB_REQUIRE(offsets != nullptr, "offsets is NULL");
  GB_TRY(gb::require_device(device));
  return gb::wcc_csr_parts({device}, 1, node_count, offsets, targets, components);
}
gb_status gb_wcc_csr_multi_u32(gb_comm* comm, uint32_t node_count, const uint32_t* offsets,
                               const uint32_t* targets, const gb_wcc_config* config, uint32_t* components) {
  GB_REQUIRE(comm != nullptr, "comm is NULL");
  GB_REQUIRE(components != nullptr, "components is NULL");
  GB_REQUIRE(config != nullptr, "config is NULL");  // chunk_size / neighbor_rounds / sampling_size: labels unchanged
  GB_REQUIRE(node_count > 0, "node_count must be > 0");
  GB_REQUIRE(offsets != nullptr, "offsets is NULL");
  const uint64_t per_dev = gb::env_u64("GB_WCC_MULTI_PARTS", 1);
  const uint32_t v = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(per_dev, 1), gb::WCC_MULTI_MAX_PARTS);
  return gb::wcc_csr_parts(gb::comm_devices(comm), v, node_count, offsets, targets, components);
}

// ---- multi-GPU WCC: the phases of wcc() (wcc.rs:158-183) over one rank's vertex range ----------------
gb_status gb_wcc_shard_phase(const gb_graph* g, const gb_wcc_config* cfg, uint32_t phase, uint32_t vertex_begin,
                             uint32_t vertex_end, uint32_t skip_label, int use_skip, uint32_t* d_parent,
                             const uint32_t* d_other, void* cuda_stream) {
  GB_REQUIRE(g && cfg && d_parent, "NULL argument");
  if (g->kind != GB_KIND_DIRECTED)
    return gb::fail(GB_ERR_UNSUPPORTED, "wcc needs a directed graph (wcc.rs:130: DirectedNeighbors)");
  GB_REQUIRE(vertex_begin <= vertex_end && vertex_end <= g->n, "bad vertex range [%u, %u)", vertex_begin, vertex_end);
  GB_REQUIRE(g->out.len == 0 || g->out.tgt.p != nullptr, "this handle holds no out targets (page-rank-only twin)");
  gb::DeviceGuard guard(g->device);
  cudaStream_t s = (cudaStream_t)cuda_stream;
  const uint32_t n = g->n, span = vertex_end - vertex_begin;
  const unsigned blk = 256;
  const uint32_t rounds = (uint32_t)std::min<uint64_t>(cfg->neighbor_rounds, 0xFFFFFFFFull);
  switch (phase) {
    case GB_WCC_INIT:
      gb::k_cc_init<<<gb::grid_for(n, blk), blk, 0, s>>>(d_parent, n);
      break;
    case GB_WCC_SAMPLE:  // sample_subgraph over the rank's vertices
      if (rounds && span)
        gb::k_cc_sample<<<gb::grid_for(span, blk), blk, 0, s>>>(g->out.off.p, g->out.tgt.p, vertex_begin, vertex_end,
                                                               rounds, d_parent);
      break;
    case GB_WCC_COMPRESS:
      gb::k_cc_compress<<<gb::grid_for(n, blk), blk, 0, s>>>(d_parent, n);
      break;
    case GB_WCC_MERGE:  // union with another rank's forest
      GB_REQUIRE(d_other != nullptr, "d_other is NULL");
      gb::k_cc_merge<<<gb::grid_for(n, blk), blk, 0, s>>>(d_parent, d_other, n);
      break;
    case GB_WCC_LINK_REMAINING:  // link_remaining over the rank's vertices, skipping the GLOBAL giant component
      if (span)
        gb::k_cc_link_remaining<<<gb::grid_for((uint64_t)span, blk), blk, 0, s>>>(
            g->out.off.p, g->out.tgt.p, g->in.off.p, g->in.tgt.p, vertex_begin, vertex_end, rounds, skip_label,
            use_skip, d_parent);
      break;
    default:
      return gb::fail(GB_ERR_INVALID, "unknown wcc shard phase %u", phase);
  }
  GB_CUDA(cudaGetLastError());
  return GB_OK;
}

gb_status gb_wcc_sample_label(const gb_graph* g, const gb_wcc_config* cfg, const uint32_t* d_parent,
                              uint32_t* label, int* found, void* cuda_stream) {
  GB_REQUIRE(g && cfg && d_parent && label && found, "NULL argument");
  gb::DeviceGuard guard(g->device);
  return gb::most_frequent_label((cudaStream_t)cuda_stream, d_parent, g->n, cfg->sampling_size, label, found);
}
}
