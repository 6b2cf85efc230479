// pr_csr.cu — PageRank from a host CSR: the part pipeline that turns a host in-CSR and its out-offsets into the
// layouts of one or several ranks (pr_csr_plans; the stages are described there and in DESIGN.md §4.1c), and the
// entry points that need nothing else.  The pipeline takes a device list, not a communicator:
// gb_page_rank_csr_u32 is its one-device, one-rank case, gb_pr_shards_csr_u32 hands its plans out as shards of the
// sweep API (pagerank.cu), and gb_page_rank_csr_multi_u32 (multi.cu) sweeps them over a communicator's buffers.
#include <algorithm>
#include <vector>

#include <cub/cub.cuh>

#include "pr_plan.cuh"

namespace gb {

// Rank r's in-degree of every original row, 0 for the rows another rank owns (the deal of 32-row slices of the
// internal order over U ranks); entry n is 0, so that an exclusive scan gives the local offsets
__global__ void k_pr_owned_deg(const uint32_t* __restrict__ in_off, const uint32_t* __restrict__ new_id, uint32_t n,
                               uint32_t U, uint32_t r, uint32_t* __restrict__ deg) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v <= n; v += gridDim.x * blockDim.x)
    deg[v] = v < n && (new_id[v] >> 5) % U == r ? in_off[v + 1] - in_off[v] : 0u;
}

constexpr uint32_t GATHER_ILP = 8;  // 32-entry loads in flight per warp while it copies one row
// One landed chunk of one part, rows [v0, v1) of the original order: a warp takes 32 consecutive rows, ballots
// those rank r owns and copies each with the whole warp, 32 entries per step, from the part's targets (a peer
// pointer when the part lives on another device; part_tgt[0] is edge part_e0) to loc_tgt + loc_off[v].  Every
// copied target is checked against n; a warp adds its count of bad ones to *bad once.
__global__ void __launch_bounds__(256) k_pr_gather_rows(const uint32_t* __restrict__ in_off,
                                                        const uint32_t* __restrict__ part_tgt, uint64_t part_e0,
                                                        uint32_t v0, uint32_t v1, const uint32_t* __restrict__ new_id,
                                                        uint32_t U, uint32_t r, const uint32_t* __restrict__ loc_off,
                                                        uint32_t* __restrict__ loc_tgt, uint32_t n,
                                                        unsigned int* __restrict__ bad) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  uint32_t nbad = 0;
  for (uint64_t base = (uint64_t)v0 + 32ull * warp; base < v1; base += 32ull * nwarps) {
    const uint64_t v = base + lane;
    uint32_t b0 = 0, d = 0, dst = 0;
    if (v < v1 && (new_id[v] >> 5) % U == r) {
      b0 = in_off[v];
      d = in_off[v + 1] - b0;
      dst = loc_off[v];
    }
    uint32_t todo = __ballot_sync(0xFFFFFFFFu, d != 0);
    while (todo) {
      const int src_lane = __ffs(todo) - 1;
      todo &= todo - 1;
      const uint32_t rb = __shfl_sync(0xFFFFFFFFu, b0, src_lane);
      const uint32_t rd = __shfl_sync(0xFFFFFFFFu, d, src_lane);
      const uint32_t rdst = __shfl_sync(0xFFFFFFFFu, dst, src_lane);
      const uint32_t* __restrict__ from = part_tgt + (rb - part_e0);
      uint32_t* __restrict__ to = loc_tgt + rdst;
      for (uint64_t i = lane; i < rd; i += 32 * GATHER_ILP) {
        uint32_t t[GATHER_ILP];
#pragma unroll
        for (uint32_t u = 0; u < GATHER_ILP; ++u) t[u] = i + 32 * u < rd ? from[i + 32 * u] : 0u;
#pragma unroll
        for (uint32_t u = 0; u < GATHER_ILP; ++u)
          if (i + 32 * u < rd) {
            nbad += t[u] >= n;
            to[i + 32 * u] = t[u];
          }
      }
    }
  }
  nbad = __reduce_add_sync(0xFFFFFFFFu, nbad);
  if (lane == 0 && nbad) atomicAdd(bad, nbad);
}

constexpr uint64_t PR_PART_CHUNK_EDGES = 1u << 23;  // 32 MiB of targets per chunk (GB_PR_PART_CHUNK_EDGES)

// One rank r on device dev: the full offsets gathered from the parts, the order stage of its layout, and the
// compact local in-CSR of the rows it owns (loc_off by original id, loc_tgt in CSR order).  A lone rank needs
// neither the gathered offsets nor the local CSR: its part is all of them.
struct PrCsrRank {
  int dev = -1;
  cudaStream_t s = nullptr;
  PeerBuf in_off, out_off;     // [n + 1] each
  LayoutBuild* build = nullptr;
  PrPlan* plan = nullptr;      // the finished layout, until the caller takes it
  DevBuf<uint32_t> loc_off, loc_tgt;
  uint64_t entries = 0;        // loc_off[n]
  DevBuf<unsigned int> bad;    // [0] in rows whose offsets decrease, [1] out rows, [2] targets >= n
  unsigned int h_bad[3] = {0, 0, 0};
  ~PrCsrRank() {
    if (dev < 0) return;
    cudaSetDevice(dev);
    if (s) cudaStreamSynchronize(s);
    layout_free(build);
    free_pr_plan(plan);
    loc_tgt.release();
    loc_off.release();
    bad.release();
    out_off.release();
    in_off.release();
    if (s) cudaStreamDestroy(s);
  }
};

gb_status check_pr_host_csr(uint32_t n, const uint32_t* in_off, const uint32_t* in_tgt, const uint32_t* out_off) {
  GB_REQUIRE(n > 0, "node_count must be > 0");
  GB_TRY(require_pr_node_count(n));  // before any upload or per-rank copy of the offsets
  GB_REQUIRE(in_off && out_off, "offset arrays are NULL");
  GB_REQUIRE(in_off[n] == out_off[n], "in and out offsets disagree on the edge count");
  GB_TRY(require_host_csr(n, in_off, in_tgt, "in"));
  return require_host_csr(n, out_off, nullptr, "out", true);
}

gb_status pr_csr_plans(const std::vector<int>& devs, uint32_t V, uint32_t n, const uint32_t* in_off,
                       const uint32_t* in_tgt, const uint32_t* out_off, uint64_t chunk_edges,
                       std::vector<PrPlan*>* plans) {
  const uint64_t m = in_off[n];
  const uint32_t U = (uint32_t)devs.size() * V;
  const bool peers = U > 1;
  const std::vector<PrPart> split = pr_split(in_off, n, U, chunk_edges);
  DeviceGuard guard(devs[0]);
  // declared after the parts, the ranks go first on any return, and each drains its stream as it goes: the
  // gathers and a lone rank's layout read the parts
  std::vector<std::unique_ptr<CsrFeed>> parts;
  std::vector<std::unique_ptr<PrCsrRank>> ranks;
  // 1. every part's in and out offsets, then its targets chunk by chunk, round robin over the parts: the copies go
  // out before the host waits for any check, so every bus is busy from the start
  uint32_t max_chunks = 0;
  for (uint32_t u = 0; u < U; ++u) {
    parts.emplace_back(new (std::nothrow) CsrFeed());
    GB_REQUIRE(parts.back() != nullptr, "host allocation failed");
    CsrFeed& q = *parts.back();
    GB_TRY(q.open(devs[u / V], split[u].r_begin, split[u].r_end, peers, true));
    GB_TRY(q.resident(split[u].e_begin, split[u].e_end, split[u].chunks.count(), peers));
    GB_TRY(q.send_offsets(in_off, out_off));
    max_chunks = std::max(max_chunks, split[u].chunks.count());
  }
  for (uint32_t k = 0; k < max_chunks; ++k)
    for (uint32_t u = 0; u < U; ++u) {
      const CsrChunks& ch = split[u].chunks;
      if (k >= ch.count()) continue;
      GB_CUDA(cudaSetDevice(parts[u]->dev));
      GB_TRY(parts[u]->send(k, in_tgt, ch.edge[k], ch.edge[k + 1] - ch.edge[k]));
    }
  // 2. rank u checks part u's rows (the slices tile [0, n]: every row once, whatever the host arrays hold), and
  // with several ranks every rank assembles the full offsets from the parts
  for (uint32_t r = 0; r < U; ++r) {
    ranks.emplace_back(new (std::nothrow) PrCsrRank());
    GB_REQUIRE(ranks.back() != nullptr, "host allocation failed");
    PrCsrRank& k = *ranks.back();
    k.dev = devs[r / V];
    GB_CUDA(cudaSetDevice(k.dev));
    GB_CUDA(cudaStreamCreateWithFlags(&k.s, cudaStreamNonBlocking));
    GB_TRY(k.bad.alloc(3));
    GB_CUDA(cudaMemsetAsync(k.bad.p, 0, 12, k.s));
    GB_TRY(parts[r]->check_monotone(k.s, split[r].r_begin, split[r].r_end, k.bad.p));
    GB_CUDA(cudaMemcpyAsync(k.h_bad, k.bad.p, 8, cudaMemcpyDeviceToHost, k.s));
    if (!peers) continue;
    GB_TRY(k.in_off.alloc((size_t)n + 1, peers));
    GB_TRY(k.out_off.alloc((size_t)n + 1, peers));
    for (uint32_t u = 0; u < U; ++u) {
      const CsrFeed& q = *parts[u];
      const size_t count = (size_t)(q.r_end - q.r_begin) + (u + 1 == U ? 1 : 0);
      if (!count) continue;
      GB_CUDA(cudaStreamWaitEvent(k.s, q.offsets_in, 0));
      GB_CUDA(cudaMemcpyPeerAsync(k.in_off.p + q.r_begin, k.dev, q.off.p, q.dev, count * 4, k.s));
      GB_CUDA(cudaMemcpyPeerAsync(k.out_off.p + q.r_begin, k.dev, q.off2.p, q.dev, count * 4, k.s));
    }
  }
  unsigned int nbad[2] = {0, 0};
  for (auto& k : ranks) {
    GB_CUDA(cudaSetDevice(k->dev));
    GB_CUDA(cudaStreamSynchronize(k->s));
    nbad[0] += k->h_bad[0];
    nbad[1] += k->h_bad[1];
  }
  GB_TRY(require_monotone("in", nbad[0]));
  GB_TRY(require_monotone("out", nbad[1]));
  // 3. order stage.  A lone rank owns every row: its part is its in-CSR, whose chunks the layout build checks
  // and classifies as they land.  Otherwise the local offsets, and the gathers of every chunk as it lands.
  for (uint32_t r = 0; r < U; ++r) {
    PrCsrRank& k = *ranks[r];
    GB_CUDA(cudaSetDevice(k.dev));
    PrSource src;
    src.device = k.dev;
    src.stream = k.s;
    src.n = n;
    src.m = m;
    src.in_off = peers ? k.in_off.p : parts[0]->off.p;
    src.out_off = peers ? k.out_off.p : parts[0]->off2.p;
    src.feed = peers ? nullptr : parts[0].get();
    src.chunks = peers ? nullptr : &split[0].chunks;
    GB_TRY(layout_begin(src, PrDeal(U, r), &k.build));
    if (!peers) {
      LayoutBuild* b = k.build;
      k.build = nullptr;
      GB_TRY(layout_end(b, src.in_off, parts[0]->tgt.p, m, &k.plan));
      continue;
    }
    const uint32_t* new_id = layout_new_id(k.build);
    {
      DevBufStreamScope scope(k.s);  // the copy streams may still be busy: release waits for this stream only
      GB_TRY(k.loc_off.alloc((size_t)n + 1));
      k_pr_owned_deg<<<grid_for((uint64_t)n + 1, 256), 256, 0, k.s>>>(k.in_off.p, new_id, n, U, r, k.loc_off.p);
      DevBuf<uint8_t> tmp;
      GB_TRY(exclusive_sum(k.s, tmp, k.loc_off.p, (int)(n + 1)));
      uint32_t total = 0;
      GB_CUDA(cudaMemcpyAsync(&total, k.loc_off.p + n, 4, cudaMemcpyDeviceToHost, k.s));
      GB_CUDA(cudaStreamSynchronize(k.s));
      k.entries = total;
      GB_TRY(k.loc_tgt.alloc(std::max<uint64_t>(k.entries, 1)));
    }
    for (uint32_t c = 0; c < max_chunks; ++c)
      for (uint32_t u = 0; u < U; ++u) {
        const CsrChunks& ch = split[u].chunks;
        if (c >= ch.count()) continue;
        const uint32_t v0 = ch.row[c], v1 = ch.row[c + 1];
        if (v1 == v0) continue;
        GB_CUDA(cudaStreamWaitEvent(k.s, parts[u]->landed[c], 0));
        k_pr_gather_rows<<<grid_for((uint64_t)(v1 - v0), 256), 256, 0, k.s>>>(
            k.in_off.p, parts[u]->tgt.p, split[u].e_begin, v0, v1, new_id, U, r, k.loc_off.p, k.loc_tgt.p, n,
            k.bad.p + 2);
      }
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaMemcpyAsync(k.h_bad + 2, k.bad.p + 2, 4, cudaMemcpyDeviceToHost, k.s));
  }
  if (peers) {
    unsigned int nbad_tgt = 0;
    for (auto& k : ranks) {
      GB_CUDA(cudaSetDevice(k->dev));
      GB_CUDA(cudaStreamSynchronize(k->s));
      nbad_tgt += k->h_bad[2];
    }
    GB_TRY(require_ids("in", nbad_tgt, n));
    // 4. every rank has gathered: the parts and the full offsets go (the order stage has read the degrees), and
    // each rank builds its layout from its local CSR, which goes too
    parts.clear();
    for (auto& k : ranks) {
      GB_CUDA(cudaSetDevice(k->dev));
      k->in_off.release();
      k->out_off.release();
    }
    for (auto& k : ranks) {
      GB_CUDA(cudaSetDevice(k->dev));
      LayoutBuild* b = k->build;
      k->build = nullptr;
      GB_TRY(layout_end(b, k->loc_off.p, k->loc_tgt.p, k->entries, &k->plan));
      DevBufStreamScope scope(k->s);
      k->loc_tgt.release();
      k->loc_off.release();
    }
  }
  plans->clear();
  for (auto& k : ranks) {
    plans->push_back(k->plan);
    k->plan = nullptr;
  }
  return GB_OK;
}

gb_status pr_csr_shards(const std::vector<int>& devs, uint32_t V, uint32_t n, const uint32_t* in_off,
                        const uint32_t* in_tgt, const uint32_t* out_off, std::vector<gb_pr_shard*>& shards) {
  GB_TRY(check_pr_host_csr(n, in_off, in_tgt, out_off));
  const uint64_t chunk_edges = std::max<uint64_t>((uint32_t)env_u64("GB_PR_PART_CHUNK_EDGES", PR_PART_CHUNK_EDGES), 1);
  std::vector<PrPlan*> plans;
  GB_TRY(pr_csr_plans(devs, V, n, in_off, in_tgt, out_off, chunk_edges, &plans));
  gb_status st = GB_OK;
  for (size_t r = 0; r < plans.size(); ++r) {  // shard_from_plan takes its plan, whatever it returns
    if (st == GB_OK) {
      st = shard_from_plan(devs[r / V], plans[r], &shards[r]);
    } else {
      DeviceGuard guard(devs[r / V]);
      free_pr_plan(plans[r]);
    }
  }
  return st;
}

// A resident digraph of a host CSR that passed check_pr_host_csr: the in-CSR, and the out-offsets for the
// out-degrees
static gb_status page_rank_digraph(int device, uint32_t n, const uint32_t* in_off, const uint32_t* in_tgt,
                                   const uint32_t* out_off, GraphPtr* g) {
  GB_TRY(new_graph(device, GB_KIND_DIRECTED, n, g));
  GB_TRY(upload_host_csr((*g)->stream, n, in_off, in_tgt, nullptr, &(*g)->in, "in"));
  return upload_host_csr((*g)->stream, n, out_off, nullptr, nullptr, &(*g)->out, "out", true);
}

}  // namespace gb

extern "C" {

gb_status gb_pr_shards_csr_u32(gb_comm* c, uint32_t ranks_per_device, uint32_t n, const uint32_t* in_off,
                               const uint32_t* in_tgt, const uint32_t* out_off, gb_pr_shard** shards) {
  GB_REQUIRE(c != nullptr, "comm is NULL");
  GB_REQUIRE(shards != nullptr, "shards is NULL");
  GB_REQUIRE(ranks_per_device >= 1, "ranks_per_device must be >= 1");
  const std::vector<int>& devs = gb::comm_devices(c);
  const uint64_t U = (uint64_t)devs.size() * ranks_per_device;
  GB_REQUIRE(U <= 8, "%zu devices x %u ranks per device: at most 8 ranks", devs.size(), ranks_per_device);
  gb::ShardSet set((uint32_t)U);
  GB_TRY(gb::pr_csr_shards(devs, ranks_per_device, n, in_off, in_tgt, out_off, set.v));
  for (uint32_t r = 0; r < U; ++r) shards[r] = set.v[r];
  set.v.clear();
  return GB_OK;
}

// One-shot PageRank of a host CSR.  The 4 bytes per edge of the targets dominate the upload, so they are
// streamed, as the one-rank case of the part pipeline (pr_csr_plans): offsets first, then the
// targets in row-aligned chunks on a copy stream, while the rank's stream sorts the degrees, picks the hot
// blocks and classifies every chunk as it lands (layout_classify, pr_layout.cu).  Only the fill pass, the
// sweeps and the copy of the ranks run after the last byte.  EXACT mode and small graphs upload everything
// first.  GB_PR_FEED_CHUNKS (default 16 chunks of ceil(m / 16) edges; 0 = upload everything, then build) and
// GB_PR_FEED_MIN_EDGES (default 2^22) are experiment knobs.
gb_status gb_page_rank_csr_u32(int device, uint32_t n, const uint32_t* in_off, const uint32_t* in_tgt,
                               const uint32_t* out_off, const gb_page_rank_config* config, float* scores,
                               uint64_t* ran_iterations, double* error) {
  GB_REQUIRE(scores != nullptr, "scores is NULL");
  GB_TRY(gb::check_pr_host_csr(n, in_off, in_tgt, out_off));
  const uint64_t m = in_off[n];
  uint32_t chunks = (uint32_t)gb::env_u64("GB_PR_FEED_CHUNKS", 16);
  if (m < (uint32_t)gb::env_u64("GB_PR_FEED_MIN_EDGES", 1u << 22)) chunks = 0;
  // the single-warp EXACT mode (small graphs) reads the CSR directly: nothing to overlap
  if (!config || config->mode == GB_PR_EXACT || (config->mode == GB_PR_AUTO && n <= 16384)) chunks = 0;
  gb::GraphPtr g;
  if (chunks == 0) {
    GB_TRY(gb::page_rank_digraph(device, n, in_off, in_tgt, out_off, &g));
    return gb::page_rank_impl(g.get(), config, nullptr, scores, ran_iterations, error);
  }
  // the graph brings the stream, the timing events and the lock; the sweeps read only the plan
  GB_TRY(gb::new_graph(device, GB_KIND_DIRECTED, n, &g));
  std::vector<gb::PrPlan*> plans;
  GB_TRY(gb::pr_csr_plans({device}, 1, n, in_off, in_tgt, out_off, std::max<uint64_t>((m + chunks - 1) / chunks, 1),
                          &plans));
  g->pr_plan = plans[0];
  return gb::page_rank_impl(g.get(), config, nullptr, scores, ran_iterations, error);
}

gb_status gb_digraph_for_page_rank_u32(int device, uint32_t n, const uint32_t* in_off, const uint32_t* in_tgt,
                                       const uint32_t* out_off, gb_graph** graph) {
  GB_REQUIRE(graph != nullptr, "graph is NULL");
  GB_TRY(gb::check_pr_host_csr(n, in_off, in_tgt, out_off));
  gb::GraphPtr g;
  GB_TRY(gb::page_rank_digraph(device, n, in_off, in_tgt, out_off, &g));
  *graph = g.release();
  return GB_OK;
}

}  // extern "C"
