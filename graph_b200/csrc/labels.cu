// labels.cu — the structures over a node-labelled undirected graph (crates/builder/src/input/dotgraph.rs):
// LabelStats (:220-313), NodeLabelIndex (:430-532) and NeighborLabelFrequencies (:367-427).
//
// Stats and index: the (label, node) pairs are radix sorted by label, stably, so every label's nodes stay in
// ascending order; a run-length encode gives the distinct labels and their frequencies, and the index offsets
// are lower bounds of each label in the sorted labels.
//
// Neighbour-label frequencies gather the label of every CSR entry (2m random 4-byte loads, the access pattern of
// PageRank's gather), sort each row's labels and run-length encode them.  Rows are served by size class:
//   deg <= 32               one warp per row: one label per lane, equal labels found with __match_any_sync and
//                           the distinct ones ranked by a shuffle loop;
//   32 < deg <= 512         one 128-thread CTA per row: cub::BlockRadixSort of 4 labels per thread;
//   512 < deg <= 2048       one 256-thread CTA per row: 8 labels per thread;
//   deg > 2048 (hub rows)   all hub entries at once: keys (hub index << label bits | label) radix sorted over the
//                           whole device and run-length encoded, so one huge row does not fall to one CTA.
// Every class writes its row's pairs at the row's CSR offset (a row holds at most deg pairs) and its pair count;
// an exclusive scan of the counts gives the pair CSR and one copy compacts it.  Nothing depends on scheduling.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "common.cuh"

namespace gb {

constexpr uint32_t NLF_WARP_MAX = 32;
constexpr uint32_t NLF_SMALL_MAX = 512;   // 128 threads x 4 labels
constexpr uint32_t NLF_LARGE_MAX = 2048;  // 256 threads x 8 labels
constexpr unsigned FULL_MASK = 0xFFFFFFFFu;

static int label_bits(uint32_t max_label) { return max_label ? 32 - __builtin_clz(max_label) : 1; }

__global__ void k_max_degree(const uint32_t* __restrict__ off, uint32_t n, unsigned int* __restrict__ mx) {
  uint32_t d = 0;
  for (uint64_t v = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; v < n; v += (uint64_t)gridDim.x * blockDim.x)
    d = max(d, off[v + 1] - off[v]);
  for (int o = 16; o; o >>= 1) d = max(d, __shfl_xor_sync(FULL_MASK, d, o));
  if ((threadIdx.x & 31) == 0) atomicMax(mx, d);
}

// offsets[l] = the first position of label l in the sorted labels, l in [0, count)
__global__ void k_label_offsets(const uint32_t* __restrict__ sorted, uint32_t n, uint64_t count,
                                uint32_t* __restrict__ offsets) {
  for (uint64_t l = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; l < count; l += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
      const uint64_t mid = (lo + hi) / 2;
      if ((uint64_t)sorted[mid] < l) lo = mid + 1;
      else hi = mid;
    }
    offsets[l] = (uint32_t)lo;
  }
}

// rows of at most NLF_WARP_MAX entries, one warp each; the other rows are left to their classes
__global__ void k_nlf_warp(const uint32_t* __restrict__ off, const uint32_t* __restrict__ tgt,
                           const uint32_t* __restrict__ labels, uint32_t n, uint32_t* __restrict__ plab,
                           uint32_t* __restrict__ pcnt, uint32_t* __restrict__ rowcnt) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t v = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; v < n; v += warps) {
    const uint32_t b = off[v], deg = off[v + 1] - b;
    if (deg > NLF_WARP_MAX) continue;
    const bool in = lane < deg;
    const uint32_t x = in ? __ldg(labels + tgt[b + lane]) : 0u;
    const uint32_t valid = __ballot_sync(FULL_MASK, in);
    const uint32_t same = __match_any_sync(FULL_MASK, x) & valid;
    const bool leader = in && (uint32_t)(__ffs(same) - 1) == lane;
    const uint32_t leaders = __ballot_sync(FULL_MASK, leader);
    uint32_t rank = 0;  // distinct labels below x
    for (uint32_t t = leaders; t; t &= t - 1) rank += __shfl_sync(FULL_MASK, x, __ffs(t) - 1) < x;
    if (leader) {
      plab[b + rank] = x;
      pcnt[b + rank] = __popc(same);
    }
    if (lane == 0) rowcnt[v] = __popc(leaders);
  }
}

// one CTA per listed row of at most T * I entries.  The labels are loaded striped (their order does not matter),
// sorted on bits [0, end_bit) into a blocked arrangement, and every run head writes its pair.  The pads are the
// largest key those bits hold, so the first deg sorted keys are the row's labels.
template <int T, int I>
__global__ void __launch_bounds__(T) k_nlf_cta(const uint32_t* __restrict__ rows, uint32_t count,
                                               const uint32_t* __restrict__ off, const uint32_t* __restrict__ tgt,
                                               const uint32_t* __restrict__ labels, int end_bit,
                                               uint32_t* __restrict__ plab, uint32_t* __restrict__ pcnt,
                                               uint32_t* __restrict__ rowcnt) {
  using Sort = cub::BlockRadixSort<uint32_t, T, I>;
  using Heads = cub::BlockDiscontinuity<uint32_t, T>;
  using Scan = cub::BlockScan<uint32_t, T>;
  __shared__ union {
    typename Sort::TempStorage sort;
    typename Heads::TempStorage heads;
    typename Scan::TempStorage scan;
  } tmp;
  __shared__ uint32_t head_pos[T * I + 1];
  const uint32_t pad = end_bit == 32 ? 0xFFFFFFFFu : (1u << end_bit) - 1;
  for (uint32_t r = blockIdx.x; r < count; r += gridDim.x) {
    const uint32_t v = rows[r];
    const uint32_t b = off[v], deg = off[v + 1] - b;
    uint32_t key[I];
#pragma unroll
    for (int k = 0; k < I; ++k) {
      const uint32_t i = k * T + threadIdx.x;
      key[k] = i < deg ? __ldg(labels + tgt[b + i]) : pad;
    }
    __syncthreads();  // the previous row is done with tmp and head_pos
    Sort(tmp.sort).Sort(key, 0, end_bit);
    __syncthreads();
    uint32_t flag[I];
    Heads(tmp.heads).FlagHeads(flag, key, cub::Inequality());
#pragma unroll
    for (int k = 0; k < I; ++k) flag[k] = flag[k] && threadIdx.x * I + k < deg;
    __syncthreads();
    uint32_t run[I], runs;
    Scan(tmp.scan).ExclusiveSum(flag, run, runs);
#pragma unroll
    for (int k = 0; k < I; ++k)
      if (flag[k]) {
        head_pos[run[k]] = threadIdx.x * I + k;
        plab[b + run[k]] = key[k];
      }
    if (threadIdx.x == 0) head_pos[runs] = deg;
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < runs; j += T) pcnt[b + j] = head_pos[j + 1] - head_pos[j];
    if (threadIdx.x == 0) rowcnt[v] = runs;
  }
}

// hub h's entries as keys (h << end_bit | label), at seg[h] onwards
__global__ void k_nlf_hub_keys(const uint32_t* __restrict__ rows, uint32_t hubs, const uint32_t* __restrict__ seg,
                               const uint32_t* __restrict__ off, const uint32_t* __restrict__ tgt,
                               const uint32_t* __restrict__ labels, int end_bit, uint64_t* __restrict__ keys) {
  for (uint32_t h = blockIdx.x; h < hubs; h += gridDim.x) {
    const uint32_t v = rows[h];
    const uint32_t b = off[v], deg = off[v + 1] - b;
    const uint64_t hi = (uint64_t)h << end_bit;
    for (uint32_t i = threadIdx.x; i < deg; i += blockDim.x) keys[seg[h] + i] = hi | __ldg(labels + tgt[b + i]);
  }
}

__global__ void k_hub_degrees(const uint32_t* __restrict__ rows, uint32_t hubs, const uint32_t* __restrict__ off,
                              uint32_t* __restrict__ deg) {
  for (uint32_t h = blockIdx.x * blockDim.x + threadIdx.x; h < hubs; h += gridDim.x * blockDim.x)
    deg[h] = off[rows[h] + 1] - off[rows[h]];
}

// first[h] = the first run of hub h among the sorted unique keys (first[hubs] = runs); the hub's pair count
__global__ void k_nlf_hub_firsts(const uint64_t* __restrict__ unique, const uint32_t* __restrict__ nruns,
                                 const uint32_t* __restrict__ rows, uint32_t hubs, int end_bit,
                                 uint32_t* __restrict__ first) {
  const uint32_t runs = *nruns;
  for (uint32_t h = blockIdx.x * blockDim.x + threadIdx.x; h <= hubs; h += gridDim.x * blockDim.x) {
    const uint64_t want = (uint64_t)h << end_bit;
    uint32_t lo = 0, hi = runs;
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (unique[mid] < want) lo = mid + 1;
      else hi = mid;
    }
    first[h] = lo;
  }
}

__global__ void k_nlf_hub_pairs(const uint64_t* __restrict__ unique, const uint32_t* __restrict__ counts,
                                const uint32_t* __restrict__ nruns, const uint32_t* __restrict__ first,
                                const uint32_t* __restrict__ rows, uint32_t hubs, const uint32_t* __restrict__ off,
                                int end_bit, uint32_t* __restrict__ plab, uint32_t* __restrict__ pcnt,
                                uint32_t* __restrict__ rowcnt) {
  const uint32_t runs = *nruns;
  const uint64_t mask = (1ull << end_bit) - 1;
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < runs; j += stride) {
    const uint32_t h = (uint32_t)(unique[j] >> end_bit);
    const uint32_t v = rows[h];
    plab[off[v] + j - first[h]] = (uint32_t)(unique[j] & mask);
    pcnt[off[v] + j - first[h]] = counts[j];
  }
  for (uint32_t h = blockIdx.x * blockDim.x + threadIdx.x; h < hubs; h += stride) rowcnt[rows[h]] = first[h + 1] - first[h];
}

// one warp per row: its pairs from the row's CSR offset to its pair offset
__global__ void k_nlf_compact(const uint32_t* __restrict__ off, const uint32_t* __restrict__ rowcnt,
                              const uint32_t* __restrict__ pair_off, uint32_t n, const uint32_t* __restrict__ plab,
                              const uint32_t* __restrict__ pcnt, uint32_t* __restrict__ out_lab,
                              uint32_t* __restrict__ out_cnt) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
  for (uint64_t v = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; v < n; v += warps) {
    const uint32_t b = off[v], c = rowcnt[v], o = pair_off[v];
    for (uint32_t k = lane; k < c; k += 32) {
      out_lab[o + k] = plab[b + k];
      out_cnt[o + k] = pcnt[b + k];
    }
  }
}

struct DegreeIn {
  const uint32_t* off;
  uint32_t lo, hi;  // lo < degree <= hi
  __device__ bool operator()(uint32_t v) const {
    const uint32_t d = off[v + 1] - off[v];
    return d > lo && d <= hi;
  }
};

static gb_status require_labeled(const gb_graph* g, const char* what) {
  GB_REQUIRE(g != nullptr, "NULL graph");
  if (g->kind != GB_KIND_UNDIRECTED)
    return fail(GB_ERR_UNSUPPORTED, "%s needs an undirected graph (UndirectedNeighbors + UndirectedDegrees)", what);
  if (!g->labels.p) return fail(GB_ERR_UNSUPPORTED, "%s needs a graph with node values (labels)", what);
  return GB_OK;
}

// The CUDA-event time of a call's device work, from its first kernel to its last (host round trips between them
// included, the copies of the results to the host not), left in g->timing for gb_graph_last_timing.
static gb_status timing_begin(const gb_graph* g) {
  g->timing = gb_timing{};
  GB_CUDA(cudaEventRecord(g->ev_begin, g->stream));
  return GB_OK;
}
static gb_status timing_end(const gb_graph* g, uint64_t launches) {
  GB_CUDA(cudaEventRecord(g->ev_end, g->stream));
  GB_CUDA(cudaEventSynchronize(g->ev_end));
  float ms = 0.0f;
  GB_CUDA(cudaEventElapsedTime(&ms, g->ev_begin, g->ev_end));
  g->timing.total_ms = ms;
  g->timing.kernel_launches = launches;
  return GB_OK;
}

// the largest label, on the host
static gb_status max_label_of(const gb_graph* g, DevBuf<uint8_t>& tmp, uint32_t* max_label) {
  cudaStream_t s = g->stream;
  DevBuf<uint32_t> d_max;
  GB_TRY(d_max.alloc(1));
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceReduce::Max(t, tb, g->labels.p, d_max.p, (int64_t)g->n, s);
  }));
  GB_CUDA(cudaMemcpyAsync(max_label, d_max.p, 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

// the labels sorted ascending, and with them the nodes (stable: each label's nodes ascending)
static gb_status sort_by_label(const gb_graph* g, DevBuf<uint8_t>& tmp, uint32_t max_label, DevBuf<uint32_t>* keys,
                               DevBuf<uint32_t>* nodes) {
  cudaStream_t s = g->stream;
  const uint64_t n = g->n;
  DevBuf<uint32_t> iota;
  GB_TRY(iota.alloc(n));
  GB_TRY(keys->alloc(n));
  GB_TRY(nodes->alloc(n));
  k_iota<<<grid_for(n, 256), 256, 0, s>>>(iota.p, n);
  GB_CUDA(cudaGetLastError());
  const int bits = label_bits(max_label);
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceRadixSort::SortPairs(t, tb, g->labels.p, keys->p, iota.p, nodes->p, (int64_t)n, 0, bits, s);
  }));
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

static gb_status label_stats(const gb_graph* g, gb_label_stats_info* st, uint32_t* labels, uint64_t* counts) {
  GB_TRY(require_labeled(g, "LabelStats"));
  GB_REQUIRE(st != nullptr, "stats is NULL");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  cudaStream_t s = g->stream;
  DevBufStreamScope scope(s);
  GB_TRY(timing_begin(g));
  DevBuf<uint8_t> tmp;
  uint32_t max_label = 0;
  GB_TRY(max_label_of(g, tmp, &max_label));
  DevBuf<uint32_t> keys, nodes, uniq, freq, small;
  GB_TRY(sort_by_label(g, tmp, max_label, &keys, &nodes));
  const uint64_t n = g->n;
  GB_TRY(uniq.alloc(n));
  GB_TRY(freq.alloc(n));
  GB_TRY(small.alloc(3));  // [0] runs, [1] max frequency, [2] max degree
  GB_CUDA(cudaMemsetAsync(small.p, 0, 12, s));
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceRunLengthEncode::Encode(t, tb, keys.p, uniq.p, freq.p, small.p, (int64_t)n, s);
  }));
  uint32_t runs = 0;
  GB_CUDA(cudaMemcpyAsync(&runs, small.p, 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceReduce::Max(t, tb, freq.p, small.p + 1, (int64_t)runs, s);
  }));
  k_max_degree<<<grid_for(n, 256), 256, 0, s>>>(g->out.off.p, g->n, small.p + 2);
  GB_CUDA(cudaGetLastError());
  GB_TRY(timing_end(g, 6));  // max, iota, sort, run-length encode, max, max degree
  uint32_t h[3] = {0, 0, 0};
  GB_CUDA(cudaMemcpyAsync(h, small.p, 12, cudaMemcpyDeviceToHost, s));
  std::vector<uint32_t> hf;
  if (counts) {
    hf.resize(runs);
    GB_CUDA(cudaMemcpyAsync(hf.data(), freq.p, 4ull * runs, cudaMemcpyDeviceToHost, s));
  }
  if (labels) GB_CUDA(cudaMemcpyAsync(labels, uniq.p, 4ull * runs, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  for (uint32_t i = 0; counts && i < runs; ++i) counts[i] = hf[i];
  st->max_degree = h[2];
  st->max_label = max_label;
  st->label_count = runs;
  st->max_label_frequency = h[1];
  return GB_OK;
}

static gb_status node_label_index(const gb_graph* g, uint32_t* max_label_out, uint32_t* offsets,
                                  uint32_t* nodes_out) {
  GB_TRY(require_labeled(g, "NodeLabelIndex"));
  GB_REQUIRE((offsets == nullptr) == (nodes_out == nullptr), "offsets and nodes must both be given, or neither");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  cudaStream_t s = g->stream;
  DevBufStreamScope scope(s);
  GB_TRY(timing_begin(g));
  DevBuf<uint8_t> tmp;
  uint32_t max_label = 0;
  GB_TRY(max_label_of(g, tmp, &max_label));
  if (max_label_out) *max_label_out = max_label;
  if (!offsets) return timing_end(g, 1);
  DevBuf<uint32_t> keys, nodes, off;
  GB_TRY(sort_by_label(g, tmp, max_label, &keys, &nodes));
  const uint64_t rows = (uint64_t)max_label + 2;  // max_label + 1 rows
  GB_TRY(off.alloc(rows));
  k_label_offsets<<<grid_for(rows, 256), 256, 0, s>>>(keys.p, g->n, rows, off.p);
  GB_CUDA(cudaGetLastError());
  GB_TRY(timing_end(g, 4));  // max, iota, sort, offsets
  GB_CUDA(cudaMemcpyAsync(offsets, off.p, rows * 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaMemcpyAsync(nodes_out, nodes.p, (size_t)g->n * 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

// the rows of one size class, listed on the device; returns their number
static gb_status select_rows(const gb_graph* g, DevBuf<uint8_t>& tmp, uint32_t lo, uint32_t hi, uint32_t* rows,
                             uint32_t* d_count, uint32_t* count) {
  cudaStream_t s = g->stream;
  const DegreeIn pred{g->out.off.p, lo, hi};
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceSelect::If(t, tb, thrust::counting_iterator<uint32_t>(0), rows, d_count, (int64_t)g->n, pred, s);
  }));
  GB_CUDA(cudaMemcpyAsync(count, d_count, 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

static gb_status neighbor_label_frequencies(const gb_graph* g, uint32_t* offsets, uint32_t* labels_out,
                                            uint32_t* counts_out) {
  GB_TRY(require_labeled(g, "NeighborLabelFrequencies"));
  GB_REQUIRE(offsets && (g->out.len == 0 || (labels_out && counts_out)), "NULL argument");
  GB_REQUIRE(g->out.len == 0 || g->out.tgt.p != nullptr, "this handle holds no targets");
  DeviceGuard guard(g->device);
  std::lock_guard<std::mutex> lock(g->mu);
  cudaStream_t s = g->stream;
  DevBufStreamScope scope(s);
  const uint32_t n = g->n;
  const uint64_t E = g->out.len;
  const uint32_t* off = g->out.off.p;
  const uint32_t* tgt = g->out.tgt.p;
  const uint32_t* lab = g->labels.p;
  GB_TRY(timing_begin(g));
  DevBuf<uint8_t> tmp;
  uint32_t max_label = 0;
  GB_TRY(max_label_of(g, tmp, &max_label));
  const int end_bit = label_bits(max_label);
  DevBuf<uint32_t> plab, pcnt, rowcnt, pair_off, rows, d_count;
  GB_TRY(plab.alloc(E));
  GB_TRY(pcnt.alloc(E));
  GB_TRY(rowcnt.alloc((uint64_t)n + 1));
  GB_TRY(pair_off.alloc((uint64_t)n + 1));
  GB_TRY(rows.alloc(n));
  GB_TRY(d_count.alloc(1));
  GB_CUDA(cudaMemsetAsync(rowcnt.p + n, 0, 4, s));
  k_nlf_warp<<<grid_for((uint64_t)n * 32, 256), 256, 0, s>>>(off, tgt, lab, n, plab.p, pcnt.p, rowcnt.p);
  GB_CUDA(cudaGetLastError());
  uint64_t launches = 2;  // the max label and the warp rows

  uint32_t cnt = 0;
  GB_TRY(select_rows(g, tmp, NLF_WARP_MAX, NLF_SMALL_MAX, rows.p, d_count.p, &cnt));
  if (cnt) {
    k_nlf_cta<128, 4><<<std::min(cnt, H100_SMS * 16u), 128, 0, s>>>(rows.p, cnt, off, tgt, lab, end_bit, plab.p,
                                                                     pcnt.p, rowcnt.p);
    GB_CUDA(cudaGetLastError());
    ++launches;
  }
  GB_TRY(select_rows(g, tmp, NLF_SMALL_MAX, NLF_LARGE_MAX, rows.p, d_count.p, &cnt));
  if (cnt) {
    k_nlf_cta<256, 8><<<std::min(cnt, H100_SMS * 8u), 256, 0, s>>>(rows.p, cnt, off, tgt, lab, end_bit, plab.p,
                                                                    pcnt.p, rowcnt.p);
    GB_CUDA(cudaGetLastError());
    ++launches;
  }
  uint32_t hubs = 0;
  GB_TRY(select_rows(g, tmp, NLF_LARGE_MAX, 0xFFFFFFFFu, rows.p, d_count.p, &hubs));
  if (hubs) {
    DevBuf<uint32_t> seg, first, hub_counts, nruns;
    GB_TRY(seg.alloc((uint64_t)hubs + 1));
    k_hub_degrees<<<grid_for(hubs, 256), 256, 0, s>>>(rows.p, hubs, off, seg.p);
    GB_CUDA(cudaGetLastError());
    GB_TRY(exclusive_sum(s, tmp, seg.p, (int64_t)hubs + 1));
    uint32_t hub_entries = 0;
    GB_CUDA(cudaMemcpyAsync(&hub_entries, seg.p + hubs, 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    DevBuf<uint64_t> keys, sorted, unique;
    GB_TRY(keys.alloc(hub_entries));
    GB_TRY(sorted.alloc(hub_entries));
    k_nlf_hub_keys<<<std::min(hubs, H100_SMS * 8u), 256, 0, s>>>(rows.p, hubs, seg.p, off, tgt, lab, end_bit, keys.p);
    GB_CUDA(cudaGetLastError());
    const int key_bits = end_bit + label_bits(hubs - 1);
    GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
      return cub::DeviceRadixSort::SortKeys(t, tb, keys.p, sorted.p, (int64_t)hub_entries, 0, key_bits, s);
    }));
    keys.release();
    GB_TRY(unique.alloc(hub_entries));
    GB_TRY(hub_counts.alloc(hub_entries));
    GB_TRY(nruns.alloc(1));
    GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
      return cub::DeviceRunLengthEncode::Encode(t, tb, sorted.p, unique.p, hub_counts.p, nruns.p,
                                                (int64_t)hub_entries, s);
    }));
    GB_TRY(first.alloc((uint64_t)hubs + 1));
    k_nlf_hub_firsts<<<grid_for((uint64_t)hubs + 1, 256), 256, 0, s>>>(unique.p, nruns.p, rows.p, hubs, end_bit,
                                                                        first.p);
    k_nlf_hub_pairs<<<grid_for(hub_entries, 256), 256, 0, s>>>(unique.p, hub_counts.p, nruns.p, first.p, rows.p, hubs,
                                                                off, end_bit, plab.p, pcnt.p, rowcnt.p);
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaStreamSynchronize(s));  // before the hub buffers go
    launches += 5;
  }
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
    return cub::DeviceScan::ExclusiveSum(t, tb, rowcnt.p, pair_off.p, (int64_t)n + 1, s);
  }));
  uint32_t pairs = 0;
  GB_CUDA(cudaMemcpyAsync(&pairs, pair_off.p + n, 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  DevBuf<uint32_t> out_lab, out_cnt;
  GB_TRY(out_lab.alloc(pairs));
  GB_TRY(out_cnt.alloc(pairs));
  k_nlf_compact<<<grid_for((uint64_t)n * 32, 256), 256, 0, s>>>(off, rowcnt.p, pair_off.p, n, plab.p, pcnt.p,
                                                                out_lab.p, out_cnt.p);
  GB_CUDA(cudaGetLastError());
  launches += 2;
  GB_TRY(timing_end(g, launches));
  GB_CUDA(cudaMemcpyAsync(offsets, pair_off.p, ((size_t)n + 1) * 4, cudaMemcpyDeviceToHost, s));
  if (pairs) {
    GB_CUDA(cudaMemcpyAsync(labels_out, out_lab.p, (size_t)pairs * 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaMemcpyAsync(counts_out, out_cnt.p, (size_t)pairs * 4, cudaMemcpyDeviceToHost, s));
  }
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

}  // namespace gb

extern "C" {

gb_status gb_label_stats(const gb_graph* graph, gb_label_stats_info* stats, uint32_t* labels, uint64_t* counts) {
  return gb::label_stats(graph, stats, labels, counts);
}

gb_status gb_node_label_index(const gb_graph* graph, uint32_t* max_label, uint32_t* offsets, uint32_t* nodes) {
  return gb::node_label_index(graph, max_label, offsets, nodes);
}

gb_status gb_neighbor_label_frequencies(const gb_graph* graph, uint32_t* offsets, uint32_t* labels,
                                        uint32_t* counts) {
  return gb::neighbor_label_frequencies(graph, offsets, labels, counts);
}

}  // extern "C"
