// pr_layout.cu — the layout build of the JACOBI PageRank sweep (pagerank.cu): vertex renumbering, hot
// column blocks, the classification of every in-edge into a block segment or the row's SELL lane, the
// SELL-32 slices, the fill, and the chunks and tasks of the column-block kernel.  build_pr_plan runs these
// as named stages and ends with the sweep's launch shapes (plan_sweep_shape, pagerank.cu).
#include <cub/cub.cuh>

#include <algorithm>
#include <cmath>

#include "pr_plan.cuh"

namespace gb {

__device__ __forceinline__ uint32_t warp_max(uint32_t v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = max(v, __shfl_xor_sync(0xFFFFFFFFu, v, o));
  return v;
}

// ---- plan construction kernels ---------------------------------------------------------------
__global__ void k_perm_keys(const uint32_t* __restrict__ in_off, const uint32_t* __restrict__ out_off,
                            uint32_t n, uint64_t* __restrict__ keys, uint32_t* __restrict__ ids) {
  for (uint32_t v = blockIdx.x * blockDim.x + threadIdx.x; v < n; v += gridDim.x * blockDim.x) {
    uint32_t indeg = in_off[v + 1] - in_off[v];
    uint32_t outdeg = out_off[v + 1] - out_off[v];
    // in-degree descending (hub rows first, rows of similar length become neighbours), then
    // out-degree descending (hot sources first inside equal in-degrees).  R-MAT's expected in- and
    // out-degree of a vertex coincide, so this is also a hot-first order of the SOURCES.
    keys[v] = ((uint64_t)(uint32_t)(~indeg) << 32) | (uint32_t)(~outdeg);
    ids[v] = v;
  }
}
__global__ void k_perm_scatter(const uint32_t* __restrict__ sorted_ids, const uint32_t* __restrict__ out_off,
                               const uint32_t* __restrict__ in_off, uint32_t n, uint32_t* __restrict__ new_id,
                               uint32_t* __restrict__ outdeg, uint32_t* __restrict__ indeg) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r <= n; r += gridDim.x * blockDim.x) {
    if (r == n) {
      indeg[n] = 0;
      continue;
    }
    uint32_t v = sorted_ids[r];
    new_id[v] = r;
    outdeg[r] = out_off[v + 1] - out_off[v];
    indeg[r] = in_off[v + 1] - in_off[v];
  }
}
__global__ void k_count_active(const uint32_t* __restrict__ indeg, uint32_t n, uint32_t* __restrict__ count) {
  uint32_t act = 0;
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < n; r += gridDim.x * blockDim.x) act += indeg[r] > 0;
  for (int o = 16; o > 0; o >>= 1) act += __shfl_xor_sync(0xFFFFFFFFu, act, o);
  if ((threadIdx.x & 31) == 0 && act) atomicAdd(count, act);
}
// out-edges leaving each source block (one CTA per block): the block's share of all gathers
__global__ void k_blk_edges(const uint32_t* __restrict__ outdeg, uint32_t n, uint32_t B,
                            unsigned long long* __restrict__ blk_edges) {
  __shared__ unsigned long long part[8];
  const uint32_t b = blockIdx.x;
  const uint64_t lo = (uint64_t)b * B, hi = min((uint64_t)n, lo + B);
  unsigned long long s = 0;
  for (uint64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) s += outdeg[i];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (uint32_t w = 0; w < blockDim.x / 32; ++w) t += part[w];
    blk_edges[b] = t;
  }
}
// rows_ge[b] = number of (global) rows with in-degree >= dmin[b] (indeg is non-increasing);
// edges_ge[b] = the in-edges of those rows (deg_prefix = inclusive prefix sums of indeg)
__global__ void k_rows_ge(const uint32_t* __restrict__ indeg, const unsigned long long* __restrict__ deg_prefix,
                          uint32_t n_active, const uint32_t* __restrict__ dmin, uint32_t nblk,
                          uint32_t* __restrict__ rows_ge, unsigned long long* __restrict__ edges_ge) {
  for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < nblk; b += gridDim.x * blockDim.x) {
    const uint32_t d = dmin[b];
    uint32_t lo = 0, hi = n_active;  // first index with indeg < d
    while (lo < hi) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (indeg[mid] >= d) lo = mid + 1;
      else hi = mid;
    }
    rows_ge[b] = lo;
    edges_ge[b] = lo ? deg_prefix[lo - 1] : 0ull;
  }
}
struct U32ToU64 {
  __host__ __device__ unsigned long long operator()(uint32_t v) const { return v; }
};

// Classification of the in-edges of the rows that own segments (local rows [n_mega, n_cb)).  An edge
// from source s (internal id) lands in block s / B; if that block is hot (rank j) and the row is inside
// the block's row prefix it belongs to segment (j, row), else to the row's SELL remainder.  One warp walks
// a row in CSR order and leaves one 8-byte RECORD per edge, so that the fill pass — which has to wait for
// the scan over all segment sizes — is a plain scatter with no lookups left:
//   segment edge:   x = block-local id | j << 16,   y = 1 << 31 | position inside the segment
//   remainder edge: x = internal source id,         y = position inside the row's SELL lane
// Positions follow the CSR order (the per-pair counter is advanced batch by batch, each batch waits for
// the previous one's counter value): the layout is deterministic.
constexpr uint32_t CB_REC_SEG = 0x80000000u;
template <bool CHECK>
__device__ __forceinline__ uint32_t cb_classify_row(uint32_t l, uint32_t b0, uint32_t d, uint32_t n,
                                                    const uint32_t* __restrict__ in_tgt,
                                                    const uint32_t* __restrict__ new_id,
                                                    const uint32_t* __restrict__ hot_of_blk,
                                                    const uint32_t* __restrict__ nrows,
                                                    const uint32_t* __restrict__ poff,
                                                    const uint32_t* __restrict__ blk, uint32_t B,
                                                    uint32_t* __restrict__ cnt, uint2* __restrict__ rec, uint32_t lane) {
  uint32_t rem = 0;
  // CB_ILP batches of 32 edges per iteration: their dependent loads (target -> internal id -> block
  // rank -> row prefix) are issued together, so a long row's single warp is not latency bound
  for (uint32_t i = 0; i < d; i += 32 * CB_ILP) {
    uint32_t j[CB_ILP], src[CB_ILP];
    bool valid[CB_ILP];
#pragma unroll
    for (uint32_t u = 0; u < CB_ILP; ++u) {
      const uint32_t k = i + 32 * u + lane;
      valid[u] = k < d;
      src[u] = 0;
      if (valid[u]) {
        uint32_t t = in_tgt[b0 + k];
        if (CHECK && t >= n) t = 0;  // reported by the chunk's id check; keep the lookups in range meanwhile
        src[u] = new_id[t];
      }
    }
#pragma unroll
    for (uint32_t u = 0; u < CB_ILP; ++u) j[u] = valid[u] ? hot_of_blk[src[u] / B] : CB_NONE;
#pragma unroll
    for (uint32_t u = 0; u < CB_ILP; ++u)
      if (j[u] != CB_NONE && l >= nrows[j[u]]) j[u] = CB_NONE;
#pragma unroll
    for (uint32_t u = 0; u < CB_ILP; ++u) {
      const bool cb = j[u] != CB_NONE;
      const uint32_t peers = __match_any_sync(0xFFFFFFFFu, j[u]);
      const uint32_t leader = (uint32_t)__ffs(peers) - 1u;
      uint32_t base = 0, local = 0;
      if (cb) {
        local = src[u] - blk[j[u]] * B;
        if (lane == leader) base = atomicAdd(cnt + poff[j[u]] + l, (uint32_t)__popc(peers));
      }
      base = __shfl_sync(0xFFFFFFFFu, base, leader);  // also orders this batch's counter update before the next
      const uint32_t rb = __ballot_sync(0xFFFFFFFFu, valid[u] && !cb);
      if (cb) {
        rec[b0 + i + 32 * u + lane] = make_uint2(local | (j[u] << 16), CB_REC_SEG | (base + __popc(peers & ((1u << lane) - 1u))));
      } else if (valid[u]) {
        rec[b0 + i + 32 * u + lane] = make_uint2(src[u], rem + __popc(rb & ((1u << lane) - 1u)));
      }
      rem += __popc(rb);
    }
  }
  return rem;
}
// rows in internal order (the row source is resident): one warp per local row
__global__ void k_cb_count(const uint32_t* __restrict__ in_off, const uint32_t* __restrict__ in_tgt,
                           const uint32_t* __restrict__ old_of, const uint32_t* __restrict__ new_id,
                           const uint32_t* __restrict__ hot_of_blk, const uint32_t* __restrict__ nrows,
                           const uint32_t* __restrict__ poff, const uint32_t* __restrict__ blk, uint32_t B,
                           uint32_t row0, uint32_t n_cb, PrDeal deal, uint32_t* __restrict__ cnt,
                           uint2* __restrict__ rec, uint32_t* __restrict__ lens,
                           unsigned long long* __restrict__ cb_edges) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  unsigned long long in_cb = 0;
  for (uint32_t l = row0 + warp; l < n_cb; l += nwarps) {
    const uint32_t old = old_of[deal_global(l, deal.P, deal.p)];
    const uint32_t b0 = in_off[old], d = in_off[old + 1] - b0;
    const uint32_t rem = cb_classify_row<false>(l, b0, d, 0u, in_tgt, new_id, hot_of_blk, nrows, poff, blk, B, cnt, rec, lane);
    if (lane == 0) {
      lens[l] = rem;
      in_cb += d - rem;
    }
  }
  if (lane == 0 && in_cb) atomicAdd(cb_edges, in_cb);
}
// rows [v0, v1) in ORIGINAL order (a chunk of the in-CSR that has just arrived over PCIe): a warp takes
// 32 consecutive rows, keeps those that are local and own segments, and walks them one after the other
__global__ void k_cb_count_rows(const uint32_t* __restrict__ in_off, const uint32_t* __restrict__ in_tgt,
                                const uint32_t* __restrict__ new_id, const uint32_t* __restrict__ hot_of_blk,
                                const uint32_t* __restrict__ nrows, const uint32_t* __restrict__ poff,
                                const uint32_t* __restrict__ blk, uint32_t B, uint32_t v0, uint32_t v1, uint32_t n,
                                uint32_t row0, uint32_t n_cb, PrDeal deal, uint32_t* __restrict__ cnt,
                                uint2* __restrict__ rec, uint32_t* __restrict__ lens,
                                unsigned long long* __restrict__ cb_edges) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  unsigned long long in_cb = 0;
  for (uint64_t base = (uint64_t)v0 + 32ull * warp; base < v1; base += 32ull * nwarps) {
    const uint64_t v = base + lane;
    uint32_t l = CB_NONE, b0 = 0, d = 0;
    if (v < v1) {
      const uint32_t gid = new_id[v], slice = gid >> 5;
      if (slice % deal.P == deal.p) {
        const uint32_t loc = ((slice / deal.P) << 5) | (gid & 31u);
        if (loc >= row0 && loc < n_cb) {
          l = loc;
          b0 = in_off[v];
          d = in_off[v + 1] - b0;
        }
      }
    }
    uint32_t todo = __ballot_sync(0xFFFFFFFFu, l != CB_NONE);
    while (todo) {
      const int src_lane = __ffs(todo) - 1;
      todo &= todo - 1;
      const uint32_t rl = __shfl_sync(0xFFFFFFFFu, l, src_lane);
      const uint32_t rb = __shfl_sync(0xFFFFFFFFu, b0, src_lane);
      const uint32_t rd = __shfl_sync(0xFFFFFFFFu, d, src_lane);
      const uint32_t rem = cb_classify_row<true>(rl, rb, rd, n, in_tgt, new_id, hot_of_blk, nrows, poff, blk, B, cnt, rec, lane);
      if (lane == 0) {
        lens[rl] = rem;
        in_cb += rd - rem;
      }
    }
  }
  if (lane == 0 && in_cb) atomicAdd(cb_edges, in_cb);
}
// ---- the longest rows (a prefix of the local rows) go through ONE stable radix sort -----------------
// A row's warp walks it 128 edges at a time, ~3 us per step: a million-edge hub would take tens of
// milliseconds on its own.  Its edges are instead keyed (row << 14 | block rank), sorted stably — so
// the edges of one (row, block) pair end up contiguous AND in CSR order — and counted / placed from the
// sorted sequence, one thread per edge.
__global__ void k_mega_deg(const uint32_t* __restrict__ indeg, uint32_t n_mega, PrDeal deal, uint32_t* __restrict__ out) {
  for (uint32_t l = blockIdx.x * blockDim.x + threadIdx.x; l < n_mega; l += gridDim.x * blockDim.x)
    out[l] = indeg[deal_global(l, deal.P, deal.p)];
}
__global__ void k_mega_keys(const uint32_t* __restrict__ in_off, const uint32_t* __restrict__ in_tgt,
                            const uint32_t* __restrict__ old_of, const uint32_t* __restrict__ new_id,
                            const uint32_t* __restrict__ hot_of_blk, const uint32_t* __restrict__ nrows, uint32_t B,
                            const uint32_t* __restrict__ moff, uint32_t n_mega, uint32_t M, PrDeal deal,
                            uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < M; i += gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = n_mega;  // row with moff[row] <= i < moff[row + 1]
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) / 2;
      if (moff[mid] <= i) lo = mid;
      else hi = mid;
    }
    const uint32_t l = lo;
    const uint32_t old = old_of[deal_global(l, deal.P, deal.p)];
    const uint32_t src = new_id[in_tgt[in_off[old] + (i - moff[l])]];
    uint32_t j = hot_of_blk[src / B];
    if (j != CB_NONE && l >= nrows[j]) j = CB_NONE;
    keys[i] = (l << CB_MEGA_JBITS) | (j == CB_NONE ? (1u << CB_MEGA_JBITS) - 1u : j);
    vals[i] = src;
  }
}
__global__ void k_mega_starts(const uint32_t* __restrict__ keys, uint32_t M, uint32_t* __restrict__ start) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < M; i += gridDim.x * blockDim.x)
    start[i] = (i == 0 || keys[i] != keys[i - 1]) ? i : 0u;  // max-scanned into "first index of my run"
}
__global__ void k_mega_counts(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ start, uint32_t M,
                              const uint32_t* __restrict__ poff, uint32_t* __restrict__ cnt,
                              uint32_t* __restrict__ lens, unsigned long long* __restrict__ cb_edges) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < M; i += gridDim.x * blockDim.x) {
    if (i + 1 < M && keys[i + 1] == keys[i]) continue;  // not the last edge of its run
    const uint32_t len = i + 1 - start[i];
    const uint32_t l = keys[i] >> CB_MEGA_JBITS, j = keys[i] & ((1u << CB_MEGA_JBITS) - 1u);
    if (j == (1u << CB_MEGA_JBITS) - 1u) {
      lens[l] = len;
    } else {
      cnt[poff[j] + l] = len;
      atomicAdd(cb_edges, (unsigned long long)len);
    }
  }
}
__global__ void k_mega_fill(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                            const uint32_t* __restrict__ start, uint32_t M, const uint32_t* __restrict__ poff,
                            const uint32_t* __restrict__ blk, uint32_t B, const uint32_t* __restrict__ goff,
                            uint16_t* __restrict__ ids, const uint2* __restrict__ slice_meta,
                            uint32_t* __restrict__ sell) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < M; i += gridDim.x * blockDim.x) {
    const uint32_t pos = i - start[i];
    const uint32_t l = keys[i] >> CB_MEGA_JBITS, j = keys[i] & ((1u << CB_MEGA_JBITS) - 1u);
    if (j == (1u << CB_MEGA_JBITS) - 1u) {
      const uint2 meta = slice_meta[l >> 5];
      sell[((uint64_t)meta.x + (uint64_t)(pos / 4) * 32 + (l & 31u)) * 4 + (pos % 4)] = vals[i];
    } else {
      ids[(uint64_t)goff[poff[j] + l] * CB_G + pos] = (uint16_t)(vals[i] - blk[j] * B);
    }
  }
}
__global__ void k_lens_tail(const uint32_t* __restrict__ indeg, uint32_t n_cb, uint32_t n_loc, PrDeal deal,
                            uint32_t* __restrict__ lens) {
  for (uint32_t l = n_cb + blockIdx.x * blockDim.x + threadIdx.x; l < n_loc; l += gridDim.x * blockDim.x)
    lens[l] = indeg[deal_global(l, deal.P, deal.p)];
}
__global__ void k_loc_edges(const uint32_t* __restrict__ indeg, uint32_t n_loc, PrDeal deal,
                            unsigned long long* __restrict__ total) {
  unsigned long long s = 0;
  for (uint32_t l = blockIdx.x * blockDim.x + threadIdx.x; l < n_loc; l += gridDim.x * blockDim.x)
    s += indeg[deal_global(l, deal.P, deal.p)];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
  if ((threadIdx.x & 31) == 0 && s) atomicAdd(total, s);
}
// edges of a pair -> groups of its segment (every pair of the staircase keeps at least one group, so
// that the row of a group follows from counting segment starts)
__global__ void k_cb_groups(uint32_t* __restrict__ cnt, uint64_t S) {
  for (uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; e < S; e += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t c = cnt[e];
    cnt[e] = c ? (c + CB_G - 1) / CB_G : 1u;
  }
}
__global__ void k_fill_u2(uint2* __restrict__ a, uint64_t count, uint2 v) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < count; i += (uint64_t)gridDim.x * blockDim.x)
    a[i] = v;
}
__global__ void k_cb_bits(const uint32_t* __restrict__ goff, uint64_t S, uint32_t* __restrict__ bits) {
  for (uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; e < S; e += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t g = goff[e];
    atomicOr(bits + (g >> 5), 1u << (g & 31u));
  }
}
// SELL slice widths: the longest lane of the slice, in 4-edge groups
__global__ void k_sell_widths(const uint32_t* __restrict__ lens, uint32_t n_loc, uint32_t num_slices,
                              uint32_t* __restrict__ units) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t sidx = warp; sidx < num_slices; sidx += nwarps) {
    const uint32_t l = 32 * sidx + lane;
    const uint32_t w = warp_max(l < n_loc ? lens[l] : 0u);
    if (lane == 0) units[sidx] = ((w + 3) / 4) * 32;  // uint4 entries of the slice
  }
}
__global__ void k_sell_meta(const uint32_t* __restrict__ units, const uint32_t* __restrict__ bases,
                            uint32_t num_slices, uint2* __restrict__ meta) {
  for (uint32_t sidx = blockIdx.x * blockDim.x + threadIdx.x; sidx < num_slices; sidx += gridDim.x * blockDim.x)
    meta[sidx] = make_uint2(bases[sidx], units[sidx] / 32);
}
// after the scan over the segment sizes: scatter the records left by the classification — block-local
// ids into the segments, all other sources into the row's SELL lane
__global__ void k_cb_fill(const uint32_t* __restrict__ in_off, const uint32_t* __restrict__ old_of,
                          const uint2* __restrict__ rec, const uint32_t* __restrict__ poff, uint32_t row0,
                          uint32_t n_cb, PrDeal deal, const uint32_t* __restrict__ goff, uint16_t* __restrict__ ids,
                          const uint2* __restrict__ slice_meta, uint32_t* __restrict__ sell) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t l = row0 + warp; l < n_cb; l += nwarps) {
    const uint32_t old = old_of[deal_global(l, deal.P, deal.p)];
    const uint32_t b0 = in_off[old], d = in_off[old + 1] - b0;
    const uint2 meta = slice_meta[l >> 5];
    for (uint32_t i = 0; i < d; i += 32 * CB_ILP) {
      uint2 r[CB_ILP];
      uint32_t g0[CB_ILP];
#pragma unroll
      for (uint32_t u = 0; u < CB_ILP; ++u) {
        const uint32_t k = i + 32 * u + lane;
        r[u] = k < d ? rec[b0 + k] : make_uint2(0u, 0xFFFFFFFFu);
      }
#pragma unroll
      for (uint32_t u = 0; u < CB_ILP; ++u)
        g0[u] = (r[u].y != 0xFFFFFFFFu && (r[u].y & CB_REC_SEG)) ? goff[poff[r[u].x >> 16] + l] : 0u;
#pragma unroll
      for (uint32_t u = 0; u < CB_ILP; ++u) {
        if (r[u].y == 0xFFFFFFFFu) continue;
        if (r[u].y & CB_REC_SEG) {
          ids[(uint64_t)g0[u] * CB_G + (r[u].y & ~CB_REC_SEG)] = (uint16_t)(r[u].x & 0xFFFFu);
        } else {
          const uint32_t q = r[u].y;
          sell[((uint64_t)meta.x + (uint64_t)(q / 4) * 32 + (l & 31u)) * 4 + (q % 4)] = r[u].x;
        }
      }
    }
  }
}
// rows without segments: the whole row goes to its SELL lane (one lane per row)
__global__ void k_sell_fill_tail(const uint32_t* __restrict__ in_off, const uint32_t* __restrict__ in_tgt,
                                 const uint32_t* __restrict__ old_of, const uint32_t* __restrict__ new_id,
                                 uint32_t n_cb, uint32_t n_loc, PrDeal deal, uint32_t num_slices,
                                 const uint2* __restrict__ meta, uint4* __restrict__ sell) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t sidx = n_cb / 32 + warp; sidx < num_slices; sidx += nwarps) {
    const uint2 m = meta[sidx];
    const uint32_t l = 32 * sidx + lane;
    if (l < n_cb) continue;  // filled by k_cb_fill (lanes of the boundary slice)
    uint32_t b = 0, d = 0;
    if (l < n_loc) {
      const uint32_t old = old_of[deal_global(l, deal.P, deal.p)];
      b = in_off[old];
      d = in_off[old + 1] - b;
    }
    for (uint32_t q = 0; q * 4 < d; ++q) {
      uint4 v = make_uint4(~0u, ~0u, ~0u, ~0u);
      const uint32_t j = 4 * q;
      if (j + 0 < d) v.x = new_id[in_tgt[b + j + 0]];
      if (j + 1 < d) v.y = new_id[in_tgt[b + j + 1]];
      if (j + 2 < d) v.z = new_id[in_tgt[b + j + 2]];
      if (j + 3 < d) v.w = new_id[in_tgt[b + j + 3]];
      sell[m.x + q * 32 + lane] = v;
    }
  }
}
__global__ void k_gather_u32(const uint32_t* __restrict__ src, const uint32_t* __restrict__ idx, uint32_t count,
                             uint32_t* __restrict__ dst) {
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += gridDim.x * blockDim.x) dst[i] = src[idx[i]];
}

// Chunks: block j's stream [gbeg[j], gbeg[j+1]) is cut every C_j groups; a cut inside a segment moves to
// the segment's end unless the segment is longer than C_j groups, in which case the cut stays and both
// neighbours handle a PART of it (side buffer + fixup), so no warp ever owns more than 2 C_j groups.
// C_j shrinks for thin blocks so that every block's stream is spread over all warps of a CTA (a lone
// warp runs at its dependency latency, ~10x below the SM's throughput).
struct CbCut {
  uint32_t pos, row;
  bool mid;
};
__device__ __forceinline__ CbCut cb_cut(const uint32_t* __restrict__ goff_j, uint32_t nr, uint32_t gend, uint32_t q,
                                        uint32_t C) {
  if (q >= gend) return CbCut{gend, nr, false};
  uint32_t lo = 0, hi = nr;  // largest row with goff_j[row] <= q
  while (hi - lo > 1) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (goff_j[mid] <= q) lo = mid;
    else hi = mid;
  }
  const uint32_t s0 = goff_j[lo], s1 = (lo + 1 < nr) ? goff_j[lo + 1] : gend;
  if (s0 == q) return CbCut{q, lo, false};
  if (s1 - s0 > C) return CbCut{q, lo, true};
  return CbCut{s1, lo + 1, false};
}
__global__ void k_cb_chunks(const uint32_t* __restrict__ goff, const uint32_t* __restrict__ poff,
                            const uint32_t* __restrict__ nrows, const uint32_t* __restrict__ gbeg,
                            const uint32_t* __restrict__ cfirst, const uint32_t* __restrict__ cgrp, uint32_t KB,
                            uint32_t n_chunks, uint4* __restrict__ chunks, uint32_t* __restrict__ tail_slot,
                            uint32_t* __restrict__ fix_list, uint32_t* __restrict__ n_fix /* [1] = largest cut row */) {
  for (uint32_t c = blockIdx.x * blockDim.x + threadIdx.x; c < n_chunks; c += gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = KB;  // block with cfirst[j] <= c < cfirst[j + 1]
    while (hi - lo > 1) {
      const uint32_t mid = lo + (hi - lo) / 2;
      if (cfirst[mid] <= c) lo = mid;
      else hi = mid;
    }
    const uint32_t j = lo, k = c - cfirst[j];
    const uint32_t C = cgrp[j];  // groups per chunk in this block (thin blocks use small chunks)
    const uint32_t* goff_j = goff + poff[j];
    const uint32_t nr = nrows[j], g0 = gbeg[j], g1 = gbeg[j + 1];
    const bool last = c + 1 == cfirst[j + 1];
    const CbCut a = cb_cut(goff_j, nr, g1, g0 + k * C, C);
    const CbCut b = last ? CbCut{g1, nr, false} : cb_cut(goff_j, nr, g1, g0 + (k + 1) * C, C);
    uint32_t fl = 0;
    if (a.mid) fl |= CB_HEAD_CONT;
    if (b.mid) fl |= CB_TAIL_CONT;
    const uint32_t last_row = b.mid ? b.row : b.row - 1;  // row of the chunk's last group
    if (a.mid && last_row == a.row) fl |= CB_INTERIOR;
    const uint32_t row_before = a.mid ? a.row : a.row - 1;
    chunks[c] = make_uint4(a.pos, b.pos, row_before, j | (fl << 24));
    tail_slot[c] = b.mid ? poff[j] + b.row : CB_NONE;
    if (b.mid && !(fl & CB_INTERIOR)) {
      fix_list[atomicAdd(n_fix, 1u)] = c;
      atomicMax(n_fix + 1, b.row);
    }
  }
}

// Bank-aware order of the ids inside each group (tools/cb_bank_model.py restates it).  A step of k_pr_cb
// reads a WINDOW of 32 G groups (G = cb_step_groups, the kernel's choice for the chunk): lane L's groups
// G L + i (i < G) feed its shared-memory reads 4i..4i+3, and each of those read instructions takes as many
// wavefronts as its most crowded bank (id & 31) holds words.  The 4 ids of a group belong to one (row,
// block) pair, so their order only changes the rounding of the group's sum.  One thread per SET i of a
// window: lanes 0..31 in turn put the 4 ids of their group G L + i into the 4 read slots in the order (of
// 24) that lands them on the least loaded banks so far; padding ids (all lanes read the same word, a
// broadcast) are free.  A set keeps its old order unless the new one lowers the sum over its slots of the
// largest bank count.  Windows are the kernel's steps: chunk c steps from g0 & ~1 by 32 G and reads groups
// outside [g0, g1) as padding (they are ordered by their own chunk), so every group is ordered by exactly
// one thread and the result does not depend on thread timing.
constexpr int CB_BANK_THREADS = 128;
__global__ void __launch_bounds__(CB_BANK_THREADS) k_cb_bank_order(const uint4* __restrict__ chunks, uint32_t n_chunks,
                                                                   uint32_t B, uint2* __restrict__ ids) {
  __shared__ uint8_t hist[4 * 32][CB_BANK_THREADS];  // [slot * 32 + bank][thread]: no two threads share a byte
  uint8_t(*h)[CB_BANK_THREADS] = hist;
  const uint32_t t = threadIdx.x, lane = t & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + t) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  // the 24 orders, slot -> id index, two bits per slot; the identity first, so ties keep the old order
  constexpr uint8_t perms[24] = {0xE4, 0xB4, 0xD8, 0x78, 0x9C, 0x6C, 0xE1, 0xB1, 0xC9, 0x39, 0x8D, 0x2D,
                                 0xD2, 0x72, 0xC6, 0x36, 0x4E, 0x1E, 0x93, 0x63, 0x87, 0x27, 0x4B, 0x1B};
  const auto clear = [&]() {
    for (int i = 0; i < 4 * 32; ++i) h[i][t] = 0;
  };
  const auto bound = [&]() {  // sum over the slots of max(1, the largest bank count)
    uint32_t tot = 0;
    for (int s = 0; s < 4; ++s) {
      uint32_t mx = 1;
      for (int b = 0; b < 32; ++b) mx = max(mx, (uint32_t)h[s * 32 + b][t]);
      tot += mx;
    }
    return tot;
  };
  uint2 out[32];
  for (uint32_t c = warp; c < n_chunks; c += nwarps) {
    const uint4 ch = chunks[c];
    const uint32_t g0 = ch.x, g1 = ch.y;
    if (g0 >= g1) continue;
    const uint32_t G = cb_step_groups(g0, g1);
    const uint32_t set = lane % G;
    for (uint32_t gw = (g0 & ~1u) + 32 * G * (lane / G); gw < g1; gw += 32 * 32) {
      clear();
      for (uint32_t L = 0; L < 32; ++L) {
        const uint32_t g = gw + G * L + set;
        if (g < g0 || g >= g1) continue;
        const uint2 v = ids[g];
        const uint32_t id[4] = {v.x & 0xFFFFu, v.x >> 16, v.y & 0xFFFFu, v.y >> 16};
        for (int s = 0; s < 4; ++s)
          if (id[s] != B) ++h[s * 32 + (id[s] & 31u)][t];
      }
      const uint32_t before = bound();
      clear();
      for (uint32_t L = 0; L < 32; ++L) {
        const uint32_t g = gw + G * L + set;
        if (g < g0 || g >= g1) continue;
        const uint2 v = ids[g];
        const uint32_t id[4] = {v.x & 0xFFFFu, v.x >> 16, v.y & 0xFFFFu, v.y >> 16};
        uint32_t cost[4][4];  // [slot][id index]: load of the id's bank in that slot so far
#pragma unroll
        for (int s = 0; s < 4; ++s)
#pragma unroll
          for (int k = 0; k < 4; ++k) cost[s][k] = id[k] == B ? 0u : h[s * 32 + (id[k] & 31u)][t];
        uint32_t best = 0, best_cost = 0xFFFFFFFFu;
#pragma unroll
        for (int p = 0; p < 24; ++p) {
          uint32_t sum = 0;
#pragma unroll
          for (int s = 0; s < 4; ++s) sum += cost[s][(perms[p] >> (2 * s)) & 3u];
          if (sum < best_cost) {
            best_cost = sum;
            best = perms[p];
          }
        }
        uint32_t o[4];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          const uint32_t k = (best >> (2 * s)) & 3u;
          o[s] = k == 0 ? id[0] : k == 1 ? id[1] : k == 2 ? id[2] : id[3];
          if (o[s] != B) ++h[s * 32 + (o[s] & 31u)][t];
        }
        out[L] = make_uint2(o[0] | (o[1] << 16), o[2] | (o[3] << 16));
      }
      if (bound() >= before) continue;
      for (uint32_t L = 0; L < 32; ++L) {
        const uint32_t g = gw + G * L + set;
        if (g >= g0 && g < g1) ids[g] = out[L];
      }
    }
  }
}

// ---- layout build ----------------------------------------------------------------------------------
// The degrees (order, hot blocks, staircase) come from the PrSource's full offsets; the rows' edges from the
// row source (row_off, row_tgt) given to layout_end, which for a resident twin is its in-CSR.
template <typename T>
static gb_status scan_exclusive(cudaStream_t s, T* data, uint64_t count) {
  GB_REQUIRE(count < (1ull << 31), "scan of %llu items is too long", (unsigned long long)count);
  DevBuf<uint8_t> tmp;
  GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) { return cub::DeviceScan::ExclusiveSum(t, tb, data, data, (int)count, s); }));
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}
template <typename T>
static gb_status upload(cudaStream_t s, DevBuf<T>* dst, const std::vector<T>& src, size_t pad = 0) {
  GB_TRY(dst->alloc(std::max<size_t>(src.size(), 1), pad));
  if (!src.empty()) GB_CUDA(cudaMemcpyAsync(dst->p, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice, s));
  GB_CUDA(cudaStreamSynchronize(s));  // src may be a temporary
  return GB_OK;
}

// What lives through the whole build; a stage's own temporaries are its locals.  Both matter: releasing a
// buffer waits for the stream (the streamed upload overlaps with those waits), and rec alone holds 8 bytes
// per in-edge, so a longer lifetime raises the build's peak memory.
struct LayoutBuild {
  PrSource src;
  PrPlan* p = nullptr;
  PrDeal deal;
  cudaStream_t s = nullptr;
  uint32_t n = 0;
  uint64_t m = 0;
  uint32_t B = 0;
  double tau = CB_TAU_DEFAULT;
  int dev_sms = (int)H100_SMS;
  // the row source (layout_end): row v's in-edges are row_tgt[row_off[v] .. row_off[v + 1]), row_entries in all
  const uint32_t* row_off = nullptr;
  const uint32_t* row_tgt = nullptr;
  uint64_t row_entries = 0;
  uint32_t n_mega = 0;  // local rows [0, n_mega) take the sort path of the build
  uint32_t M = 0;       // their in-edges
  std::vector<uint32_t> h_nrows, h_poff;  // the staircase on the host
  DevBuf<uint32_t> old_of;  // internal id -> original id
  DevBuf<uint32_t> indeg;   // in-degree by internal id [n + 1]
  DevBuf<unsigned long long> counters;  // [0] active rows, [1] local edges, [2] edges in segments, [3] fix count
  DevBuf<uint32_t> hot_of_blk;  // source block -> hot rank (CB_NONE: not hot)
  DevBuf<uint32_t> goff;  // [S + 1] edges per pair -> groups per pair -> first group of each pair
  DevBuf<uint32_t> lens;  // [n_loc] SELL lane lengths
  DevBuf<uint32_t> mega_keys, mega_vals, mega_start, mega_off;  // sorted edges of the rows on the sort path
  DevBuf<uint2> rec;      // one record per in-edge of the other rows that own segments
  // the stages, in this order
  gb_status layout_order();
  gb_status layout_hot_blocks();
  gb_status layout_classify();
  gb_status layout_sell();
  gb_status layout_fill();
  gb_status layout_chunks();
};

// permutation (in-degree descending, then out-degree descending, then id), the active rows (a prefix of
// the internal order) and this rank's share of them
gb_status LayoutBuild::layout_order() {
  {
    DevBuf<uint64_t> keys, keys_alt;
    DevBuf<uint32_t> ids, ids_alt;
    GB_TRY(keys.alloc(n));
    GB_TRY(keys_alt.alloc(n));
    GB_TRY(ids.alloc(n));
    GB_TRY(ids_alt.alloc(n));
    k_perm_keys<<<grid_for(n, 256), 256, 0, s>>>(src.in_off, src.out_off, n, keys.p, ids.p);
    cub::DoubleBuffer<uint64_t> kb(keys.p, keys_alt.p);
    cub::DoubleBuffer<uint32_t> vb(ids.p, ids_alt.p);
    DevBuf<uint8_t> tmp;
    GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) { return cub::DeviceRadixSort::SortPairs(t, tb, kb, vb, (int)n, 0, 64, s); }));
    GB_TRY(p->new_id.alloc(n));
    GB_TRY(p->outdeg.alloc(n));
    GB_TRY(indeg.alloc((size_t)n + 1));
    k_perm_scatter<<<grid_for(n, 256), 256, 0, s>>>(vb.Current(), src.out_off, src.in_off, n, p->new_id.p,
                                                   p->outdeg.p, indeg.p);
    GB_TRY(old_of.alloc(n));
    GB_CUDA(cudaMemcpyAsync(old_of.p, vb.Current(), (size_t)n * 4, cudaMemcpyDeviceToDevice, s));
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaStreamSynchronize(s));
  }
  GB_TRY(counters.alloc(4));
  GB_CUDA(cudaMemsetAsync(counters.p, 0, 32, s));
  k_count_active<<<grid_for(n, 256), 256, 0, s>>>(indeg.p, n, reinterpret_cast<uint32_t*>(counters.p));
  unsigned long long h = 0;
  GB_CUDA(cudaMemcpyAsync(&h, counters.p, 8, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  p->n_active = (uint32_t)h;
  p->n_loc = deal_count(p->n_active, deal.P, deal.p);
  if (p->n_loc) k_loc_edges<<<grid_for(p->n_loc, 256), 256, 0, s>>>(indeg.p, p->n_loc, deal, counters.p + 1);
  return GB_OK;
}

// Hot blocks: block b carries the share e_b / m of all gathers; a row of in-degree d expects d * e_b / m
// edges from it, and gets a segment when that is at least tau.  Blocks are ranked by their row prefix,
// longest first (the staircase).
gb_status LayoutBuild::layout_hot_blocks() {
  const uint32_t nblk = (uint32_t)(((uint64_t)n + B - 1) / B);
  std::vector<uint32_t> h_hot(nblk, CB_NONE), h_blk;
  if (p->n_loc && m) {
    DevBuf<unsigned long long> blk_edges, deg_prefix, edges_ge;
    DevBuf<uint32_t> dmin, rows_ge;
    GB_TRY(blk_edges.alloc(nblk));
    GB_TRY(dmin.alloc(nblk + 1));  // + one probe: the rows long enough for the sort path of the build
    GB_TRY(rows_ge.alloc(nblk + 1));
    GB_TRY(edges_ge.alloc(nblk + 1));
    GB_TRY(deg_prefix.alloc(std::max<uint32_t>(p->n_active, 1)));
    {
      cub::TransformInputIterator<unsigned long long, U32ToU64, const uint32_t*> it(indeg.p, U32ToU64());
      DevBuf<uint8_t> tmp;
      GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
        return cub::DeviceScan::InclusiveSum(t, tb, it, deg_prefix.p, (int)p->n_active, s);
      }));
      GB_CUDA(cudaStreamSynchronize(s));
    }
    k_blk_edges<<<nblk, 256, 0, s>>>(p->outdeg.p, n, B, blk_edges.p);
    std::vector<unsigned long long> h_edges(nblk);
    GB_CUDA(cudaMemcpyAsync(h_edges.data(), blk_edges.p, (size_t)nblk * 8, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    std::vector<uint32_t> h_dmin(nblk + 1, 0xFFFFFFFFu);
    h_dmin[nblk] = (uint32_t)env_u64("GB_PR_MEGA", CB_MEGA_DEG) + 1;
    for (uint32_t b = 0; b < nblk; ++b)
      if (h_edges[b]) {
        const double d = std::ceil(tau * (double)m / (double)h_edges[b]);
        h_dmin[b] = d >= 4294967295.0 ? 0xFFFFFFFFu : std::max<uint32_t>(1u, (uint32_t)d);
      }
    GB_CUDA(cudaMemcpyAsync(dmin.p, h_dmin.data(), (size_t)(nblk + 1) * 4, cudaMemcpyHostToDevice, s));
    k_rows_ge<<<grid_for(nblk + 1, 128), 128, 0, s>>>(indeg.p, deg_prefix.p, p->n_active, dmin.p, nblk + 1,
                                                       rows_ge.p, edges_ge.p);
    std::vector<uint32_t> h_rows(nblk + 1);
    std::vector<unsigned long long> h_ege(nblk + 1);
    GB_CUDA(cudaMemcpyAsync(h_rows.data(), rows_ge.p, (size_t)(nblk + 1) * 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaMemcpyAsync(h_ege.data(), edges_ge.p, (size_t)(nblk + 1) * 8, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    n_mega = deal_count(h_rows[nblk], deal.P, deal.p);
    // every block that some local row expects tau edges from: a thin block costs one block load (~2 us on
    // one SM), while its ids would otherwise lengthen the SELL lanes of the hub rows, which one lane walks
    // serially
    std::vector<uint32_t> order;
    for (uint32_t b = 0; b < nblk; ++b)
      if (h_dmin[b] != 0xFFFFFFFFu && deal_count(h_rows[b], deal.P, deal.p) != 0) order.push_back(b);
    std::sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) {
      return h_rows[x] != h_rows[y] ? h_rows[x] > h_rows[y] : x < y;
    });
    if (order.size() > CB_MAX_BLOCKS) order.resize(CB_MAX_BLOCKS);
    uint64_t S = 0;
    for (uint32_t j = 0; j < order.size(); ++j) {
      const uint32_t b = order[j];
      h_hot[b] = j;
      h_blk.push_back(b);
      h_nrows.push_back(deal_count(h_rows[b], deal.P, deal.p));
      h_poff.push_back((uint32_t)S);
      S += h_nrows.back();
      GB_REQUIRE(S < 0xFFFFFFF0ull, "column-block staircase too large (%llu pairs)", (unsigned long long)S);
    }
    h_poff.push_back((uint32_t)S);
    p->S = S;
  }
  p->KB = (uint32_t)h_blk.size();
  if (p->KB) p->last_hot_block = *std::max_element(h_blk.begin(), h_blk.end());
  p->n_cb = p->KB ? h_nrows[0] : 0;
  if (h_poff.empty()) h_poff.push_back(0);
  GB_TRY(upload(s, &hot_of_blk, h_hot));
  GB_TRY(upload(s, &p->blk, h_blk));
  GB_TRY(upload(s, &p->nrows, h_nrows));
  GB_TRY(upload(s, &p->poff, h_poff));
  return GB_OK;
}

// Segment sizes (pairs of the staircase) and SELL lane lengths: the longest rows are keyed and sorted once
// (the sorted edges are kept for layout_fill), every other row that owns segments is classified into one
// record per in-edge; the targets are classified chunk by chunk as they arrive when they stream in from a
// part (PrSource::feed).  Ends with goff = the first group of every pair.
gb_status LayoutBuild::layout_classify() {
  GB_TRY(goff.alloc(p->S + 1));
  GB_CUDA(cudaMemsetAsync(goff.p, 0, (p->S + 1) * 4, s));
  GB_TRY(lens.alloc(std::max<uint32_t>(p->n_loc, 1)));
  n_mega = std::min(n_mega, std::min(p->n_cb, (1u << (32 - CB_MEGA_JBITS)) - 1u));
  if (p->KB >= (1u << CB_MEGA_JBITS) - 1u) n_mega = 0;
  if (n_mega) {
    DevBuf<uint32_t> mdeg;
    GB_TRY(mdeg.alloc(n_mega));
    k_mega_deg<<<grid_for(n_mega, 128), 128, 0, s>>>(indeg.p, n_mega, deal, mdeg.p);
    std::vector<uint32_t> h_moff(n_mega + 1, 0);
    GB_CUDA(cudaMemcpyAsync(h_moff.data() + 1, mdeg.p, (size_t)n_mega * 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    uint64_t acc = 0;
    for (uint32_t r = 0; r < n_mega; ++r) {
      acc += h_moff[r + 1];
      if (acc >= 0xFFFFFFF0ull) {  // more mega edges than a 32-bit sort index holds: shorten the prefix
        n_mega = r;
        acc -= h_moff[r + 1];
        break;
      }
      h_moff[r + 1] = (uint32_t)acc;
    }
    h_moff.resize(n_mega + 1);
    M = n_mega ? h_moff[n_mega] : 0;
    if (M) GB_TRY(upload(s, &mega_off, h_moff));
    else n_mega = 0;
  }
  p->n_mega = n_mega;
  if (p->n_cb > n_mega) {
    uint32_t dmax = 0;  // a record holds a 31-bit position
    GB_CUDA(cudaMemcpyAsync(&dmax, indeg.p + deal_global(n_mega, deal.P, deal.p), 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    GB_REQUIRE(dmax < 0x7FFFFFFFu, "a row with %u in-edges outside the sort path of the layout build", dmax);
    GB_TRY(rec.alloc(std::max<uint64_t>(row_entries, 1)));
  }
  if (const CsrFeed* feed = src.feed) {
    // the targets arrive chunk by chunk: check and classify each chunk as soon as it is there
    DevBuf<unsigned int> bad;
    GB_TRY(bad.alloc(1));
    GB_CUDA(cudaMemsetAsync(bad.p, 0, 4, s));
    for (uint32_t k = 0; k < src.chunks->count(); ++k) {
      const uint32_t v0 = src.chunks->row[k], v1 = src.chunks->row[k + 1];
      const uint64_t e0 = src.chunks->edge[k], e1 = src.chunks->edge[k + 1];
      GB_CUDA(cudaStreamWaitEvent(s, feed->landed[k], 0));
      check_ids_async(s, row_tgt + e0, e1 - e0, n, bad.p);
      if (p->n_cb > n_mega && v1 > v0)
        k_cb_count_rows<<<grid_for((uint64_t)(v1 - v0), 256), 256, 0, s>>>(
            row_off, row_tgt, p->new_id.p, hot_of_blk.p, p->nrows.p, p->poff.p, p->blk.p, B, v0, v1, n,
            n_mega, p->n_cb, deal, goff.p, rec.p, lens.p, counters.p + 2);
    }
    unsigned int nbad = 0;
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaMemcpyAsync(&nbad, bad.p, 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    GB_TRY(require_ids("in", nbad, n));
  } else if (p->n_cb > n_mega) {
    k_cb_count<<<grid_for((uint64_t)(p->n_cb - n_mega) * 32, 256), 256, 0, s>>>(
        row_off, row_tgt, old_of.p, p->new_id.p, hot_of_blk.p, p->nrows.p, p->poff.p, p->blk.p, B,
        n_mega, p->n_cb, deal, goff.p, rec.p, lens.p, counters.p + 2);
  }
  if (M) {
    DevBuf<uint32_t> keys_in, vals_in;
    GB_TRY(keys_in.alloc(M));
    GB_TRY(vals_in.alloc(M));
    GB_TRY(mega_keys.alloc(M));
    GB_TRY(mega_vals.alloc(M));
    GB_TRY(mega_start.alloc(M));
    k_mega_keys<<<grid_for(M, 256), 256, 0, s>>>(row_off, row_tgt, old_of.p, p->new_id.p,
                                                 hot_of_blk.p, p->nrows.p, B, mega_off.p, n_mega, M, deal,
                                                 keys_in.p, vals_in.p);
    uint32_t row_bits = 1;
    while ((1u << row_bits) < n_mega) ++row_bits;
    uint32_t* start = mega_start.p;
    DevBuf<uint8_t> tmp, stmp;
    GB_TRY(cub_call(tmp, [&](void* t, size_t& tb) {
      return cub::DeviceRadixSort::SortPairs(t, tb, keys_in.p, mega_keys.p, vals_in.p, mega_vals.p, (int)M,
                                             0, (int)(CB_MEGA_JBITS + row_bits), s);
    }));
    k_mega_starts<<<grid_for(M, 256), 256, 0, s>>>(mega_keys.p, M, start);
    GB_TRY(cub_call(stmp, [&](void* t, size_t& tb) {
      return cub::DeviceScan::InclusiveScan(t, tb, start, start, cub::Max(), (int)M, s);
    }));
    GB_CUDA(cudaMemsetAsync(lens.p, 0, (size_t)n_mega * 4, s));
    k_mega_counts<<<grid_for(M, 256), 256, 0, s>>>(mega_keys.p, start, M, p->poff.p, goff.p, lens.p,
                                                   counters.p + 2);
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaStreamSynchronize(s));  // keys_in / vals_in / tmp / stmp are released here
  }
  if (p->n_loc > p->n_cb)
    k_lens_tail<<<grid_for(p->n_loc - p->n_cb, 256), 256, 0, s>>>(indeg.p, p->n_cb, p->n_loc, deal, lens.p);
  if (p->S) {
    k_cb_groups<<<grid_for(p->S, 256), 256, 0, s>>>(goff.p, p->S);
    GB_TRY(scan_exclusive(s, goff.p, p->S + 1));
    uint32_t ng = 0;
    GB_CUDA(cudaMemcpyAsync(&ng, goff.p + p->S, 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    p->NG = ng;
  }
  unsigned long long h[3] = {0, 0, 0};
  GB_CUDA(cudaMemcpyAsync(h, counters.p, 24, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  p->loc_edges = h[1];
  p->cb_edges = h[2];
  return GB_OK;
}

// SELL-32 slices of all local rows: widths, offsets, the padded lane array
gb_status LayoutBuild::layout_sell() {
  p->num_slices = (p->n_loc + 31) / 32;
  if (!p->num_slices) return GB_OK;
  DevBuf<uint32_t> units, bases;
  GB_TRY(units.alloc(p->num_slices));
  GB_TRY(bases.alloc(p->num_slices));
  k_sell_widths<<<grid_for((uint64_t)p->num_slices * 32, 256), 256, 0, s>>>(lens.p, p->n_loc, p->num_slices, units.p);
  GB_CUDA(cudaMemcpyAsync(bases.p, units.p, (size_t)p->num_slices * 4, cudaMemcpyDeviceToDevice, s));
  GB_TRY(scan_exclusive(s, bases.p, p->num_slices));
  uint32_t last_base = 0, last_units = 0;
  GB_CUDA(cudaMemcpyAsync(&last_base, bases.p + p->num_slices - 1, 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaMemcpyAsync(&last_units, units.p + p->num_slices - 1, 4, cudaMemcpyDeviceToHost, s));
  GB_CUDA(cudaStreamSynchronize(s));
  const size_t total_units = (size_t)last_base + last_units;
  GB_TRY(p->slice_meta.alloc(p->num_slices));
  GB_TRY(p->sell.alloc(total_units, 64));
  GB_CUDA(cudaMemsetAsync(p->sell.p, 0xFF, (total_units + 64) * sizeof(uint4), s));  // ~0 = padding
  k_sell_meta<<<grid_for(p->num_slices, 256), 256, 0, s>>>(units.p, bases.p, p->num_slices, p->slice_meta.p);
  GB_CUDA(cudaGetLastError());
  GB_CUDA(cudaStreamSynchronize(s));
  return GB_OK;
}

// fill: segments + SELL remainders of the rows below n_cb, whole rows above
gb_status LayoutBuild::layout_fill() {
  GB_TRY(p->cb_ids.alloc(std::max<uint64_t>(p->NG, 1), 64));
  GB_TRY(p->cb_bits.alloc(p->NG / 32 + 8));  // a 128-group step reads 5 words from its first
  GB_CUDA(cudaMemsetAsync(p->cb_bits.p, 0, (p->NG / 32 + 8) * 4, s));
  uint16_t* ids = reinterpret_cast<uint16_t*>(p->cb_ids.p);
  uint32_t* sell = reinterpret_cast<uint32_t*>(p->sell.p);
  if (p->NG) {
    k_fill_u2<<<grid_for(p->NG + 64, 256), 256, 0, s>>>(p->cb_ids.p, p->NG + 64, make_uint2(B | (B << 16), B | (B << 16)));
    k_cb_bits<<<grid_for(p->S, 256), 256, 0, s>>>(goff.p, p->S, p->cb_bits.p);
    if (M)
      k_mega_fill<<<grid_for(M, 256), 256, 0, s>>>(mega_keys.p, mega_vals.p, mega_start.p, M,
                                                       p->poff.p, p->blk.p, B, goff.p, ids, p->slice_meta.p, sell);
    if (p->n_cb > n_mega)
      k_cb_fill<<<grid_for((uint64_t)(p->n_cb - n_mega) * 32, 256), 256, 0, s>>>(
          row_off, old_of.p, rec.p, p->poff.p, n_mega, p->n_cb, deal, goff.p, ids, p->slice_meta.p,
          sell);
    GB_CUDA(cudaGetLastError());
    GB_CUDA(cudaStreamSynchronize(s));
  }
  if (p->n_loc > p->n_cb) {
    k_sell_fill_tail<<<grid_for((uint64_t)(p->num_slices - p->n_cb / 32) * 32, 256), 256, 0, s>>>(
        row_off, row_tgt, old_of.p, p->new_id.p, p->n_cb, p->n_loc, deal, p->num_slices,
        p->slice_meta.p, p->sell.p);
    GB_CUDA(cudaGetLastError());
  }
  return GB_OK;
}

// Chunks of the column-block kernel, the bank order of the ids inside them, and every persistent CTA's
// share of them (tasks); then the sweep's per-pair and per-row buffers.
gb_status LayoutBuild::layout_chunks() {
  p->grid_cb = 0;
  if (p->NG) {
    // first group of every block's stream
    DevBuf<uint32_t> gbeg;
    GB_TRY(gbeg.alloc(p->KB + 1));
    k_gather_u32<<<grid_for(p->KB + 1, 128), 128, 0, s>>>(goff.p, p->poff.p, p->KB + 1, gbeg.p);
    std::vector<uint32_t> h_gbeg(p->KB + 1);
    GB_CUDA(cudaMemcpyAsync(h_gbeg.data(), gbeg.p, (size_t)(p->KB + 1) * 4, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    // ~8 tasks per SM keep the dynamic schedule level; a task is 32 chunks (one per warp) of 512..2048
    // groups (fewer, longer chunks = fewer segments cut by chunk boundaries); a thin block is cut into
    // >= 64 chunks (down to one 64-group step each) so that all warps share it — a lone warp runs at
    // its dependency latency, ~10x below the SM's throughput
    uint32_t C = (uint32_t)env_u64("GB_PR_CHUNK", 0);
    const uint32_t T = std::min<uint32_t>(std::max<uint32_t>((uint32_t)env_u64("GB_PR_TASK_CHUNKS", CB_TASK_CHUNKS), 32u), 128u);
    if (!C) C = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(p->NG / ((uint64_t)dev_sms * 8 * T), 16384 / T), 65536 / T);
    C = std::max<uint32_t>(32u, (C + 31) / 32 * 32);
    p->chunk_groups = C;
    std::vector<uint32_t> h_cfirst(p->KB + 1, 0), h_cgrp(p->KB, C);
    std::vector<uint2> h_tasks;
    for (uint32_t j = 0; j < p->KB; ++j) {
      const uint32_t G = h_gbeg[j + 1] - h_gbeg[j];
      h_cgrp[j] = std::min<uint32_t>(C, std::max<uint32_t>(std::min<uint32_t>(64u, C), (G / 64 + 63) / 64 * 64));
      const uint32_t nc = (G + h_cgrp[j] - 1) / h_cgrp[j];
      h_cfirst[j + 1] = h_cfirst[j] + nc;
      for (uint32_t c = 0; c < nc; c += T)
        h_tasks.push_back(make_uint2(h_cfirst[j] + c, (std::min(nc, c + T) - c) | (j << 8)));
    }
    p->n_chunks = h_cfirst[p->KB];
    p->n_tasks = (uint32_t)h_tasks.size();
    p->grid_cb = (unsigned)std::min<uint64_t>(p->n_tasks, (uint64_t)dev_sms);  // one persistent CTA per SM
    GB_TRY(upload(s, &p->tasks, h_tasks));
    DevBuf<uint32_t> cfirst, cgrp;
    GB_TRY(upload(s, &cfirst, h_cfirst));
    GB_TRY(upload(s, &cgrp, h_cgrp));
    GB_TRY(p->chunks.alloc(p->n_chunks, 1));
    GB_TRY(p->tail_slot.alloc(p->n_chunks));
    GB_TRY(p->fix_list.alloc(p->n_chunks));
    GB_TRY(p->side.alloc((size_t)2 * p->n_chunks + 2));
    GB_CUDA(cudaMemsetAsync(p->side.p, 0, ((size_t)2 * p->n_chunks + 2) * 8, s));
    GB_CUDA(cudaMemsetAsync(p->chunks.p + p->n_chunks, 0, sizeof(uint4), s));  // sentinel: ends every fixup walk
    uint32_t* d_nfix = reinterpret_cast<uint32_t*>(counters.p + 3);
    k_cb_chunks<<<grid_for(p->n_chunks, 128), 128, 0, s>>>(goff.p, p->poff.p, p->nrows.p, gbeg.p, cfirst.p, cgrp.p,
                                                         p->KB, p->n_chunks, p->chunks.p, p->tail_slot.p,
                                                         p->fix_list.p, d_nfix);
    k_cb_bank_order<<<grid_for((uint64_t)p->n_chunks * 32, CB_BANK_THREADS), CB_BANK_THREADS, 0, s>>>(
        p->chunks.p, p->n_chunks, B, p->cb_ids.p);
    GB_CUDA(cudaGetLastError());
    uint32_t h_fix[2] = {0, 0};
    GB_CUDA(cudaMemcpyAsync(h_fix, d_nfix, 8, cudaMemcpyDeviceToHost, s));
    GB_CUDA(cudaStreamSynchronize(s));
    p->n_fix = h_fix[0];
    p->fix_max_row = h_fix[1];
  } else {
    GB_TRY(p->chunks.alloc(1));
    GB_TRY(p->tail_slot.alloc(1));
    GB_TRY(p->fix_list.alloc(1));
    GB_TRY(p->side.alloc(2));
    GB_TRY(p->tasks.alloc(1));
  }
  GB_TRY(p->task_ctr.alloc(std::max<unsigned>(p->grid_cb, 1)));
  GB_CUDA(cudaMemsetAsync(p->task_ctr.p, 0, (size_t)std::max<unsigned>(p->grid_cb, 1) * 4, s));
  GB_TRY(p->partial.alloc(std::max<uint64_t>(p->S, 1)));
  GB_CUDA(cudaMemsetAsync(p->partial.p, 0, std::max<uint64_t>(p->S, 1) * 4, s));
  GB_TRY(p->rem.alloc(std::max<uint32_t>(p->n_cb, 1)));
  std::vector<uint32_t> h_kb((p->n_cb + 31) / 32);
  for (size_t w = 0; w < h_kb.size(); ++w) h_kb[w] = fin_blocks_of(h_nrows.data(), p->KB, (uint32_t)w * 32);
  GB_TRY(upload(s, &p->fin_kb, h_kb));
  return GB_OK;
}

// The order stage runs first, on its own: a caller that builds its rows from the internal order (the local
// CSR of gb_pr_shards_csr_u32) reads layout_new_id before it hands the rows to layout_end.
gb_status layout_begin(const PrSource& src, PrDeal deal, LayoutBuild** out) {
  GB_REQUIRE(deal.P >= 1 && deal.p < deal.P, "bad shard %u of %u", deal.p, deal.P);
  DeviceGuard guard(src.device);
  LayoutBuild* b = new (std::nothrow) LayoutBuild();
  if (!b) return fail(GB_ERR_OOM, "host allocation failed");
  b->p = new (std::nothrow) PrPlan();
  if (!b->p) {
    delete b;
    return fail(GB_ERR_OOM, "host allocation failed");
  }
  b->src = src;
  b->deal = deal;
  b->s = src.stream;
  b->n = src.n;
  b->m = src.m;
  b->p->n = src.n;
  b->p->m = src.m;
  b->p->deal = deal;
  // every temporary of the build is used on src.stream only: releasing one waits for that stream, not for
  // the device (a copy stream may still be bringing in the targets, see PrSource::feed)
  DevBufStreamScope scope(src.stream);
  gb_status st = [&]() -> gb_status {
    GB_CUDA(cudaDeviceGetAttribute(&b->dev_sms, cudaDevAttrMultiProcessorCount, src.device));
    // knobs (experiments; defaults are the measured optima)
    const uint32_t B = (uint32_t)env_u64("GB_PR_BLOCK", CB_BLOCK_DEFAULT);
    b->B = b->p->B = std::min<uint32_t>(std::max<uint32_t>(B & ~1023u, 1024u), CB_BLOCK_MAX);
    if (const char* e = getenv("GB_PR_TAU")) b->tau = atof(e);
    if (!(b->tau > 0.0)) b->tau = 1e30;  // tau <= 0 switches the column blocks off
    return b->layout_order();
  }();
  if (st != GB_OK) {
    layout_free(b);
    return st;
  }
  *out = b;
  return GB_OK;
}

const uint32_t* layout_new_id(const LayoutBuild* b) { return b->p->new_id.p; }

gb_status layout_end(LayoutBuild* b, const uint32_t* row_off, const uint32_t* row_tgt, uint64_t row_entries,
                     PrPlan** out_plan) {
  DeviceGuard guard(b->src.device);
  b->row_off = row_off;
  b->row_tgt = row_tgt;
  b->row_entries = row_entries;
  gb_status st = [&]() -> gb_status {
    DevBufStreamScope scope(b->s);
    GB_TRY(b->layout_hot_blocks());
    GB_TRY(b->layout_classify());
    GB_TRY(b->layout_sell());
    GB_TRY(b->layout_fill());
    GB_TRY(b->layout_chunks());
    return plan_sweep_shape(b->p, b->h_nrows, b->h_poff, b->dev_sms, b->s);
  }();
  if (st == GB_OK) {
    *out_plan = b->p;
    b->p = nullptr;
  }
  layout_free(b);
  return st;
}

void layout_free(LayoutBuild* b) {
  if (!b) return;
  DeviceGuard guard(b->src.device);
  DevBufStreamScope scope(b->s);
  free_pr_plan(b->p);
  delete b;
}

gb_status build_pr_plan(const PrSource& src, PrDeal deal, const uint32_t* row_off, const uint32_t* row_tgt,
                        uint64_t row_entries, PrPlan** out_plan) {
  LayoutBuild* b = nullptr;
  GB_TRY(layout_begin(src, deal, &b));
  return layout_end(b, row_off, row_tgt, row_entries, out_plan);
}

gb_status build_pr_plan(const gb_graph* g, PrDeal deal, PrPlan** out_plan) {
  PrSource src;
  src.device = g->device;
  src.stream = g->stream;
  src.n = g->n;
  src.m = g->in.len;
  src.in_off = g->in.off.p;
  src.out_off = g->out.off.p;
  return build_pr_plan(src, deal, g->in.off.p, g->in.tgt.p, g->in.len, out_plan);
}

}  // namespace gb
