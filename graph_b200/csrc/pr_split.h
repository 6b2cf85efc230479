// pr_split.h — how gb_page_rank_csr_multi_u32 / gb_pr_shards_csr_u32 cut a host in-CSR into parts (and
// gb_page_rank_csr_u32 into the chunks of its one part), kept free of CUDA so that it can be tested on the CPU.
//
// Part u of U takes the rows [R_u, R_{u+1}), R_0 = 0, R_U = n, where R_u is the first row whose offset reaches
// floor(m u / U): cuts fall at rows, so a part holds at most about m / U edges plus one row, and a hub longer
// than m / U leaves parts empty.  The part uploads in_off[R_u .. R_{u+1}], out_off[R_u .. R_{u+1}] and the
// targets [E_u, E_{u+1}), E_u = in_off[R_u], in row-aligned chunks cut the same way.
//
// Whatever the host arrays hold, the searches end inside their ranges (wcc_first_row_past), the row slices tile
// [0, n] (so each row v < n is checked for in_off[v] <= in_off[v + 1] by exactly one part, the one whose rows
// hold it), and every edge bound is clamped into [0, m] and into its part's range, so that no copy leaves the
// host array or the part's buffer.  Beyond the probes of those searches the split reads in_off[n] only.
#pragma once

#include <algorithm>
#include <cstdint>
#include <vector>

#include "wcc_split.h"

namespace gb {

struct PrPart {
  uint32_t r_begin = 0, r_end = 0;   // rows [r_begin, r_end): offsets [r_begin .. r_end] go to the device
  uint64_t e_begin = 0, e_end = 0;   // targets [e_begin, e_end)
  std::vector<uint32_t> chunk_row;   // [K + 1] chunk k holds the rows [chunk_row[k], chunk_row[k + 1])
  std::vector<uint64_t> chunk_edge;  // [K + 1] and the targets [chunk_edge[k], chunk_edge[k + 1])
};

// rows [r0, r1] cut into k slices of about equal edge counts: cut i (0 < i < k) is the first row in [r0, r1]
// whose offset reaches e0 + (e1 - e0) i / k, and no earlier than cut i - 1
inline std::vector<uint32_t> pr_row_cuts(const uint32_t* off, uint32_t r0, uint32_t r1, uint64_t e0, uint64_t e1,
                                         uint32_t k) {
  std::vector<uint32_t> cut(k + 1, r0);
  cut[k] = r1;
  for (uint32_t i = 1; i < k; ++i) {
    const uint64_t want = e0 + (e1 - e0) * i / k;
    cut[i] = std::max(cut[i - 1], r0 + wcc_first_row_past(off + r0, r1 - r0, want, false));
  }
  return cut;
}

// in_off: node_count + 1 host offsets with in_off[0] == 0 (checked by the caller); parts >= 1; a part's targets
// go in chunks of about chunk_edges (>= 1) edges, at most 4096 chunks
inline std::vector<PrPart> pr_split(const uint32_t* in_off, uint32_t n, uint32_t parts, uint64_t chunk_edges) {
  const uint64_t m = in_off[n];
  const std::vector<uint32_t> rows = pr_row_cuts(in_off, 0, n, 0, m, parts);
  std::vector<PrPart> out(parts);
  uint64_t prev_end = 0;
  for (uint32_t u = 0; u < parts; ++u) {
    PrPart& q = out[u];
    q.r_begin = rows[u];
    q.r_end = rows[u + 1];
    q.e_begin = u == 0 ? 0 : std::min<uint64_t>(std::max<uint64_t>(in_off[q.r_begin], prev_end), m);
    q.e_end = u + 1 == parts ? m : std::min<uint64_t>(std::max<uint64_t>(in_off[q.r_end], q.e_begin), m);
    prev_end = q.e_end;
    const uint64_t len = q.e_end - q.e_begin;
    const uint32_t k = (uint32_t)std::min<uint64_t>(std::max<uint64_t>((len + chunk_edges - 1) / chunk_edges, 1), 4096);
    q.chunk_row = pr_row_cuts(in_off, q.r_begin, q.r_end, q.e_begin, q.e_end, k);
    q.chunk_edge.assign(k + 1, q.e_begin);
    q.chunk_edge[k] = q.e_end;
    for (uint32_t i = 1; i < k; ++i)
      q.chunk_edge[i] = std::min<uint64_t>(std::max<uint64_t>(in_off[q.chunk_row[i]], q.chunk_edge[i - 1]), q.e_end);
  }
  return out;
}

}  // namespace gb
