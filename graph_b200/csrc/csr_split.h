// csr_split.h — how the one-shot calls cut a host CSR into the slices and chunks they stream to the device
// (CsrFeed, common.cuh), kept free of CUDA so that it can be tested on the CPU.  Each call has its own rule,
// because each consumer may start on a chunk at a different point: WCC links any edge at once, PageRank needs
// whole rows, and triangle count needs every earlier row as well.
//
// Every rule needs nothing of the host offsets beyond off[0] == 0 (checked by the caller): whatever they hold,
// the searches end inside their ranges, the row slices tile [0, n] (so the device monotone check sees each row
// exactly once) and every edge bound is clamped into [0, m], so that no copy leaves the host array or its
// device buffer.  The device check then fails the call before anything indexes with bad offsets.
#pragma once

#include <algorithm>
#include <cstdint>
#include <vector>

namespace gb {

// The first i in [0, n] with off[i] > e (strict) or off[i] >= e, n when there is none.  On monotone offsets
// these are upper_bound and lower_bound; on any others the search still ends, inside [0, n], after at most
// log2(n + 1) + 1 probes.
inline uint32_t first_row_past(const uint32_t* off, uint32_t n, uint64_t e, bool strict) {
  uint32_t lo = 0, hi = n;  // the answer lies in [lo, hi]
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (strict ? off[mid] > e : off[mid] >= e) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

// Row-aligned chunks: chunk k holds the rows [row[k], row[k + 1]) and the edges [edge[k], edge[k + 1])
struct CsrChunks {
  std::vector<uint32_t> row;   // [K + 1]
  std::vector<uint64_t> edge;  // [K + 1]
  uint32_t count() const { return (uint32_t)row.size() - 1; }
};

// ---- WCC (gb_wcc_csr_u32, gb_wcc_csr_multi_u32): edge-cut parts ---------------------------------------------
// Part p of P takes the edges [E_p, E_{p+1}), E_p = floor(m p / P) rounded down to a multiple of 4 (E_P = m):
// cuts fall at edges, not rows, as the chunks of gb_wcc_csr_u32 do, and a part may be empty.  It uploads the
// offsets of the rows its edges touch, offsets[r_begin .. r_end] (r_end - r_begin + 1 entries), about n + 2P
// entries over all parts.  Slice 0 starts at 0, the last ends at n, every slice starts no later than where the
// previous one ended and ends no earlier.  So each row v < n is checked by exactly one part, the one whose rows
// [check_begin, r_end) hold it; and when the offsets are monotone, offsets[r_begin] <= E_p and
// E_{p+1} <= offsets[r_end].
struct WccPartRange {
  uint64_t e_begin, e_end;     // edges [e_begin, e_end)
  uint32_t r_begin, r_end;     // offsets[r_begin .. r_end] go to the device; rows r_begin .. r_end - 1
  uint32_t check_begin;        // this part checks rows [check_begin, r_end) (the previous part's r_end)
};

// off: node_count + 1 host offsets with off[0] == 0; parts >= 1
inline std::vector<WccPartRange> wcc_split(const uint32_t* off, uint32_t n, uint32_t parts) {
  const uint64_t m = off[n];
  std::vector<WccPartRange> out(parts);
  uint32_t prev_end = 0;
  for (uint32_t p = 0; p < parts; ++p) {
    WccPartRange& r = out[p];
    r.e_begin = (m * p / parts) & ~3ull;
    r.e_end = p + 1 == parts ? m : (m * (p + 1) / parts) & ~3ull;
    // the last row that starts at or before e_begin, and the first row boundary at or after e_end
    const uint32_t lo = first_row_past(off, n, r.e_begin, true);
    const uint32_t first = lo > 0 ? lo - 1 : 0;
    const uint32_t last = first_row_past(off, n, r.e_end, false);
    r.r_begin = p == 0 ? 0 : std::min(first, prev_end);
    r.r_end = p + 1 == parts ? n : std::max(last, prev_end);
    r.check_begin = prev_end;
    prev_end = r.r_end;
  }
  return out;
}

// ---- PageRank (gb_page_rank_csr_u32, gb_page_rank_csr_multi_u32, gb_pr_shards_csr_u32): equal-edge row parts
// Part u of U takes the rows [R_u, R_{u+1}), R_0 = 0, R_U = n, where R_u is the first row whose offset reaches
// floor(m u / U): cuts fall at rows, so a part holds at most about m / U edges plus one row, and a hub longer
// than m / U leaves parts empty.  The part uploads in_off[R_u .. R_{u+1}], out_off[R_u .. R_{u+1}] and the
// targets [E_u, E_{u+1}), E_u = in_off[R_u], in row-aligned chunks cut the same way (gb_page_rank_csr_u32 is
// the one-part case).  Beyond the probes of the searches the split reads in_off[n] only.
struct PrPart {
  uint32_t r_begin = 0, r_end = 0;   // rows [r_begin, r_end): offsets [r_begin .. r_end] go to the device
  uint64_t e_begin = 0, e_end = 0;   // targets [e_begin, e_end)
  CsrChunks chunks;                  // tile [r_begin, r_end) and [e_begin, e_end)
};

// rows [r0, r1] cut into k slices of about equal edge counts: cut i (0 < i < k) is the first row in [r0, r1]
// whose offset reaches e0 + (e1 - e0) i / k, and no earlier than cut i - 1
inline std::vector<uint32_t> pr_row_cuts(const uint32_t* off, uint32_t r0, uint32_t r1, uint64_t e0, uint64_t e1,
                                         uint32_t k) {
  std::vector<uint32_t> cut(k + 1, r0);
  cut[k] = r1;
  for (uint32_t i = 1; i < k; ++i) {
    const uint64_t want = e0 + (e1 - e0) * i / k;
    cut[i] = std::max(cut[i - 1], r0 + first_row_past(off + r0, r1 - r0, want, false));
  }
  return cut;
}

// in_off: node_count + 1 host offsets with in_off[0] == 0; parts >= 1; a part's targets go in chunks of about
// chunk_edges (>= 1) edges, at most 4096 chunks
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
    CsrChunks& c = q.chunks;
    c.row = pr_row_cuts(in_off, q.r_begin, q.r_end, q.e_begin, q.e_end, k);
    c.edge.assign(k + 1, q.e_begin);
    c.edge[k] = q.e_end;
    for (uint32_t i = 1; i < k; ++i)
      c.edge[i] = std::min<uint64_t>(std::max<uint64_t>(in_off[c.row[i]], c.edge[i - 1]), q.e_end);
  }
  return out;
}

// ---- triangle count (gb_triangle_count_csr_u32): greedy chunks ------------------------------------------------
// Chunk k holds the rows [row[k], row[k + 1]) and the entries [edge[k], edge[k + 1]) = [off[row[k]],
// off[row[k + 1]]), row[0] = 0, row[K] = n: cuts fall at rows.  Each chunk takes as many whole rows as fit in C
// entries, empty rows included, so every chunk holds at most C entries unless its one non-empty row is longer
// than C: such a hub stands alone, with only the empty rows next to it.  Every chunk but a lone chunk of an
// edgeless CSR holds at least one entry, every chunk takes at least one row, and there are at most
// 2 ceil(m / C) + 1 chunks.
// off: node_count + 1 host offsets with off[0] == 0, n >= 1; chunk_entries >= 1
inline CsrChunks tc_split(const uint32_t* off, uint32_t n, uint64_t chunk_entries) {
  const uint64_t m = off[n];
  CsrChunks c;
  c.row.push_back(0);
  c.edge.push_back(0);
  uint32_t r = 0;
  uint64_t e = 0;
  // the last row boundary in [lo, n] whose offset is <= x, lo - 1 when there is none
  auto last_within = [&](uint32_t lo, uint64_t x) -> uint32_t {
    return (uint32_t)((uint64_t)lo + first_row_past(off + lo, n - lo + 1, x, true) - 1);
  };
  while (r < n) {
    // p: the last row boundary within C entries of off[r]
    const uint32_t p = std::max(r, last_within(r + 1, (uint64_t)off[r] + chunk_entries));
    uint32_t b = p;
    if (p < n && off[p] == off[r]) {
      // rows [r, p) are empty and row p is longer than C: a hub.  It takes the empty rows around it, so that
      // no chunk is left without entries
      b = std::max(p + 1, last_within(p + 1, off[p + 1]));
    }
    const uint64_t eb = b == n ? m : std::min<uint64_t>(std::max<uint64_t>(off[b], e), m);
    c.row.push_back(b);
    c.edge.push_back(eb);
    r = b;
    e = eb;
  }
  return c;
}

}  // namespace gb
