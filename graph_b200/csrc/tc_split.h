// tc_split.h — how gb_triangle_count_csr_u32 cuts a host undirected CSR into the chunks it uploads and counts
// one by one, kept free of CUDA so that it can be tested on the CPU.
//
// Chunk k holds the rows [row[k], row[k + 1]) and the entries [entry[k], entry[k + 1]) = [off[row[k]],
// off[row[k + 1]]): cuts fall at rows.  Chunks are cut greedily: each takes as many whole rows as fit in C
// entries, empty rows included, so every chunk holds at most C entries unless its one non-empty row is longer
// than C: such a hub stands alone, with only the empty rows next to it.  Every chunk but a lone chunk of an
// edgeless CSR holds at least one entry, and there are at most 2 ceil(m / C) + 1 chunks.
//
// Whatever the host array holds, the searches end inside [0, n] (wcc_first_row_past), every chunk takes at
// least one row, and the entry bounds are clamped into [0, m] and kept non-decreasing, so no copy leaves the
// host array; the device monotone check then fails the call before anything indexes with such offsets.
#pragma once

#include <algorithm>
#include <cstdint>
#include <vector>

#include "wcc_split.h"

namespace gb {

struct TcChunks {
  std::vector<uint32_t> row;    // [K + 1]: row[0] = 0, row[K] = n
  std::vector<uint64_t> entry;  // [K + 1]: entry[0] = 0, entry[K] = m
  uint32_t count() const { return (uint32_t)row.size() - 1; }
};

// off: node_count + 1 host offsets with off[0] == 0 (checked by the caller), n >= 1; chunk_entries >= 1
inline TcChunks tc_split(const uint32_t* off, uint32_t n, uint64_t chunk_entries) {
  const uint64_t m = off[n];
  TcChunks c;
  c.row.push_back(0);
  c.entry.push_back(0);
  uint32_t r = 0;
  uint64_t e = 0;
  // the last row boundary in [lo, n] whose offset is <= x, lo - 1 when there is none
  auto last_within = [&](uint32_t lo, uint64_t x) -> uint32_t {
    return (uint32_t)((uint64_t)lo + wcc_first_row_past(off + lo, n - lo + 1, x, true) - 1);
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
    c.entry.push_back(eb);
    r = b;
    e = eb;
  }
  return c;
}

}  // namespace gb
