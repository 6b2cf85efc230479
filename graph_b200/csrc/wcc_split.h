// wcc_split.h — how gb_wcc_csr_multi_u32 cuts a host out-CSR into parts, kept free of CUDA so that it can be
// tested on the CPU.
//
// Part p of P takes the edges [E_p, E_{p+1}), E_p = floor(m p / P) rounded down to a multiple of 4 (E_P = m):
// cuts fall at edges, not rows, as the chunks of gb_wcc_csr_u32 do, and a part may be empty.  It uploads the
// offsets of the rows its edges touch, offsets[r_begin .. r_end] (r_end - r_begin + 1 entries), about n + 2P
// entries over all parts.  Whatever the host array holds, the slices tile [0, n]: slice 0 starts at 0, the
// last ends at n, every slice starts no later than where the previous one ended and ends no earlier.  So each
// row v < n is checked for offsets[v] <= offsets[v + 1] by exactly one part, the one whose rows
// [check_begin, r_end) hold it, even when non-monotone offsets misled the binary searches below; and when the
// offsets are monotone, offsets[r_begin] <= E_p and E_{p+1} <= offsets[r_end].
#pragma once

#include <algorithm>
#include <cstdint>
#include <vector>

namespace gb {

struct WccPartRange {
  uint64_t e_begin, e_end;     // edges [e_begin, e_end)
  uint32_t r_begin, r_end;     // offsets[r_begin .. r_end] go to the device; rows r_begin .. r_end - 1
  uint32_t check_begin;        // this part checks rows [check_begin, r_end) (the previous part's r_end)
};

// The first i in [0, n] with off[i] > e (strict) or off[i] >= e, n when there is none.  On monotone offsets
// these are upper_bound and lower_bound; on any others the search still ends, inside [0, n], after at most
// log2(n + 1) + 1 probes, so the split needs nothing of the host array beyond off[0] == 0.
inline uint32_t wcc_first_row_past(const uint32_t* off, uint32_t n, uint64_t e, bool strict) {
  uint32_t lo = 0, hi = n;  // the answer lies in [lo, hi]
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2;
    if (strict ? off[mid] > e : off[mid] >= e) hi = mid;
    else lo = mid + 1;
  }
  return lo;
}

// off: node_count + 1 host offsets with off[0] == 0 (checked by the caller); parts >= 1
inline std::vector<WccPartRange> wcc_split(const uint32_t* off, uint32_t n, uint32_t parts) {
  const uint64_t m = off[n];
  std::vector<WccPartRange> out(parts);
  uint32_t prev_end = 0;
  for (uint32_t p = 0; p < parts; ++p) {
    WccPartRange& r = out[p];
    r.e_begin = (m * p / parts) & ~3ull;
    r.e_end = p + 1 == parts ? m : (m * (p + 1) / parts) & ~3ull;
    // the last row that starts at or before e_begin, and the first row boundary at or after e_end
    const uint32_t lo = wcc_first_row_past(off, n, r.e_begin, true);
    const uint32_t first = lo > 0 ? lo - 1 : 0;
    const uint32_t last = wcc_first_row_past(off, n, r.e_end, false);
    r.r_begin = p == 0 ? 0 : std::min(first, prev_end);
    r.r_end = p + 1 == parts ? n : std::max(last, prev_end);
    r.check_begin = prev_end;
    prev_end = r.r_end;
  }
  return out;
}

}  // namespace gb
