// CPU check of the chunk cut of gb_triangle_count_csr_u32 (graph_b200/csrc/csr_split.h).  For every case and
// chunk size C: the chunks cover the rows [0, n) exactly once, in order, each with at least one row; every
// boundary is row-aligned (edge[k] == off[row[k]]) and the entries end at m; a chunk holds at most C entries
// unless it has a single non-empty row (a hub longer than C), and every such hub stands alone; only an edgeless
// CSR has an empty chunk; no chunk could have taken the next row (the cut is greedy), so there are at most
// 2 ceil(m / C) + 1 chunks; and on offsets that are not monotone the cut still ends, with entry bounds
// non-decreasing inside [0, m].  Then the chunk size the triangle count and SSSP take (tc_chunk_entries): the
// default, a knob, a knob below ceil(m / 4096), and m = 0.
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

#include "csr_split.h"

static int failures = 0;
static long checked = 0;

#define EXPECT(cond, ...)                                                          \
  do {                                                                             \
    if (!(cond) && ++failures <= 20) {                                             \
      std::printf("FAIL %s (C=%llu): ", name, (unsigned long long)chunk_entries); \
      std::printf(__VA_ARGS__);                                                    \
      std::printf("\n");                                                           \
    }                                                                              \
  } while (0)

static bool monotone(const std::vector<uint32_t>& off) {
  for (size_t i = 0; i + 1 < off.size(); ++i)
    if (off[i] > off[i + 1]) return false;
  return true;
}

static void check(const char* name, const std::vector<uint32_t>& off, uint64_t chunk_entries) {
  const uint32_t n = (uint32_t)off.size() - 1;
  const uint64_t m = off[n];
  const gb::CsrChunks c = gb::tc_split(off.data(), n, chunk_entries);
  ++checked;
  const uint32_t K = c.count();
  EXPECT(c.row.size() == c.edge.size() && K >= 1, "%zu row bounds, %zu entry bounds", c.row.size(), c.edge.size());
  if (c.row.size() != c.edge.size() || K < 1) return;
  EXPECT(c.row[0] == 0 && c.row[K] == n, "rows [%u, %u), n = %u", c.row[0], c.row[K], n);
  EXPECT(c.edge[0] == 0 && c.edge[K] == m, "entries [%llu, %llu), m = %llu", (unsigned long long)c.edge[0],
         (unsigned long long)c.edge[K], (unsigned long long)m);
  std::vector<int> covered(n, 0);
  for (uint32_t k = 0; k < K; ++k) {
    EXPECT(c.row[k] < c.row[k + 1], "chunk %u rows [%u, %u)", k, c.row[k], c.row[k + 1]);
    EXPECT(c.edge[k] <= c.edge[k + 1] && c.edge[k + 1] <= m, "chunk %u entries [%llu, %llu)", k,
           (unsigned long long)c.edge[k], (unsigned long long)c.edge[k + 1]);
    for (uint32_t v = c.row[k]; v < c.row[k + 1] && v < n; ++v) ++covered[v];
    if (!monotone(off)) continue;
    EXPECT(c.edge[k] == off[c.row[k]], "chunk %u starts at entry %llu, row %u at %u", k,
           (unsigned long long)c.edge[k], c.row[k], off[c.row[k]]);
    const uint64_t len = c.edge[k + 1] - c.edge[k];
    uint32_t live = 0;  // rows with entries
    for (uint32_t v = c.row[k]; v < c.row[k + 1]; ++v) live += off[v + 1] > off[v];
    const bool single = live == 1;
    EXPECT(len <= chunk_entries || single, "chunk %u: %llu entries over %u rows", k, (unsigned long long)len, live);
    for (uint32_t v = c.row[k]; v < c.row[k + 1]; ++v)  // a hub stands alone
      EXPECT(off[v + 1] - off[v] <= chunk_entries || single, "hub row %u shares chunk %u", v, k);
    if (k + 1 < K)  // greedy: the next row did not fit
      EXPECT(off[c.row[k + 1] + 1] - off[c.row[k]] > chunk_entries, "chunk %u could have taken row %u", k,
             c.row[k + 1]);
    EXPECT(len > 0 || K == 1, "chunk %u of %u is empty", k, K);
  }
  for (uint32_t v = 0; v < n; ++v) EXPECT(covered[v] == 1, "row %u covered %d times", v, covered[v]);
  if (monotone(off))
    EXPECT(K <= 2 * ((m + chunk_entries - 1) / chunk_entries) + 1, "%u chunks for m = %llu", K,
           (unsigned long long)m);
}

static std::vector<uint32_t> from_degrees(const std::vector<uint32_t>& deg) {
  std::vector<uint32_t> off(deg.size() + 1, 0);
  for (size_t i = 0; i < deg.size(); ++i) off[i + 1] = off[i] + deg[i];
  return off;
}

int main() {
  const uint64_t sizes[] = {1, 2, 3, 7, 16, 100, 1000, 1u << 20};
  std::mt19937 rng(11);
  std::vector<std::pair<const char*, std::vector<uint32_t>>> cases;
  for (int t = 0; t < 20; ++t) {  // random degrees, some rows empty
    std::vector<uint32_t> deg(1 + rng() % 2000);
    for (auto& d : deg) d = rng() % 4 == 0 ? 0 : rng() % 40;
    cases.push_back({"random", from_degrees(deg)});
  }
  cases.push_back({"one node, no edge", {0, 0}});
  cases.push_back({"one node, self-loops", {0, 9}});
  cases.push_back({"no edges", std::vector<uint32_t>(1001, 0)});
  {  // empty rows at both ends
    std::vector<uint32_t> deg(300, 0);
    for (size_t i = 100; i < 200; ++i) deg[i] = 1 + rng() % 9;
    cases.push_back({"empty rows at both ends", from_degrees(deg)});
  }
  {  // one hub row longer than every chunk size but the last, empty rows around it
    std::vector<uint32_t> deg(1000, 0);
    deg[500] = 100000;
    cases.push_back({"hub", from_degrees(deg)});
    for (size_t i = 0; i < deg.size(); i += 3) deg[i] = 1 + rng() % 5;
    cases.push_back({"hub between rows", from_degrees(deg)});
    deg.assign(50, 2);
    deg[0] = 5000;
    deg[49] = 7000;
    cases.push_back({"hubs first and last", from_degrees(deg)});
  }
  {  // long runs of empty rows: entries only every 1000th row
    std::vector<uint32_t> deg(20000, 0);
    for (size_t i = 0; i < deg.size(); i += 1000) deg[i] = 4 + rng() % 64;
    cases.push_back({"runs of empty rows", from_degrees(deg)});
  }
  for (int t = 0; t < 20; ++t) {  // offsets that are not monotone
    std::vector<uint32_t> deg(1 + rng() % 3000);
    for (auto& d : deg) d = rng() % 30;
    std::vector<uint32_t> off = from_degrees(deg);
    const uint32_t n = (uint32_t)off.size() - 1;
    for (int k = 0; k < 1 + t % 4; ++k) {
      const uint32_t v = 1 + rng() % n;  // off[0] stays 0
      off[v] = t % 2 ? (uint32_t)rng() : off[v] / 3;
    }
    if (t == 0) off[n] = 0;  // offsets[n] = m = 0 below interior offsets
    cases.push_back({"not monotone", off});
  }
  for (auto& c : cases)
    for (uint64_t chunk_entries : sizes) check(c.first, c.second, chunk_entries);
  {  // the hub stands alone, with the rows before and after it in chunks of their own
    std::vector<uint32_t> deg = {1, 2, 3, 50, 1, 1};
    const std::vector<uint32_t> off = from_degrees(deg);
    const gb::CsrChunks c = gb::tc_split(off.data(), 6, 10);
    const char* name = "hub alone";
    const uint64_t chunk_entries = 10;
    EXPECT(c.row == (std::vector<uint32_t>{0, 3, 4, 6}), "rows %zu bounds", c.row.size());
    EXPECT(c.edge == (std::vector<uint64_t>{0, 6, 56, 58}), "entries %zu bounds", c.edge.size());
    ++checked;
  }
  {  // the chunk size: the knob when set, else ceil(m / 16) but at least 2^20; never below ceil(m / 4096)
    const char* name = "tc_chunk_entries";
    const uint64_t chunk_entries = 0;
    const uint64_t M = 1ull << 20;
    struct Rule { uint64_t m, knob, want; };
    const Rule rules[] = {
        {0, 0, M},                                     // m = 0: the floor
        {0, 5, 5},                                     // m = 0, knob set
        {1000, 0, M},                                  // small m: the floor
        {16 * M, 0, M},                                // ceil(m / 16) == 2^20
        {16 * M + 1, 0, M + 1},                        // ceil(m / 16) above the floor
        {0xFFFFFFFFull, 0, 0x10000000ull},             // the largest m: ceil(m / 16)
        {1000, 7, 7},                                  // the knob, below the default
        {1000, 3 * M, 3 * M},                          // the knob, above the default
        {4096 * 100, 50, 100},                         // the knob below ceil(m / 4096)
        {4096 * 100 + 1, 100, 101},                    // ... by a rounding
        {4096 * 100, 100, 100},                        // the knob at ceil(m / 4096)
    };
    for (const Rule& r : rules) {
      const uint64_t got = gb::tc_chunk_entries(r.m, r.knob);
      EXPECT(got == r.want, "m = %llu, knob = %llu: %llu, want %llu", (unsigned long long)r.m,
             (unsigned long long)r.knob, (unsigned long long)got, (unsigned long long)r.want);
      ++checked;
    }
  }
  std::printf("tc_split: %ld cases, %d failures\n", checked, failures);
  if (failures) return 1;
  std::printf("tc_split ok\n");
  return 0;
}
