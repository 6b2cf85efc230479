// CPU check of the send order of gb_sssp_csr_u32 (sssp_send_order, graph_b200/csrc/csr_split.h) over the chunks
// of tc_split.  For every case, chunk size and start: the order is a permutation of the chunks; its first chunk
// holds the start's row; it runs on from there and wraps round to chunk 0; and every prefix of it holds one
// cyclic interval of rows from the first chunk's first row, so that "row u has landed" is the distance from
// that row, modulo n, below the number of rows sent.  Cases: the start in the first, a middle and the last
// chunk, a hub chunk, n = 1 and m = 0.
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

#include "csr_split.h"

static int failures = 0;
static long checked = 0;

#define EXPECT(cond, ...)                                                                               \
  do {                                                                                                  \
    if (!(cond) && ++failures <= 20) {                                                                  \
      std::printf("FAIL %s (C=%llu, start=%u): ", name, (unsigned long long)chunk_entries, start);     \
      std::printf(__VA_ARGS__);                                                                         \
      std::printf("\n");                                                                                \
    }                                                                                                   \
  } while (0)

static void check(const char* name, const std::vector<uint32_t>& off, uint64_t chunk_entries, uint32_t start) {
  const uint32_t n = (uint32_t)off.size() - 1;
  const gb::CsrChunks c = gb::tc_split(off.data(), n, chunk_entries);
  const uint32_t K = c.count();
  const std::vector<uint32_t> order = gb::sssp_send_order(c, start);
  ++checked;
  EXPECT(order.size() == K, "%zu entries for %u chunks", order.size(), K);
  if (order.size() != K) return;
  const uint32_t ks = order[0];
  EXPECT(c.row[ks] <= start && start < c.row[ks + 1], "chunk %u holds rows [%u, %u)", ks, c.row[ks], c.row[ks + 1]);
  std::vector<int> seen(K, 0);
  for (uint32_t j = 0; j < K; ++j) {
    EXPECT(order[j] == (ks + j) % K, "order[%u] = %u", j, order[j]);
    if (order[j] < K) ++seen[order[j]];
  }
  for (uint32_t k = 0; k < K; ++k) EXPECT(seen[k] == 1, "chunk %u sent %d times", k, seen[k]);
  // the rows of the first j chunks, against the cyclic interval [first, first + span) modulo n
  const uint32_t first = c.row[ks];
  std::vector<char> landed(n, 0);
  for (uint32_t j = 1; j <= K; ++j) {
    const uint32_t k = order[j - 1];
    for (uint32_t v = c.row[k]; v < c.row[k + 1]; ++v) landed[v] = 1;
    uint32_t span = n;
    if (j < K) {
      const uint32_t stop = c.row[order[j]];
      span = stop > first ? stop - first : stop + (n - first);
    }
    for (uint32_t u = 0; u < n; ++u) {
      const bool in = (u >= first ? u - first : u + (n - first)) < span;
      EXPECT(in == (landed[u] != 0), "after %u chunks row %u: interval %d, landed %d", j, u, (int)in, landed[u]);
    }
  }
}

static std::vector<uint32_t> from_degrees(const std::vector<uint32_t>& deg) {
  std::vector<uint32_t> off(deg.size() + 1, 0);
  for (size_t i = 0; i < deg.size(); ++i) off[i + 1] = off[i] + deg[i];
  return off;
}

int main() {
  const uint64_t sizes[] = {1, 3, 16, 100, 1u << 20};
  std::mt19937 rng(7);
  std::vector<std::pair<const char*, std::vector<uint32_t>>> cases;
  for (int t = 0; t < 6; ++t) {  // random degrees, some rows empty
    std::vector<uint32_t> deg(1 + rng() % 400);
    for (auto& d : deg) d = rng() % 4 == 0 ? 0 : rng() % 20;
    cases.push_back({"random", from_degrees(deg)});
  }
  cases.push_back({"n = 1, no edge", {0, 0}});
  cases.push_back({"n = 1, self-loops", {0, 9}});
  cases.push_back({"m = 0", std::vector<uint32_t>(301, 0)});
  {  // a hub row longer than every chunk size but the last, empty and short rows around it
    std::vector<uint32_t> deg(300, 0);
    for (size_t i = 0; i < deg.size(); i += 3) deg[i] = 1 + rng() % 5;
    deg[150] = 5000;
    cases.push_back({"hub", from_degrees(deg)});
  }
  for (auto& cs : cases) {
    const uint32_t n = (uint32_t)cs.second.size() - 1;
    for (uint64_t chunk_entries : sizes) {
      const gb::CsrChunks c = gb::tc_split(cs.second.data(), n, chunk_entries);
      const uint32_t K = c.count();
      // the start in the first chunk, a middle one and the last, at the first and last row of each; the hub row
      std::vector<uint32_t> starts = {0, c.row[1] - 1, c.row[K / 2], c.row[K / 2 + 1] - 1, c.row[K - 1], n - 1};
      if (n > 150) starts.push_back(150);
      for (uint32_t s : starts) check(cs.first, cs.second, chunk_entries, s);
    }
  }
  {  // by hand: chunks {0..2}, {3} (a hub), {4, 5}; start 3 sends 1, 2, 0
    const std::vector<uint32_t> off = from_degrees({1, 2, 3, 50, 1, 1});
    const gb::CsrChunks c = gb::tc_split(off.data(), 6, 10);
    const char* name = "hub alone";
    const uint64_t chunk_entries = 10;
    const uint32_t start = 3;
    EXPECT(gb::sssp_send_order(c, 3) == (std::vector<uint32_t>{1, 2, 0}), "order");
    EXPECT(gb::sssp_send_order(c, 5) == (std::vector<uint32_t>{2, 0, 1}), "order from the last chunk");
    EXPECT(gb::sssp_send_order(c, 0) == (std::vector<uint32_t>{0, 1, 2}), "order from the first chunk");
    ++checked;
  }
  std::printf("sssp_send_order: %ld cases, %d failures\n", checked, failures);
  if (failures) return 1;
  std::printf("sssp_send_order ok\n");
  return 0;
}
