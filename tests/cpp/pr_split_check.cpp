// CPU check of the part split of gb_page_rank_csr_multi_u32 / gb_pr_shards_csr_u32 (graph_b200/csrc/csr_split.h).
// For every case and part count U = 1..8: the row slices tile [0, n] in order, so every row is checked by
// exactly one part; each part's chunks tile its rows and its edges; every bound stays inside [0, m] and inside
// its part, on malformed offsets too; and on monotone offsets the parts cut at rows, their edge ranges are the
// rows' edges and tile [0, m], each part holds at most ceil(m / U) edges plus one row, and the cuts are the
// first rows whose offsets reach floor(m u / U).  The one-part split of gb_page_rank_csr_u32, cut into
// ceil(m / c) edges per chunk, yields at most min(c, 4096) chunks.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

#include "csr_split.h"

static int failures = 0;
static long checked = 0;

#define EXPECT(cond, ...)                                      \
  do {                                                         \
    if (!(cond) && ++failures <= 20) {                         \
      std::printf("FAIL %s (U=%u, C=%llu): ", name, parts,    \
                  (unsigned long long)chunk);                  \
      std::printf(__VA_ARGS__);                                \
      std::printf("\n");                                       \
    }                                                          \
  } while (0)

static bool monotone(const std::vector<uint32_t>& off) {
  for (size_t i = 0; i + 1 < off.size(); ++i)
    if (off[i] > off[i + 1]) return false;
  return true;
}

static void check(const char* name, const std::vector<uint32_t>& off, uint32_t parts, uint64_t chunk) {
  const uint32_t n = (uint32_t)off.size() - 1;
  const uint64_t m = off[n];
  const bool mono = monotone(off);
  const std::vector<gb::PrPart> s = gb::pr_split(off.data(), n, parts, chunk);
  ++checked;
  EXPECT(s.size() == parts, "%zu parts", s.size());
  if (s.size() != parts) return;
  std::vector<int> checks(n, 0);
  for (uint32_t u = 0; u < parts; ++u) {
    const gb::PrPart& q = s[u];
    EXPECT(q.r_begin == (u ? s[u - 1].r_end : 0), "part %u starts at row %u", u, q.r_begin);
    EXPECT(q.r_begin <= q.r_end && q.r_end <= n, "part %u rows [%u, %u)", u, q.r_begin, q.r_end);
    EXPECT(q.e_begin <= q.e_end && q.e_end <= m, "part %u edges [%llu, %llu)", u, (unsigned long long)q.e_begin,
           (unsigned long long)q.e_end);
    EXPECT(q.e_begin == (u ? s[u - 1].e_end : 0), "part %u starts at edge %llu", u, (unsigned long long)q.e_begin);
    for (uint32_t v = q.r_begin; v < q.r_end && v < n; ++v) ++checks[v];
    // chunks: rows and edges tile the part's, in order, inside it
    const size_t K = q.chunks.row.size() - 1;
    EXPECT(K >= 1 && q.chunks.edge.size() == K + 1, "part %u has %zu chunks", u, K);
    if (K < 1 || q.chunks.edge.size() != K + 1) continue;
    EXPECT(q.chunks.row[0] == q.r_begin && q.chunks.row[K] == q.r_end, "part %u chunk rows [%u, %u]", u,
           q.chunks.row[0], q.chunks.row[K]);
    EXPECT(q.chunks.edge[0] == q.e_begin && q.chunks.edge[K] == q.e_end, "part %u chunk edges", u);
    for (size_t k = 0; k < K; ++k) {
      EXPECT(q.chunks.row[k] <= q.chunks.row[k + 1], "part %u chunk %zu rows [%u, %u)", u, k, q.chunks.row[k],
             q.chunks.row[k + 1]);
      EXPECT(q.chunks.edge[k] <= q.chunks.edge[k + 1], "part %u chunk %zu edges", u, k);
      if (mono)  // a chunk's edges are its rows' edges
        EXPECT(q.chunks.edge[k] == off[q.chunks.row[k]] && q.chunks.edge[k + 1] == off[q.chunks.row[k + 1]],
               "part %u chunk %zu edges [%llu, %llu) of rows [%u, %u)", u, k, (unsigned long long)q.chunks.edge[k],
               (unsigned long long)q.chunks.edge[k + 1], q.chunks.row[k], q.chunks.row[k + 1]);
    }
    if (!mono) continue;
    EXPECT(q.e_begin == off[q.r_begin] && q.e_end == off[q.r_end], "part %u edges [%llu, %llu) of rows [%u, %u)", u,
           (unsigned long long)q.e_begin, (unsigned long long)q.e_end, q.r_begin, q.r_end);
    if (u > 0) {  // the first row whose offset reaches floor(m u / U)
      const uint64_t want = m * u / parts;
      EXPECT(off[q.r_begin] >= want && (q.r_begin == 0 || off[q.r_begin - 1] < want),
             "part %u starts at row %u (offset %u) for edge %llu", u, q.r_begin, off[q.r_begin],
             (unsigned long long)want);
    }
    uint64_t longest = 0;
    for (uint32_t v = q.r_begin; v < q.r_end; ++v) longest = std::max<uint64_t>(longest, off[v + 1] - off[v]);
    EXPECT(q.e_end - q.e_begin <= (m + parts - 1) / parts + longest, "part %u holds %llu edges (m %llu, row %llu)",
           u, (unsigned long long)(q.e_end - q.e_begin), (unsigned long long)m, (unsigned long long)longest);
    const size_t want_chunks = std::min<uint64_t>(std::max<uint64_t>((q.e_end - q.e_begin + chunk - 1) / chunk, 1), 4096);
    EXPECT(K == want_chunks, "part %u: %zu chunks for %llu edges", u, K, (unsigned long long)(q.e_end - q.e_begin));
  }
  EXPECT(s[parts - 1].r_end == n && s[parts - 1].e_end == m, "the last part ends at row %u, edge %llu",
         s[parts - 1].r_end, (unsigned long long)s[parts - 1].e_end);
  for (uint32_t v = 0; v < n; ++v) EXPECT(checks[v] == 1, "row %u is checked %d times", v, checks[v]);
}

static std::vector<uint32_t> from_degrees(const std::vector<uint32_t>& deg) {
  std::vector<uint32_t> off(deg.size() + 1, 0);
  for (size_t i = 0; i < deg.size(); ++i) off[i + 1] = off[i] + deg[i];
  return off;
}

// gb_page_rank_csr_u32's split: one part in chunks of ceil(m / c) edges (at least 1) for c chunks asked, which
// must come out as at most min(c, 4096) chunks that tile [0, n] and [0, m]
static void one_device(const char* name, const std::vector<uint32_t>& off) {
  const uint32_t n = (uint32_t)off.size() - 1, parts = 1;
  const uint64_t m = off[n];
  for (uint64_t c : {1ull, 3ull, 7ull, 16ull, 5000ull}) {
    const uint64_t chunk = std::max<uint64_t>((m + c - 1) / c, 1);
    check(name, off, parts, chunk);
    const size_t K = gb::pr_split(off.data(), n, parts, chunk)[0].chunks.row.size() - 1;
    EXPECT(K <= std::min<uint64_t>(c, 4096), "%zu chunks for %llu asked", K, (unsigned long long)c);
  }
}

static void all_parts(const char* name, const std::vector<uint32_t>& off) {
  for (uint64_t chunk : {1ull, 3ull, 64ull, 1ull << 23})
    for (uint32_t parts = 1; parts <= 8; ++parts) check(name, off, parts, chunk);
  one_device(name, off);
}

int main() {
  std::mt19937_64 rng(12345);
  // random degrees, sparse and dense
  for (int t = 0; t < 40; ++t) {
    const uint32_t n = 1 + (uint32_t)(rng() % 3000);
    std::vector<uint32_t> deg(n);
    const uint32_t top = t % 2 ? 3 : 40;
    for (auto& d : deg) d = (uint32_t)(rng() % top);
    all_parts("random", from_degrees(deg));
  }
  // tiny: n = 1..6 with every degree pattern of 0..2 per row
  for (uint32_t n = 1; n <= 6; ++n) {
    uint32_t combos = 1;
    for (uint32_t i = 0; i < n; ++i) combos *= 3;
    for (uint32_t c = 0; c < combos; ++c) {
      std::vector<uint32_t> deg(n);
      uint32_t x = c;
      for (auto& d : deg) {
        d = x % 3;
        x /= 3;
      }
      all_parts("tiny", from_degrees(deg));
    }
  }
  // hub-heavy: one row longer than m / U (empty parts), hubs at the ends, two hubs
  for (uint32_t at : {0u, 1u, 500u, 998u, 999u}) {
    std::vector<uint32_t> deg(1000, 1);
    deg[at] = 100000;
    all_parts("hub", from_degrees(deg));
    deg.assign(1000, 0);
    deg[at] = 7;
    all_parts("lone row", from_degrees(deg));
  }
  {
    std::vector<uint32_t> deg(4000, 0);
    deg[10] = 50000;
    deg[3000] = 50000;
    for (uint32_t i = 100; i < 200; ++i) deg[i] = 3;
    all_parts("two hubs", from_degrees(deg));
  }
  // all empty
  for (uint32_t n : {1u, 2u, 31u, 1000u}) all_parts("empty", std::vector<uint32_t>(n + 1, 0));
  // non-monotone offsets (off[0] == 0 as the caller checks): random values, a decreasing run, a spike
  for (int t = 0; t < 60; ++t) {
    const uint32_t n = 1 + (uint32_t)(rng() % 500);
    std::vector<uint32_t> off(n + 1);
    off[0] = 0;
    for (uint32_t i = 1; i <= n; ++i) off[i] = (uint32_t)(rng() % (t % 3 == 0 ? 0xFFFFFFFFull : 2000));
    all_parts("non-monotone", off);
    std::vector<uint32_t> deg(n, 4);
    std::vector<uint32_t> good = from_degrees(deg);
    const uint32_t at = 1 + (uint32_t)(rng() % n);
    good[at] = t % 2 ? 0xFFFFFFF0u : 0u;
    all_parts("spike", good);
  }
  {
    std::vector<uint32_t> off(1001);
    off[0] = 0;
    for (uint32_t i = 1; i <= 1000; ++i) off[i] = 5000 - 5 * i;
    all_parts("decreasing", off);
  }
  if (failures) {
    std::printf("%d failures in %ld splits\n", failures, checked);
    return 1;
  }
  std::printf("pr_split ok: %ld splits\n", checked);
  return 0;
}
