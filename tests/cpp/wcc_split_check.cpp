// CPU check of the part split of gb_wcc_csr_multi_u32 (graph_b200/csrc/csr_split.h).  For every case and part
// count: the edge ranges partition [0, m) in order with cuts at multiples of 4; the row slices tile [0, n]
// (the first starts at 0, the last ends at n, each starts no later than the previous one ended and ends no
// earlier) and their checked rows cover [0, n) exactly once; and on monotone offsets every edge of a part lies
// inside that part's rows, with about n + 2P offsets uploaded in all.
#include <cstdint>
#include <cstdio>
#include <random>
#include <vector>

#include "csr_split.h"

static int failures = 0;
static long checked = 0;

#define EXPECT(cond, ...)                                    \
  do {                                                       \
    if (!(cond) && ++failures <= 20) {                       \
      std::printf("FAIL %s (P=%u): ", name, parts);          \
      std::printf(__VA_ARGS__);                              \
      std::printf("\n");                                     \
    }                                                        \
  } while (0)

static bool monotone(const std::vector<uint32_t>& off) {
  for (size_t i = 0; i + 1 < off.size(); ++i)
    if (off[i] > off[i + 1]) return false;
  return true;
}

static void check(const char* name, const std::vector<uint32_t>& off, uint32_t parts) {
  const uint32_t n = (uint32_t)off.size() - 1;
  const uint64_t m = off[n];
  const std::vector<gb::WccPartRange> s = gb::wcc_split(off.data(), n, parts);
  ++checked;
  EXPECT(s.size() == parts, "%zu parts", s.size());
  if (s.size() != parts) return;
  uint64_t uploaded = 0;
  std::vector<int> covered(n, 0);
  for (uint32_t p = 0; p < parts; ++p) {
    const gb::WccPartRange& r = s[p];
    EXPECT(r.e_begin == (p ? s[p - 1].e_end : 0), "part %u starts at edge %llu", p, (unsigned long long)r.e_begin);
    EXPECT(r.e_begin <= r.e_end && r.e_end <= m, "part %u edges [%llu, %llu)", p, (unsigned long long)r.e_begin,
           (unsigned long long)r.e_end);
    EXPECT(r.e_begin % 4 == 0, "part %u starts at edge %llu", p, (unsigned long long)r.e_begin);
    EXPECT(r.r_begin <= r.r_end && r.r_end <= n, "part %u rows [%u, %u]", p, r.r_begin, r.r_end);
    EXPECT(r.r_begin == (p ? std::min(r.r_begin, s[p - 1].r_end) : 0), "part %u starts at row %u after %u", p,
           r.r_begin, p ? s[p - 1].r_end : 0);
    EXPECT(r.check_begin == (p ? s[p - 1].r_end : 0), "part %u checks from row %u", p, r.check_begin);
    EXPECT(r.r_begin <= r.check_begin && r.check_begin <= r.r_end, "part %u checks [%u, %u) of [%u, %u]", p,
           r.check_begin, r.r_end, r.r_begin, r.r_end);
    for (uint32_t v = r.check_begin; v < r.r_end; ++v) ++covered[v];
    uploaded += r.r_end - r.r_begin + 1;
    if (monotone(off) && r.e_begin < r.e_end) {
      EXPECT(off[r.r_begin] <= r.e_begin && r.e_end <= off[r.r_end], "part %u edges [%llu, %llu) outside rows [%u, %u]",
             p, (unsigned long long)r.e_begin, (unsigned long long)r.e_end, r.r_begin, r.r_end);
    }
  }
  EXPECT(s.back().e_end == m, "edges end at %llu, m = %llu", (unsigned long long)s.back().e_end, (unsigned long long)m);
  EXPECT(s.back().r_end == n, "rows end at %u, n = %u", s.back().r_end, n);
  for (uint32_t v = 0; v < n; ++v) EXPECT(covered[v] == 1, "row %u checked %d times", v, covered[v]);
  if (monotone(off)) EXPECT(uploaded <= (uint64_t)n + 2 * parts, "%llu offsets uploaded", (unsigned long long)uploaded);
}

static std::vector<uint32_t> from_degrees(const std::vector<uint32_t>& deg) {
  std::vector<uint32_t> off(deg.size() + 1, 0);
  for (size_t i = 0; i < deg.size(); ++i) off[i + 1] = off[i] + deg[i];
  return off;
}

int main() {
  const uint32_t part_counts[] = {1, 2, 3, 4, 5, 8, 13, 16, 64};
  std::mt19937 rng(7);
  std::vector<std::pair<const char*, std::vector<uint32_t>>> cases;
  for (int t = 0; t < 20; ++t) {  // random degrees, some rows empty
    std::vector<uint32_t> deg(1 + rng() % 2000);
    for (auto& d : deg) d = rng() % 4 == 0 ? 0 : rng() % 40;
    cases.push_back({"random", from_degrees(deg)});
  }
  for (uint32_t m = 0; m < 40; ++m) {  // m < 4P for most part counts; m == 0
    std::vector<uint32_t> deg(1 + m % 7, 0);
    for (uint32_t e = 0; e < m; ++e) ++deg[rng() % deg.size()];
    cases.push_back({"few edges", from_degrees(deg)});
  }
  cases.push_back({"one node, no edge", {0, 0}});
  cases.push_back({"one node, self-loops", {0, 9}});
  {  // one hub row spanning every part, empty rows around it
    std::vector<uint32_t> deg(1000, 0);
    deg[500] = 100000;
    cases.push_back({"hub", from_degrees(deg)});
    deg[0] = 3;
    deg[999] = 5;
    cases.push_back({"hub between rows", from_degrees(deg)});
  }
  {  // all edges in the last two rows
    std::vector<uint32_t> deg(5000, 0);
    deg[4998] = 777;
    deg[4999] = 1234;
    cases.push_back({"last two rows", from_degrees(deg)});
  }
  {  // long runs of empty rows: edges only every 1000th row
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
    for (uint32_t parts : part_counts) check(c.first, c.second, parts);
  std::printf("wcc_split: %ld cases, %d failures\n", checked, failures);
  if (failures) return 1;
  std::printf("wcc_split ok\n");
  return 0;
}
