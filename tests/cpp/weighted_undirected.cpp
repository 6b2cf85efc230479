// UndirectedCsrGraph<u32, (), f32> through include/graph_b200.hpp: GraphBuilder::build_undirected_weighted,
// DirectedCsrGraph::to_undirected_weighted and UndirectedCsrGraph::neighbors_with_values.  argv[1] is tests/golden.
// Exits 0 and prints "weighted_undirected ok" when every check passes; prints the first failure otherwise.
#include <cstdio>
#include <cstring>
#include <string>
#include <tuple>
#include <vector>

#include "graph_b200.hpp"

using namespace graph::prelude;

#define EXPECT(cond)                                                \
  do {                                                              \
    if (!(cond)) {                                                  \
      std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); \
      return 1;                                                     \
    }                                                               \
  } while (0)

using Row = std::vector<std::pair<std::uint32_t, float>>;

static Row row_of(const UndirectedCsrGraph& g, std::uint32_t node) {
  Row r;
  auto [b, e] = g.neighbors_with_values(node);
  for (const Target* t = b; t != e; ++t) r.emplace_back(t->target, t->value);
  return r;
}

// every row, targets and values, of two graphs agree (values bit for bit)
static bool same_rows(const UndirectedCsrGraph& a, const UndirectedCsrGraph& b) {
  if (a.node_count() != b.node_count() || a.edge_count() != b.edge_count()) return false;
  for (std::uint32_t v = 0; v < a.node_count(); ++v) {
    Row x = row_of(a, v), y = row_of(b, v);
    if (x.size() != y.size()) return false;
    for (std::size_t i = 0; i < x.size(); ++i)
      if (x[i].first != y[i].first || std::memcmp(&x[i].second, &y[i].second, 4) != 0) return false;
  }
  return true;
}

template <typename F>
static int status_of(F&& f) {
  try {
    f();
  } catch (const graph::Error& e) {
    return e.status;
  }
  return GB_OK;
}

int main(int argc, char** argv) {
  if (argc < 2) {
    std::printf("usage: %s <tests/golden>\n", argv[0]);
    return 64;
  }
  const std::string dir = argv[1];
  try {
    // tests/golden/test.wel
    const std::vector<std::tuple<std::uint32_t, std::uint32_t, float>> wel = {
        {0, 1, 0.1f}, {0, 2, 0.2f}, {1, 2, 0.3f}, {1, 3, 0.4f}, {2, 4, 0.5f}, {3, 4, 0.6f}};
    {  // Unsorted: outgoing pass, then incoming pass, each in edge-list order
      UndirectedCsrGraph g = GraphBuilder().edges_with_values(wel).build_undirected_weighted();
      EXPECT(g.node_count() == 5 && g.edge_count() == 6);
      EXPECT((row_of(g, 1) == Row{{2, 0.3f}, {3, 0.4f}, {0, 0.1f}}));
      EXPECT((row_of(g, 2) == Row{{4, 0.5f}, {0, 0.2f}, {1, 0.3f}}));
      UndirectedCsrGraph f = GraphBuilder().with_values().path(dir + "/test.wel").build_undirected_weighted();
      EXPECT(same_rows(g, f));
    }
    {  // Sorted: rows ascending by target
      UndirectedCsrGraph g =
          GraphBuilder().csr_layout(CsrLayout::Sorted).edges_with_values(wel).build_undirected_weighted();
      EXPECT((row_of(g, 1) == Row{{0, 0.1f}, {2, 0.3f}, {3, 0.4f}}));
      EXPECT((row_of(g, 2) == Row{{0, 0.2f}, {1, 0.3f}, {4, 0.5f}}));
      // to_undirected_weighted: the out-CSR's entries in CSR order with their values
      DirectedCsrGraph d = GraphBuilder().edges_with_values(wel).build_directed();
      EXPECT(same_rows(d.to_undirected_weighted(CsrLayout::Sorted), g));
      // the unweighted conversion keeps its behaviour: same targets, no values
      UndirectedCsrGraph u = d.to_undirected(CsrLayout::Sorted);
      auto [b, e] = u.neighbors(1);
      EXPECT(e - b == 3 && b[0] == 0 && b[1] == 2 && b[2] == 3);
      EXPECT(status_of([&] { u.neighbors_with_values(1); }) == GB_ERR_INVALID);
    }
    {  // Deduplicated: the first value of each run of equal targets; self-loops removed
      UndirectedCsrGraph g = GraphBuilder()
                                 .csr_layout(CsrLayout::Deduplicated)
                                 .edges_with_values({{0, 1, 1.f}, {1, 0, 2.f}, {0, 0, 3.f}, {0, 1, 4.f}, {1, 2, 5.f}})
                                 .build_undirected_weighted();
      EXPECT((row_of(g, 0) == Row{{1, 1.f}}));
      EXPECT((row_of(g, 1) == Row{{0, 2.f}, {2, 5.f}}));
      EXPECT((row_of(g, 2) == Row{{1, 5.f}}));
      // make_degree_ordered needs EV: Ord, which f32 is not: refused, the graph unchanged
      EXPECT(status_of([&] { g.make_degree_ordered(); }) == GB_ERR_UNSUPPORTED);
      EXPECT((row_of(g, 1) == Row{{0, 2.f}, {2, 5.f}}));
    }
    {  // a binary file with Target<u32, f32> records keeps its rows and values as stored
      UndirectedCsrGraph g = GraphBuilder()
                                 .file_format(FileFormat::Binary)
                                 .with_values()
                                 .path(dir + "/binary_undirected_u32_values.bin")
                                 .build_undirected_weighted();
      EXPECT(g.node_count() == 4 && g.edge_count() == 6);
      float want = 0.f;
      for (std::uint32_t v = 0; v < 4; ++v)
        for (auto& [t, w] : row_of(g, v)) {
          (void)t;
          EXPECT(w == want);
          want += 0.25f;
        }
    }
    // a builder without values refuses, as does a binary file without values
    EXPECT(status_of([] { GraphBuilder().edges({{0, 1}}).build_undirected_weighted(); }) == GB_ERR_INVALID);
    EXPECT(status_of([&] {
             GraphBuilder().file_format(FileFormat::Binary).with_values().path(dir + "/binary_undirected_u32.bin")
                 .build_undirected_weighted();
           }) == GB_ERR_INVALID);
    // the unweighted build keeps ignoring the values it was given
    UndirectedCsrGraph plain = GraphBuilder().edges_with_values(wel).build_undirected();
    EXPECT(status_of([&] { plain.neighbors_with_values(0); }) == GB_ERR_INVALID);
  } catch (const graph::Error& e) {
    std::printf("graph::Error %d: %s\n", (int)e.status, e.what());
    return (int)e.status;
  }
  std::printf("weighted_undirected ok\n");
  return 0;
}
