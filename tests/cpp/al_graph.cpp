// DirectedALGraph / UndirectedALGraph through include/graph_b200.hpp: the reference's adj_list.rs unit tests
// (adj_list.rs:783-1051) and its crate doc-test (lib.rs:234-255), through GraphBuilder::build_directed_al /
// build_undirected_al, add_edge, add_edge_with_value, the MissingNode error, to_csr() and the algorithm overloads.
// Exits 0 and prints "al_graph ok" when every check passes; prints the first failure otherwise.
#include <cstdio>
#include <cstring>
#include <functional>
#include <string>
#include <thread>
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

using V = std::vector<std::uint32_t>;
using Edges = std::vector<std::pair<std::uint32_t, std::uint32_t>>;

static bool same(const std::vector<Target>& a, const std::vector<std::pair<std::uint32_t, float>>& b) {
  if (a.size() != b.size()) return false;
  for (std::size_t i = 0; i < a.size(); ++i)
    if (a[i].target != b[i].first || std::memcmp(&a[i].value, &b[i].second, 4) != 0) return false;
  return true;
}

static bool missing_node(const std::function<void()>& f, const std::string& node) {
  try {
    f();
  } catch (const graph::Error& e) {
    return e.status == GB_ERR_INVALID &&
           std::string(e.what()).rfind("node \"" + node + "\" does not exist in the graph", 0) == 0;
  }
  return false;
}

template <typename G>
static G build(CsrLayout layout, const Edges& e);
template <>
DirectedALGraph build(CsrLayout layout, const Edges& e) {
  return GraphBuilder().csr_layout(layout).edges(e).build_directed_al();
}
template <>
UndirectedALGraph build(CsrLayout layout, const Edges& e) {
  return GraphBuilder().csr_layout(layout).edges(e).build_undirected_al();
}
static V row0(const DirectedALGraph& g, std::uint32_t n) { return g.out_neighbors(n); }
static V row0(const UndirectedALGraph& g, std::uint32_t n) { return g.neighbors(n); }

// adj_list.rs:811-853, 882-908 (directed) and 910-959, 996-1022 (undirected)
template <typename G>
static int add_edge_cases(bool directed) {
  G g = build<G>(CsrLayout::Unsorted, {{0, 2}, {1, 2}});
  EXPECT(row0(g, 0) == V({2}));
  g.add_edge(0, 1);
  EXPECT(row0(g, 0) == V({2, 1}));
  if (!directed) EXPECT(row0(g, 1) == V({2, 0}));
  g.add_edge(0, 2);
  EXPECT(row0(g, 0) == V({2, 1, 2}));
  EXPECT(missing_node([&] { g.add_edge(0, 3); }, "3"));
  EXPECT(row0(g, 0) == V({2, 1, 2}));

  G s = build<G>(CsrLayout::Sorted, {{0, 2}, {1, 2}});
  s.add_edge(0, 1);
  EXPECT(row0(s, 0) == V({1, 2}));
  if (!directed) EXPECT(row0(s, 1) == V({0, 2}));
  s.add_edge(0, 1);
  EXPECT(row0(s, 0) == V({1, 1, 2}));

  G d = build<G>(CsrLayout::Deduplicated, {{0, 2}, {1, 2}, {1, 3}});
  EXPECT(row0(d, 0) == V({2}));
  if (!directed) EXPECT(row0(d, 1) == V({2, 3}));
  d.add_edge(0, 1);
  EXPECT(row0(d, 0) == V({1, 2}));
  if (!directed) EXPECT(row0(d, 1) == V({0, 2, 3}));
  d.add_edge(0, 1);
  EXPECT(row0(d, 0) == V({1, 2}));
  d.add_edge(0, 3);
  EXPECT(row0(d, 0) == V({1, 2, 3}));

  G p = build<G>(CsrLayout::Unsorted, {{0, 1}, {0, 2}, {0, 3}});
  std::vector<std::thread> ts;
  for (int i = 0; i < 4; ++i) ts.emplace_back([&] { p.add_edge(0, 1); });
  for (auto& t : ts) t.join();
  EXPECT(p.edge_count() == 7);
  return 0;
}

int main() {
  // adj_list.rs:783-796
  DirectedALGraph g = GraphBuilder().csr_layout(CsrLayout::Sorted).edges({{0, 1}, {0, 2}, {1, 2}}).build_directed_al();
  EXPECT(g.node_count() == 3 && g.edge_count() == 3);
  EXPECT(g.out_degree(0) == 2 && g.out_neighbors(0) == V({1, 2}));
  EXPECT(g.in_degree(2) == 2 && g.in_neighbors(2) == V({0, 1}));
  // adj_list.rs:1023-1051
  UndirectedALGraph u = GraphBuilder().csr_layout(CsrLayout::Sorted).edges({{0, 1}, {0, 2}, {1, 2}}).build_undirected_al();
  EXPECT(u.node_count() == 3 && u.edge_count() == 3);
  EXPECT(u.degree(0) == 2 && u.degree(2) == 2);
  EXPECT(u.neighbors(0) == V({1, 2}) && u.neighbors(2) == V({0, 1}));
  UndirectedALGraph c = GraphBuilder().csr_layout(CsrLayout::Sorted).edges({{0, 1}, {1, 0}}).build_undirected_al();
  EXPECT(c.node_count() == 2 && c.edge_count() == 2 && c.degree(0) == 2 && c.degree(1) == 2);
  EXPECT(c.neighbors(0) == V({1, 1}) && c.neighbors(1) == V({0, 0}));

  if (add_edge_cases<DirectedALGraph>(true)) return 1;
  if (add_edge_cases<UndirectedALGraph>(false)) return 1;

  // adj_list.rs:855-880 and 961-994: add_edge_with_value
  auto wd = GraphBuilder().edges_with_values({{0, 2, 4.2f}, {1, 2, 13.37f}}).build_directed_al();
  EXPECT(same(wd.out_neighbors_with_values(0), {{2, 4.2f}}));
  wd.add_edge_with_value(0, 1, 19.84f);
  EXPECT(same(wd.out_neighbors_with_values(0), {{2, 4.2f}, {1, 19.84f}}));
  wd.add_edge_with_value(0, 2, 1.23f);
  EXPECT(same(wd.out_neighbors_with_values(0), {{2, 4.2f}, {1, 19.84f}, {2, 1.23f}}));
  auto wu = GraphBuilder().edges_with_values({{0, 2, 4.2f}, {1, 2, 13.37f}}).build_undirected_al();
  EXPECT(same(wu.neighbors_with_values(1), {{2, 13.37f}}));
  wu.add_edge_with_value(0, 1, 19.84f);
  EXPECT(same(wu.neighbors_with_values(0), {{2, 4.2f}, {1, 19.84f}}));
  EXPECT(same(wu.neighbors_with_values(1), {{2, 13.37f}, {0, 19.84f}}));
  wu.add_edge_with_value(0, 2, 1.23f);
  EXPECT(same(wu.neighbors_with_values(0), {{2, 4.2f}, {1, 19.84f}, {2, 1.23f}}));

  // the crate doc-test, lib.rs:234-255
  auto doc = GraphBuilder().edges({{0, 1}, {0, 2}, {1, 2}, {1, 3}, {2, 3}}).build_directed_al();
  EXPECT(doc.node_count() == 4 && doc.edge_count() == 5);
  EXPECT(doc.out_degree(1) == 2 && doc.in_degree(1) == 1);
  EXPECT(doc.out_neighbors(1) == V({2, 3}) && doc.in_neighbors(1) == V({0}));
  doc.add_edge(1, 0);
  EXPECT(doc.edge_count() == 6 && doc.out_neighbors(1) == V({2, 3, 0}));

  // to_csr() and the algorithm overloads: the same results as on the snapshot's rows
  DirectedCsrGraph snap = doc.to_csr();
  EXPECT(snap.edge_count() == 6);
  auto [r1, it1, e1] = page_rank(doc, PageRankConfig::new_(10, 0.0, 0.85f));
  auto [r2, it2, e2] = page_rank(snap, PageRankConfig::new_(10, 0.0, 0.85f));
  EXPECT(it1 == it2 && r1.size() == r2.size() && std::memcmp(r1.data(), r2.data(), r1.size() * 4) == 0);
  EXPECT(wcc_afforest(doc).to_vec() == wcc_afforest(snap).to_vec());
  auto dist = delta_stepping(wd, DeltaSteppingConfig::new_(0, 1.0f));
  EXPECT(dist.size() == 3 && dist[0] == 0.0f && dist[1] == 19.84f && dist[2] == 1.23f);
  auto tri = GraphBuilder().csr_layout(CsrLayout::Deduplicated).edges({{0, 1}, {1, 2}, {2, 0}, {2, 2}, {2, 3}})
                 .build_undirected_al();
  // the reference's count on these rows (oracle.triangle_count): the self-loop of node 2 takes part in 4 more
  EXPECT(global_triangle_count(tri) == 5);
  EXPECT(tri.neighbors(2) == V({0, 1, 2, 3}));  // Deduplicated adjacency lists keep self-loops
  std::printf("al_graph ok\n");
  return 0;
}
