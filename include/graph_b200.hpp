// graph_b200.hpp — C++17 host API over the C ABI, mirroring `graph::prelude` of neo4j-labs/graph.
//
// The reference's compiled-language surface is Rust (crates/algos/src/prelude.rs:1-7 re-exports
// page_rank::*, wcc::*, sssp::*, triangle_count::* and graph_builder::prelude).  Rust is not available
// in this image, so this header is the compiled host side: same names, argument meaning, defaults and
// result shapes, header-only over include/graph_b200.h.  Where the reference panics (index out of
// range) or returns graph_builder::Error this API throws graph::Error.
//
//   using namespace graph::prelude;
//   DirectedCsrGraph g = GraphBuilder().csr_layout(CsrLayout::Sorted).edges({{0, 1}, {0, 2}, {1, 2}}).build_directed();
//   auto [ranks, iterations, error] = page_rank(g, PageRankConfig::new_(10, 1e-4, 0.85f));
#pragma once
#include <array>
#include <cstdint>
#include <fstream>
#include <iterator>
#include <stdexcept>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "graph_b200.h"

namespace graph {

struct Error : std::runtime_error {  // graph_builder::Error, crates/builder/src/lib.rs:274-302
  gb_status status;
  Error(gb_status st, const std::string& msg) : std::runtime_error(msg), status(st) {}
};

namespace detail {
inline void check(gb_status st) {
  if (st != GB_OK) throw Error(st, gb_last_error());
}
}  // namespace detail

namespace prelude {

// crates/builder/src/graph/csr.rs:35-45
enum class CsrLayout { Unsorted = GB_LAYOUT_UNSORTED, Sorted = GB_LAYOUT_SORTED, Deduplicated = GB_LAYOUT_DEDUPLICATED };

// input formats of `GraphBuilder::file_format(..).path(..)` (builder.rs:283-361; input/graph500.rs, input/edgelist.rs)
// Binary: the file of SerializeGraphOp (input/binary.rs), loaded as stored by gb_[di]graph_load_u32
enum class FileFormat { Graph500, EdgeList, Binary };

// crates/algos/src/page_rank.rs:14-56
struct PageRankConfig {
  static constexpr std::size_t DEFAULT_MAX_ITERATIONS = 20;
  static constexpr double DEFAULT_TOLERANCE = 1e-4;
  static constexpr float DEFAULT_DAMPING_FACTOR = 0.85f;
  std::size_t max_iterations = DEFAULT_MAX_ITERATIONS;
  double tolerance = DEFAULT_TOLERANCE;
  float damping_factor = DEFAULT_DAMPING_FACTOR;
  static PageRankConfig new_(std::size_t max_iterations, double tolerance, float damping_factor) {
    return PageRankConfig{max_iterations, tolerance, damping_factor};
  }
};

// crates/algos/src/wcc.rs:40-79
struct WccConfig {
  static constexpr std::size_t DEFAULT_CHUNK_SIZE = 16384;
  static constexpr std::size_t DEFAULT_NEIGHBOR_ROUNDS = 2;
  static constexpr std::size_t DEFAULT_SAMPLING_SIZE = 1024;
  std::size_t chunk_size = DEFAULT_CHUNK_SIZE;
  std::size_t neighbor_rounds = DEFAULT_NEIGHBOR_ROUNDS;
  std::size_t sampling_size = DEFAULT_SAMPLING_SIZE;
};

// crates/algos/src/sssp.rs:18-36
struct DeltaSteppingConfig {
  std::size_t start_node;
  float delta;
  static DeltaSteppingConfig new_(std::size_t start_node, float delta) { return {start_node, delta}; }
};

// #[repr(C)] Target<u32, f32>, crates/builder/src/graph/mod.rs:6-10
struct Target {
  std::uint32_t target;
  float value;
};

class CsrGraphBase {
 public:
  CsrGraphBase() = default;
  explicit CsrGraphBase(gb_graph* g) : g_(g) {}
  CsrGraphBase(const CsrGraphBase&) = delete;
  CsrGraphBase& operator=(const CsrGraphBase&) = delete;
  CsrGraphBase(CsrGraphBase&& o) noexcept : g_(o.g_), host_(std::move(o.host_)) { o.g_ = nullptr; }
  CsrGraphBase& operator=(CsrGraphBase&& o) noexcept {
    if (this != &o) {
      reset();
      g_ = o.g_;
      host_ = std::move(o.host_);
      o.g_ = nullptr;
    }
    return *this;
  }
  ~CsrGraphBase() { reset(); }

  std::uint32_t node_count() const { return info().node_count; }  // Graph::node_count, lib.rs:315-321
  std::uint64_t edge_count() const { return info().edge_count; }
  gb_graph* handle() const { return g_; }
  // SerializeGraphOp::serialize, graph_ops.rs:232-238 (NI = u32)
  void serialize(const std::string& path) const { detail::check(gb_graph_serialize(g_, path.c_str())); }

 protected:
  struct HostCsr {
    std::vector<std::uint32_t> off, tgt;
  };
  void reset() {
    if (g_) gb_graph_free(g_);
    g_ = nullptr;
  }
  gb_graph_info info() const {
    gb_graph_info i{};
    detail::check(gb_graph_get_info(g_, &i));
    return i;
  }
  const HostCsr& mirror(gb_csr_which which) const {  // neighbour slices come from a host copy
    auto& h = host_[static_cast<int>(which)];
    if (h.off.empty()) {
      std::uint64_t len = 0;
      detail::check(gb_graph_csr_len(g_, which, &len));
      h.off.resize(static_cast<std::size_t>(node_count()) + 1);
      h.tgt.resize(len);
      detail::check(gb_graph_copy_csr(g_, which, h.off.data(), len ? h.tgt.data() : nullptr, nullptr));
    }
    return h;
  }
  std::pair<const std::uint32_t*, const std::uint32_t*> row(gb_csr_which which, std::uint32_t node) const {
    const HostCsr& h = mirror(which);
    if (node >= node_count()) throw std::out_of_range("node id out of range");  // Idx::new assert, index.rs:51-54
    return {h.tgt.data() + h.off[node], h.tgt.data() + h.off[node + 1]};
  }
  gb_graph* g_ = nullptr;
  mutable std::array<HostCsr, 3> host_;
};

class UndirectedCsrGraph;

// DirectedCsrGraph<u32>, crates/builder/src/graph/csr.rs:364-368; traits :466-520
class DirectedCsrGraph : public CsrGraphBase {
 public:
  using CsrGraphBase::CsrGraphBase;
  std::uint32_t out_degree(std::uint32_t n) const { auto r = row(GB_CSR_OUT, n); return static_cast<std::uint32_t>(r.second - r.first); }
  std::uint32_t in_degree(std::uint32_t n) const { auto r = row(GB_CSR_IN, n); return static_cast<std::uint32_t>(r.second - r.first); }
  std::pair<const std::uint32_t*, const std::uint32_t*> out_neighbors(std::uint32_t n) const { return row(GB_CSR_OUT, n); }
  std::pair<const std::uint32_t*, const std::uint32_t*> in_neighbors(std::uint32_t n) const { return row(GB_CSR_IN, n); }
  inline UndirectedCsrGraph to_undirected(CsrLayout layout = CsrLayout::Unsorted) const;  // graph_ops.rs:229
};

// UndirectedCsrGraph<u32>, csr.rs:658-661; traits :682-725
class UndirectedCsrGraph : public CsrGraphBase {
 public:
  using CsrGraphBase::CsrGraphBase;
  std::uint32_t degree(std::uint32_t n) const { auto r = row(GB_CSR_UNDIRECTED, n); return static_cast<std::uint32_t>(r.second - r.first); }
  std::pair<const std::uint32_t*, const std::uint32_t*> neighbors(std::uint32_t n) const { return row(GB_CSR_UNDIRECTED, n); }
  void make_degree_ordered() {  // RelabelByDegreeOp, graph_ops.rs:173
    detail::check(gb_make_degree_ordered(g_));
    for (auto& h : host_) h = HostCsr{};
  }
};

inline UndirectedCsrGraph DirectedCsrGraph::to_undirected(CsrLayout layout) const {
  gb_graph* u = nullptr;
  detail::check(gb_to_undirected(g_, static_cast<gb_layout>(layout), &u));
  return UndirectedCsrGraph(u);
}

// GraphBuilder, crates/builder/src/builder.rs:123-539 (the in-memory edge-list states)
class GraphBuilder {
 public:
  GraphBuilder& csr_layout(CsrLayout l) { layout_ = l; return *this; }
  GraphBuilder& device(int d) { device_ = d; return *this; }
  GraphBuilder& edges(const std::vector<std::pair<std::uint32_t, std::uint32_t>>& e) {
    src_.clear(); dst_.clear(); w_.clear();
    for (auto& p : e) { src_.push_back(p.first); dst_.push_back(p.second); }
    return *this;
  }
  GraphBuilder& edges_with_values(const std::vector<std::tuple<std::uint32_t, std::uint32_t, float>>& e) {
    src_.clear(); dst_.clear(); w_.clear();
    for (auto& t : e) { src_.push_back(std::get<0>(t)); dst_.push_back(std::get<1>(t)); w_.push_back(std::get<2>(t)); }
    return *this;
  }
  GraphBuilder& node_count(std::uint32_t n) { n_ = n; return *this; }
  // file_format(format).path(p): read the file with the library's native readers (csrc/io.cu)
  GraphBuilder& file_format(FileFormat f) { format_ = f; return *this; }
  // read the third column of a text edge list as f32 edge values (the reference selects this through
  // the graph type's EV parameter: DirectedCsrGraph<u32, (), f32>)
  GraphBuilder& with_values(bool on = true) { with_values_ = on; return *this; }
  GraphBuilder& path(const std::string& p) {
    std::ifstream in(p, std::ios::binary);
    if (!in) throw Error(GB_ERR_INVALID, "cannot open " + p);  // Error::IoError, lib.rs:276-281
    src_.clear(); dst_.clear(); w_.clear();
    binary_path_.clear();
    if (format_ == FileFormat::Binary) {  // the CSRs are read as stored at build time (csr.rs:636-656)
      binary_path_ = p;
      return *this;
    }
    std::vector<char> bytes((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
    std::uint64_t m = 0;
    if (format_ == FileFormat::Graph500) {
      src_.resize(bytes.size() / 12);
      dst_.resize(bytes.size() / 12);
      detail::check(gb_graph500_decode(bytes.data(), bytes.size(), src_.data(), dst_.data(), &m, &n_));
    } else {
      detail::check(gb_edge_list_parse(bytes.data(), bytes.size(), nullptr, nullptr, nullptr, &m));
      src_.resize(m);
      dst_.resize(m);
      // the value column travels with the edges when the builder was asked for values (EV = f32,
      // edgelist.rs:237-241: a missing value is EV::default())
      if (with_values_) w_.resize(m);
      detail::check(gb_edge_list_parse(bytes.data(), bytes.size(), src_.data(), dst_.data(),
                                       with_values_ ? w_.data() : nullptr, &m));
      n_ = 0;  // max id + 1
    }
    return *this;
  }
  // what the builder currently holds (after edges(..) or path(..))
  std::size_t pending_edge_count() const { return src_.size(); }
  std::uint32_t pending_node_count() const { return n_; }  // 0 = "max id + 1" at build time
  const std::vector<std::uint32_t>& pending_sources() const { return src_; }
  const std::vector<std::uint32_t>& pending_targets() const { return dst_; }
  const std::vector<float>& pending_values() const { return w_; }
  DirectedCsrGraph build_directed() const {
    gb_graph* g = nullptr;
    if (!binary_path_.empty()) {
      detail::check(gb_digraph_load_u32(device_, binary_path_.c_str(), GB_FORMAT_BINARY, static_cast<gb_layout>(layout_),
                                        with_values_ ? 1 : 0, &g));
      return DirectedCsrGraph(g);
    }
    detail::check(gb_digraph_from_edges_u32(device_, src_.data(), dst_.data(), w_.empty() ? nullptr : w_.data(), src_.size(), n_,
                                            static_cast<gb_layout>(layout_), &g));
    return DirectedCsrGraph(g);
  }
  UndirectedCsrGraph build_undirected() const {
    gb_graph* g = nullptr;
    if (!binary_path_.empty()) {
      detail::check(gb_graph_load_u32(device_, binary_path_.c_str(), GB_FORMAT_BINARY, static_cast<gb_layout>(layout_), &g));
      return UndirectedCsrGraph(g);
    }
    detail::check(gb_graph_from_edges_u32(device_, src_.data(), dst_.data(), src_.size(), n_, static_cast<gb_layout>(layout_), &g));
    return UndirectedCsrGraph(g);
  }

 private:
  CsrLayout layout_ = CsrLayout::Unsorted;  // CsrLayout::default()
  FileFormat format_ = FileFormat::EdgeList;
  bool with_values_ = false;
  int device_ = 0;
  std::uint32_t n_ = 0;
  std::string binary_path_;  // set by path(..) for FileFormat::Binary
  std::vector<std::uint32_t> src_, dst_;
  std::vector<float> w_;
};

// page_rank(&graph, config) -> (Vec<f32>, usize, f64)          crates/algos/src/page_rank.rs:58
inline std::tuple<std::vector<float>, std::size_t, double> page_rank(const DirectedCsrGraph& g, PageRankConfig c) {
  gb_page_rank_config cfg{c.max_iterations, c.tolerance, c.damping_factor, GB_PR_AUTO};
  std::vector<float> scores(g.node_count());
  std::uint64_t it = 0;
  double err = 0.0;
  detail::check(gb_page_rank(g.handle(), &cfg, scores.data(), &it, &err));
  return {std::move(scores), static_cast<std::size_t>(it), err};
}
// page_rank of a host CSR (in offsets / targets, out offsets: node_count + 1, in_offsets[node_count] and
// node_count + 1 entries) over the devices of a communicator, with no resident twin (gb_page_rank_csr_multi_u32):
// each device uploads about 1/ndev of the arrays; the sharded JACOBI schedule of gb_page_rank_multi
inline std::tuple<std::vector<float>, std::size_t, double> page_rank_csr_multi(
    gb_comm* comm, std::uint32_t node_count, const std::uint32_t* in_offsets, const std::uint32_t* in_targets,
    const std::uint32_t* out_offsets, PageRankConfig c) {
  gb_page_rank_config cfg{c.max_iterations, c.tolerance, c.damping_factor, GB_PR_JACOBI};
  std::vector<float> scores(node_count);
  std::uint64_t it = 0;
  double err = 0.0;
  detail::check(gb_page_rank_csr_multi_u32(comm, node_count, in_offsets, in_targets, out_offsets, &cfg,
                                           scores.data(), &it, &err));
  return {std::move(scores), static_cast<std::size_t>(it), err};
}

// wcc_afforest(&graph, config) -> impl Components; `to_vec()` / `component(n)`   wcc.rs:95-99,127
struct Components {
  std::vector<std::uint32_t> ids;
  std::uint32_t component(std::uint32_t node) const { return ids.at(node); }
  const std::vector<std::uint32_t>& to_vec() const { return ids; }
};
inline Components wcc_afforest(const DirectedCsrGraph& g, WccConfig c = {}) {
  gb_wcc_config cfg{c.chunk_size, c.neighbor_rounds, c.sampling_size};
  Components out;
  out.ids.resize(g.node_count());
  detail::check(gb_wcc(g.handle(), &cfg, out.ids.data()));
  return out;
}
// wcc_baseline(&graph, config) of a host out-CSR (offsets: node_count + 1 entries, targets: offsets[node_count]),
// streamed to the device without a resident twin (gb_wcc_csr_u32); the same labels as wcc_afforest
inline Components wcc_baseline_csr(std::uint32_t node_count, const std::uint32_t* offsets,
                                   const std::uint32_t* targets, WccConfig c = {}, int device = 0) {
  gb_wcc_config cfg{c.chunk_size, c.neighbor_rounds, c.sampling_size};
  Components out;
  out.ids.resize(node_count);
  detail::check(gb_wcc_csr_u32(device, node_count, offsets, targets, &cfg, out.ids.data()));
  return out;
}
// global_triangle_count of a host undirected CSR (same layout), streamed to the device in row-aligned chunks and
// counted as they land, without a resident twin (gb_triangle_count_csr_u32); the number global_triangle_count
// gives on UndirectedCsrGraph::from_csr of the same arrays
inline std::uint64_t global_triangle_count_csr(std::uint32_t node_count, const std::uint32_t* offsets,
                                               const std::uint32_t* targets, int device = 0) {
  std::uint64_t t = 0;
  detail::check(gb_triangle_count_csr_u32(device, node_count, offsets, targets, &t));
  return t;
}

// delta_stepping(&graph, config) -> Vec<AtomicF32>             sssp.rs:38
inline std::vector<float> delta_stepping(const DirectedCsrGraph& g, DeltaSteppingConfig c) {
  gb_sssp_config cfg{c.start_node, c.delta};
  std::vector<float> dist(g.node_count());
  detail::check(gb_sssp(g.handle(), &cfg, dist.data()));
  return dist;
}

// global_triangle_count(&graph) -> u64                         triangle_count.rs:22
inline std::uint64_t global_triangle_count(const UndirectedCsrGraph& g) {
  std::uint64_t t = 0;
  detail::check(gb_triangle_count(g.handle(), &t));
  return t;
}
// relabel_graph(&mut graph)                                    triangle_count.rs:12-20
inline void relabel_graph(UndirectedCsrGraph& g) { g.make_degree_ordered(); }

}  // namespace prelude
}  // namespace graph
