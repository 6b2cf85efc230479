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
// DotGraph: the node-labelled .graph file (input/dotgraph.rs), built as a labelled twin by gb_[di]graph_load_labeled_u32
enum class FileFormat { Graph500, EdgeList, Binary, DotGraph };

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
  CsrGraphBase(CsrGraphBase&& o) noexcept : g_(o.g_), host_(std::move(o.host_)), labels_(std::move(o.labels_)) {
    o.g_ = nullptr;
  }
  CsrGraphBase& operator=(CsrGraphBase&& o) noexcept {
    if (this != &o) {
      reset();
      g_ = o.g_;
      host_ = std::move(o.host_);
      labels_ = std::move(o.labels_);
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
  // the same for a labelled graph (NI = u32, NV = u32): NodeValues, then the CSRs; throws graph::Error on a graph
  // without labels.  build_[un]directed_labeled() reads the file back.
  void serialize_labeled(const std::string& path) const {
    detail::check(gb_graph_serialize_labeled(g_, path.c_str()));
  }
  // NodeValues::node_value, csr.rs:64-76 (labelled graphs; throws graph::Error on a graph without labels)
  std::uint32_t node_value(std::uint32_t node) const {
    if (labels_.empty()) {
      labels_.resize(node_count());
      detail::check(gb_graph_node_values(g_, labels_.data()));
    }
    if (node >= labels_.size()) throw std::out_of_range("node id out of range");
    return labels_[node];
  }

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
  mutable std::vector<std::uint32_t> labels_;
};

// LabelStats (dotgraph.rs:213-219); label_frequency as (label, count) pairs, labels ascending
struct LabelStats {
  std::uint32_t max_degree = 0;
  std::size_t label_count = 0;
  std::uint32_t max_label = 0;
  std::size_t max_label_frequency = 0;
  std::vector<std::pair<std::uint32_t, std::uint64_t>> label_frequency;
};

// NodeLabelIndex (dotgraph.rs:430-532): nodes(label) lists the nodes with that label, ascending
struct NodeLabelIndex {
  std::vector<std::uint32_t> offsets, node_ids;
  std::pair<const std::uint32_t*, const std::uint32_t*> nodes(std::uint32_t label) const {
    if (offsets.empty() || label >= offsets.size() - 1) throw std::out_of_range("label out of range");
    return {node_ids.data() + offsets[label], node_ids.data() + offsets[label + 1]};
  }
};

// NeighborLabelFrequencies (dotgraph.rs:367-427) as a pair CSR; get(node, label) is 0 for an absent label
struct NeighborLabelFrequencies {
  std::vector<std::uint32_t> offsets, labels, counts;
  std::size_t len(std::uint32_t node) const { return offsets.at(node + 1) - offsets.at(node); }
  std::size_t get(std::uint32_t node, std::uint32_t label) const {
    for (std::uint32_t i = offsets.at(node); i < offsets.at(node + 1); ++i)
      if (labels[i] == label) return counts[i];
    return 0;
  }
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
  // to_undirected keeping the f32 values (csr.rs:391-406): UndirectedCsrGraph<u32, (), f32>; needs a weighted digraph
  inline UndirectedCsrGraph to_undirected_weighted(CsrLayout layout = CsrLayout::Unsorted) const;
};

// UndirectedCsrGraph<u32>, csr.rs:658-661; traits :682-725
class UndirectedCsrGraph : public CsrGraphBase {
 public:
  using CsrGraphBase::CsrGraphBase;
  std::uint32_t degree(std::uint32_t n) const { auto r = row(GB_CSR_UNDIRECTED, n); return static_cast<std::uint32_t>(r.second - r.first); }
  std::pair<const std::uint32_t*, const std::uint32_t*> neighbors(std::uint32_t n) const { return row(GB_CSR_UNDIRECTED, n); }
  // UndirectedNeighborsWithValues::neighbors_with_values (csr.rs:715-725) of a graph with f32 values; throws
  // graph::Error on a graph without values
  std::pair<const Target*, const Target*> neighbors_with_values(std::uint32_t n) const {
    const HostCsr& h = mirror(GB_CSR_UNDIRECTED);
    if (n >= node_count()) throw std::out_of_range("node id out of range");
    if (!values_read_) {
      std::vector<float> w(h.tgt.size());
      std::vector<std::uint32_t> off(h.off.size());
      detail::check(gb_graph_copy_csr(g_, GB_CSR_UNDIRECTED, off.data(), nullptr, w.data()));
      targets_.resize(h.tgt.size());
      for (std::size_t i = 0; i < w.size(); ++i) targets_[i] = Target{h.tgt[i], w[i]};
      values_read_ = true;
    }
    return {targets_.data() + h.off[n], targets_.data() + h.off[n + 1]};
  }
  void make_degree_ordered() {  // RelabelByDegreeOp, graph_ops.rs:173 (labels are not permuted: graph_b200.h)
    detail::check(gb_make_degree_ordered(g_));
    for (auto& h : host_) h = HostCsr{};
    targets_.clear();
    values_read_ = false;
  }
  LabelStats label_stats() const {  // LabelStats::from_graph, dotgraph.rs:220-313
    gb_label_stats_info st{};
    detail::check(gb_label_stats(g_, &st, nullptr, nullptr));
    std::vector<std::uint32_t> labels(st.label_count);
    std::vector<std::uint64_t> counts(st.label_count);
    detail::check(gb_label_stats(g_, &st, labels.data(), counts.data()));
    LabelStats out{st.max_degree, static_cast<std::size_t>(st.label_count), st.max_label,
                   static_cast<std::size_t>(st.max_label_frequency), {}};
    for (std::size_t i = 0; i < labels.size(); ++i) out.label_frequency.emplace_back(labels[i], counts[i]);
    return out;
  }
  NodeLabelIndex node_label_index() const {  // NodeLabelIndex::from_stats, dotgraph.rs:430-532
    std::uint32_t max_label = 0;
    detail::check(gb_node_label_index(g_, &max_label, nullptr, nullptr));
    NodeLabelIndex idx;
    idx.offsets.resize(static_cast<std::size_t>(max_label) + 2);
    idx.node_ids.resize(node_count());
    detail::check(gb_node_label_index(g_, nullptr, idx.offsets.data(), idx.node_ids.data()));
    return idx;
  }
  NeighborLabelFrequencies neighbor_label_frequencies() const {  // dotgraph.rs:367-427
    const gb_graph_info i = info();
    NeighborLabelFrequencies f;
    f.offsets.resize(static_cast<std::size_t>(i.node_count) + 1);
    f.labels.resize(i.target_count ? i.target_count : 1);
    f.counts.resize(i.target_count ? i.target_count : 1);
    detail::check(gb_neighbor_label_frequencies(g_, f.offsets.data(), f.labels.data(), f.counts.data()));
    f.labels.resize(f.offsets.back());
    f.counts.resize(f.offsets.back());
    return f;
  }

 private:
  mutable std::vector<Target> targets_;  // host AoS copy for neighbors_with_values, read once
  mutable bool values_read_ = false;
};

inline UndirectedCsrGraph DirectedCsrGraph::to_undirected(CsrLayout layout) const {
  gb_graph* u = nullptr;
  detail::check(gb_to_undirected(g_, static_cast<gb_layout>(layout), &u));
  return UndirectedCsrGraph(u);
}

inline UndirectedCsrGraph DirectedCsrGraph::to_undirected_weighted(CsrLayout layout) const {
  gb_graph* u = nullptr;
  detail::check(gb_to_undirected_weighted(g_, static_cast<gb_layout>(layout), &u));
  return UndirectedCsrGraph(u);
}

// Adjacency-list graphs, crates/builder/src/graph/adj_list.rs: DirectedALGraph<u32, (), EV> and
// UndirectedALGraph<u32, (), EV> with EV = () or f32.  They take new edges (EdgeMutation::add_edge,
// EdgeMutationWithValues::add_edge_with_value, lib.rs:415-456); a missing node throws graph::Error with the
// reference's message (`node "3" does not exist in the graph ...`).  Neighbours are returned as copies, since rows
// move when edges are added.  to_csr() snapshots the rows into an immutable CSR graph, on which the algorithms run.
class ALGraphBase {
 public:
  explicit ALGraphBase(gb_algraph* g = nullptr) : g_(g) {}
  ALGraphBase(const ALGraphBase&) = delete;
  ALGraphBase& operator=(const ALGraphBase&) = delete;
  ALGraphBase(ALGraphBase&& o) noexcept : g_(o.g_) { o.g_ = nullptr; }
  ALGraphBase& operator=(ALGraphBase&& o) noexcept {
    if (this != &o) {
      if (g_) gb_algraph_free(g_);
      g_ = o.g_;
      o.g_ = nullptr;
    }
    return *this;
  }
  ~ALGraphBase() {
    if (g_) gb_algraph_free(g_);
  }
  std::uint32_t node_count() const { return info().node_count; }  // adj_list.rs:311-322, :475-487
  std::uint64_t edge_count() const { return info().edge_count; }
  gb_algraph* handle() const { return g_; }
  // len(src) add_edge calls in order, as one device batch: all or nothing
  void add_edges(const std::vector<std::uint32_t>& src, const std::vector<std::uint32_t>& dst,
                 const std::vector<float>& values = {}) {
    if (src.size() != dst.size()) throw Error(GB_ERR_INVALID, "src and dst must have the same length");
    if (!values.empty() && values.size() != src.size()) throw Error(GB_ERR_INVALID, "values must have one entry per edge");
    detail::check(gb_algraph_add_edges_u32(g_, src.data(), dst.data(), values.empty() ? nullptr : values.data(),
                                           src.size()));
  }
  void add_edge(std::uint32_t source, std::uint32_t target) { add_edges({source}, {target}); }
  void add_edge_with_value(std::uint32_t source, std::uint32_t target, float value) {
    add_edges({source}, {target}, {value});
  }

 protected:
  gb_graph_info info() const {
    gb_graph_info i{};
    detail::check(gb_algraph_get_info(g_, &i));
    return i;
  }
  std::uint32_t degree_of(gb_csr_which which, std::uint32_t node) const {
    std::uint32_t len = 0;
    detail::check(gb_algraph_copy_row(g_, which, node, 0, nullptr, nullptr, &len));
    return len;
  }
  std::vector<std::uint32_t> row(gb_csr_which which, std::uint32_t node) const {
    std::vector<std::uint32_t> t;
    std::uint32_t len = degree_of(which, node);
    for (;;) {  // another thread may add edges between the two calls
      t.resize(len);
      std::uint32_t got = 0;
      detail::check(gb_algraph_copy_row(g_, which, node, len, t.data(), nullptr, &got));
      if (got <= len) {
        t.resize(got);
        return t;
      }
      len = got;
    }
  }
  std::vector<Target> row_with_values(gb_csr_which which, std::uint32_t node) const {
    std::vector<std::uint32_t> t;
    std::vector<float> w;
    std::uint32_t len = degree_of(which, node);
    for (;;) {
      t.resize(len);
      w.resize(len);
      std::uint32_t got = 0;
      detail::check(gb_algraph_copy_row(g_, which, node, len, t.data(), w.data(), &got));
      if (got <= len) break;
      len = got;
    }
    std::vector<Target> out(t.size());
    for (std::size_t i = 0; i < t.size(); ++i) out[i] = Target{t[i], w[i]};
    return out;
  }
  gb_graph* snapshot() const {
    gb_graph* s = nullptr;
    detail::check(gb_algraph_to_graph(g_, &s));
    return s;
  }
  gb_algraph* g_ = nullptr;
};

// DirectedALGraph, adj_list.rs:279-450
class DirectedALGraph : public ALGraphBase {
 public:
  using ALGraphBase::ALGraphBase;
  std::uint32_t out_degree(std::uint32_t n) const { return degree_of(GB_CSR_OUT, n); }
  std::uint32_t in_degree(std::uint32_t n) const { return degree_of(GB_CSR_IN, n); }
  std::vector<std::uint32_t> out_neighbors(std::uint32_t n) const { return row(GB_CSR_OUT, n); }
  std::vector<std::uint32_t> in_neighbors(std::uint32_t n) const { return row(GB_CSR_IN, n); }
  std::vector<Target> out_neighbors_with_values(std::uint32_t n) const { return row_with_values(GB_CSR_OUT, n); }
  std::vector<Target> in_neighbors_with_values(std::uint32_t n) const { return row_with_values(GB_CSR_IN, n); }
  DirectedCsrGraph to_csr() const { return DirectedCsrGraph(snapshot()); }
};

// UndirectedALGraph, adj_list.rs:452-595
class UndirectedALGraph : public ALGraphBase {
 public:
  using ALGraphBase::ALGraphBase;
  std::uint32_t degree(std::uint32_t n) const { return degree_of(GB_CSR_UNDIRECTED, n); }
  std::vector<std::uint32_t> neighbors(std::uint32_t n) const { return row(GB_CSR_UNDIRECTED, n); }
  std::vector<Target> neighbors_with_values(std::uint32_t n) const { return row_with_values(GB_CSR_UNDIRECTED, n); }
  UndirectedCsrGraph to_csr() const { return UndirectedCsrGraph(snapshot()); }
};

// GraphBuilder, crates/builder/src/builder.rs:123-539 (the in-memory edge-list states)
class GraphBuilder {
 public:
  GraphBuilder& csr_layout(CsrLayout l) { layout_ = l; return *this; }
  GraphBuilder& device(int d) { device_ = d; return *this; }
  GraphBuilder& edges(const std::vector<std::pair<std::uint32_t, std::uint32_t>>& e) {
    src_.clear(); dst_.clear(); w_.clear();
    values_ = false;
    for (auto& p : e) { src_.push_back(p.first); dst_.push_back(p.second); }
    return *this;
  }
  GraphBuilder& edges_with_values(const std::vector<std::tuple<std::uint32_t, std::uint32_t, float>>& e) {
    src_.clear(); dst_.clear(); w_.clear();
    values_ = true;
    for (auto& t : e) { src_.push_back(std::get<0>(t)); dst_.push_back(std::get<1>(t)); w_.push_back(std::get<2>(t)); }
    return *this;
  }
  GraphBuilder& node_count(std::uint32_t n) { n_ = n; return *this; }
  // GraphBuilder::node_values (builder.rs:388, 425): one label per node; the node count is their number
  GraphBuilder& node_values(const std::vector<std::uint32_t>& labels) { labels_ = labels; return *this; }
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
    labels_.clear();
    // a file read with with_values() holds values when its format has them (a binary file's are checked at build)
    values_ = with_values_ && (format_ == FileFormat::EdgeList || format_ == FileFormat::Binary);
    // Binary: the CSRs are read as stored at build time (csr.rs:636-656); DotGraph: loaded as a labelled graph
    if (format_ == FileFormat::Binary || format_ == FileFormat::DotGraph) {
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
    if (!binary_path_.empty() && format_ == FileFormat::DotGraph) {
      detail::check(gb_digraph_load_labeled_u32(device_, binary_path_.c_str(), static_cast<gb_layout>(layout_), &g));
      return DirectedCsrGraph(g);
    }
    if (!binary_path_.empty()) {
      detail::check(gb_digraph_load_u32(device_, binary_path_.c_str(), GB_FORMAT_BINARY, static_cast<gb_layout>(layout_),
                                        with_values_ ? 1 : 0, &g));
      return DirectedCsrGraph(g);
    }
    if (!labels_.empty()) {
      detail::check(gb_digraph_from_edges_labeled_u32(device_, src_.data(), dst_.data(), src_.size(), labels_.data(),
                                                      static_cast<std::uint32_t>(labels_.size()),
                                                      static_cast<gb_layout>(layout_), &g));
      return DirectedCsrGraph(g);
    }
    detail::check(gb_digraph_from_edges_u32(device_, src_.data(), dst_.data(), w_.empty() ? nullptr : w_.data(), src_.size(), n_,
                                            static_cast<gb_layout>(layout_), &g));
    return DirectedCsrGraph(g);
  }
  UndirectedCsrGraph build_undirected() const {
    gb_graph* g = nullptr;
    if (!binary_path_.empty() && format_ == FileFormat::DotGraph) {
      detail::check(gb_graph_load_labeled_u32(device_, binary_path_.c_str(), static_cast<gb_layout>(layout_), &g));
      return UndirectedCsrGraph(g);
    }
    if (!binary_path_.empty()) {
      detail::check(gb_graph_load_u32(device_, binary_path_.c_str(), GB_FORMAT_BINARY, static_cast<gb_layout>(layout_), &g));
      return UndirectedCsrGraph(g);
    }
    if (!labels_.empty()) {
      detail::check(gb_graph_from_edges_labeled_u32(device_, src_.data(), dst_.data(), src_.size(), labels_.data(),
                                                    static_cast<std::uint32_t>(labels_.size()),
                                                    static_cast<gb_layout>(layout_), &g));
      return UndirectedCsrGraph(g);
    }
    detail::check(gb_graph_from_edges_u32(device_, src_.data(), dst_.data(), src_.size(), n_, static_cast<gb_layout>(layout_), &g));
    return UndirectedCsrGraph(g);
  }
  // UndirectedCsrGraph<u32, (), f32> (the reference's EV = f32 undirected build, csr.rs:124-221): from
  // edges_with_values(..), or from a file read with with_values() (edge list or Binary); both entries of an edge
  // carry its value.  Throws graph::Error when the builder holds no values.
  UndirectedCsrGraph build_undirected_weighted() const {
    if (!values_) throw Error(GB_ERR_INVALID, "build_undirected_weighted needs edges_with_values(..) or a file read with with_values()");
    gb_graph* g = nullptr;
    if (!binary_path_.empty()) {
      detail::check(gb_graph_load_weighted_u32(device_, binary_path_.c_str(), GB_FORMAT_BINARY, static_cast<gb_layout>(layout_), &g));
      return UndirectedCsrGraph(g);
    }
    detail::check(gb_graph_from_weighted_edges_u32(device_, src_.data(), dst_.data(), w_.data(), src_.size(), n_,
                                                   static_cast<gb_layout>(layout_), &g));
    return UndirectedCsrGraph(g);
  }
  // DirectedCsrGraph<u32, NV> / UndirectedCsrGraph<u32, NV> from file_format(FileFormat::Binary).path(p), as
  // build::<DirectedCsrGraph<u32, u32>>() reads a binary file: NodeValues of label_bytes each (4: u32, 8: u64 /
  // usize, narrowed), then the CSRs as stored.  Throws graph::Error for any other source.
  DirectedCsrGraph build_directed_labeled(std::uint32_t label_bytes = 4) const {
    gb_graph* g = nullptr;
    detail::check(gb_digraph_load_labeled_binary_u32(device_, labeled_binary_path().c_str(),
                                                     static_cast<gb_layout>(layout_), label_bytes, &g));
    return DirectedCsrGraph(g);
  }
  UndirectedCsrGraph build_undirected_labeled(std::uint32_t label_bytes = 4) const {
    gb_graph* g = nullptr;
    detail::check(gb_graph_load_labeled_binary_u32(device_, labeled_binary_path().c_str(),
                                                   static_cast<gb_layout>(layout_), label_bytes, &g));
    return UndirectedCsrGraph(g);
  }
  // DirectedALGraph / UndirectedALGraph from the pending edges (adj_list.rs:406-450, :559-595): with values
  // (EV = f32) when the builder holds them (edges_with_values(..), or an edge list read with with_values()).
  // Graph500 and edge-list files; Binary and DotGraph files and node values have no adjacency-list form here.
  DirectedALGraph build_directed_al() const { return DirectedALGraph(build_al(GB_KIND_DIRECTED)); }
  UndirectedALGraph build_undirected_al() const { return UndirectedALGraph(build_al(GB_KIND_UNDIRECTED)); }

 private:
  const std::string& labeled_binary_path() const {
    if (binary_path_.empty() || format_ != FileFormat::Binary)
      throw Error(GB_ERR_INVALID, "build_directed_labeled / build_undirected_labeled read file_format(FileFormat::Binary).path(p)");
    return binary_path_;
  }
  gb_algraph* build_al(gb_graph_kind kind) const {
    if (!binary_path_.empty() || !labels_.empty())
      throw Error(GB_ERR_UNSUPPORTED, "adjacency-list graphs are built from edges, Graph500 or edge-list files");
    gb_algraph* g = nullptr;
    detail::check(gb_algraph_from_edges_u32(device_, kind, src_.data(), dst_.data(), values_ ? w_.data() : nullptr,
                                            src_.size(), n_, static_cast<gb_layout>(layout_), values_ ? 1 : 0, &g));
    return g;
  }
  CsrLayout layout_ = CsrLayout::Unsorted;  // CsrLayout::default()
  FileFormat format_ = FileFormat::EdgeList;
  bool with_values_ = false;
  bool values_ = false;  // the pending edges (or file) carry f32 values
  int device_ = 0;
  std::uint32_t n_ = 0;
  std::string binary_path_;  // set by path(..) for FileFormat::Binary and FileFormat::DotGraph
  std::vector<std::uint32_t> src_, dst_, labels_;
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
// wcc(&GraphBuilder::new().file_format(format).path(path).build::<DirectedCsrGraph<u32>>()) in one pass over the
// file, without building the graph (gb_wcc_file_u32): each chunk's edges are linked on the device as they are
// decoded.  The labels of wcc_afforest on the loaded graph; throws graph::Error where the load fails, except that
// Graph500, edge-list and DotGraph files of 2^32 - 1 edges or more are accepted.
inline Components wcc_file(const std::string& path, FileFormat format, WccConfig c = {}, int device = 0) {
  gb_wcc_config cfg{c.chunk_size, c.neighbor_rounds, c.sampling_size};
  gb_components* h = nullptr;
  detail::check(gb_wcc_file_u32(device, path.c_str(), static_cast<gb_file_format>(format), &cfg, &h));
  struct Free {
    gb_components* h;
    ~Free() { gb_components_free(h); }
  } free_h{h};
  std::uint32_t n = 0;
  detail::check(gb_components_node_count(h, &n));
  Components out;
  out.ids.resize(n);
  detail::check(gb_components_copy(h, out.ids.data()));
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
// delta_stepping of a host weighted out-CSR (offsets[node_count + 1], targets and f32 weights[offsets[node_count]]),
// streamed to the device in row-aligned chunks from the start's chunk on and relaxed as they land, without a
// resident twin or an in-CSR (gb_sssp_csr_u32); the distances delta_stepping gives on DirectedCsrGraph::from_csr
// of the same arrays
inline std::vector<float> delta_stepping_csr(std::uint32_t node_count, const std::uint32_t* offsets,
                                             const std::uint32_t* targets, const float* weights,
                                             DeltaSteppingConfig c, int device = 0) {
  gb_sssp_config cfg{c.start_node, c.delta};
  std::vector<float> dist(node_count);
  detail::check(gb_sssp_csr_u32(device, node_count, offsets, targets, weights, &cfg, dist.data()));
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

// The algorithms on adjacency-list graphs: the reference's are generic over the traits both storage types
// implement, so they run here on a snapshot of the rows (to_csr()), whose results the rows alone define.
inline std::tuple<std::vector<float>, std::size_t, double> page_rank(const DirectedALGraph& g, PageRankConfig c) {
  return page_rank(g.to_csr(), c);
}
inline Components wcc_afforest(const DirectedALGraph& g, WccConfig c = {}) { return wcc_afforest(g.to_csr(), c); }
inline std::vector<float> delta_stepping(const DirectedALGraph& g, DeltaSteppingConfig c) {
  return delta_stepping(g.to_csr(), c);
}
inline std::uint64_t global_triangle_count(const UndirectedALGraph& g) { return global_triangle_count(g.to_csr()); }

}  // namespace prelude
}  // namespace graph
