// Labelled binary graph files through include/graph_b200.hpp: CsrGraphBase::serialize_labeled and
// GraphBuilder::build_directed_labeled / build_undirected_labeled.  argv[1] is tests/golden, argv[2] a writable
// directory.  Exits 0 and prints "labeled_binary ok" when every check passes; prints the first failure otherwise.
#include <cstdio>
#include <string>
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

template <typename F>
static int status_of(F&& f) {
  try {
    f();
  } catch (const graph::Error& e) {
    return e.status;
  }
  return GB_OK;
}

static std::vector<std::uint32_t> labels_of(const CsrGraphBase& g) {
  std::vector<std::uint32_t> out;
  for (std::uint32_t v = 0; v < g.node_count(); ++v) out.push_back(g.node_value(v));
  return out;
}

static std::vector<std::uint32_t> row(std::pair<const std::uint32_t*, const std::uint32_t*> r) {
  return std::vector<std::uint32_t>(r.first, r.second);
}

static std::vector<char> bytes_of(const std::string& path) {
  std::ifstream in(path, std::ios::binary);
  return std::vector<char>((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
}

int main(int argc, char** argv) {
  if (argc < 3) {
    std::printf("usage: %s <tests/golden> <scratch dir>\n", argv[0]);
    return 64;
  }
  const std::string dir = argv[1], tmp = argv[2];
  const std::vector<std::uint32_t> golden_labels = {7, 0, 0xFFFFFFFFu, 3};
  try {
    {  // the labelled goldens at both widths: the same twin
      DirectedCsrGraph a = GraphBuilder()
                               .file_format(FileFormat::Binary)
                               .path(dir + "/binary_labeled_directed_u32.bin")
                               .build_directed_labeled();
      DirectedCsrGraph b = GraphBuilder()
                               .file_format(FileFormat::Binary)
                               .path(dir + "/binary_labeled_directed_usize_values.bin")
                               .build_directed_labeled(8);
      EXPECT(a.node_count() == 4 && a.edge_count() == 6 && b.edge_count() == 6);
      EXPECT(labels_of(a) == golden_labels && labels_of(b) == golden_labels);
      for (std::uint32_t v = 0; v < 4; ++v) {
        EXPECT(row(a.out_neighbors(v)) == row(b.out_neighbors(v)));
        EXPECT(row(a.in_neighbors(v)) == row(b.in_neighbors(v)));
      }
      EXPECT((row(a.out_neighbors(1)) == std::vector<std::uint32_t>{2, 3}));
      // saved and rebuilt: the u32 golden byte for byte
      a.serialize_labeled(tmp + "/a.bin");
      EXPECT(bytes_of(tmp + "/a.bin") == bytes_of(dir + "/binary_labeled_directed_u32.bin"));
      b.serialize_labeled(tmp + "/b.bin");
      EXPECT(bytes_of(tmp + "/b.bin") == bytes_of(tmp + "/a.bin"));
    }
    {  // a labelled undirected twin from node_values(..): the builder round trip and the label structures
      UndirectedCsrGraph g = GraphBuilder()
                                 .csr_layout(CsrLayout::Sorted)
                                 .edges({{0, 1}, {0, 2}, {1, 2}, {1, 3}, {2, 4}, {3, 4}})
                                 .node_values({0, 1, 2, 1, 2})
                                 .build_undirected();
      g.serialize_labeled(tmp + "/u.bin");
      UndirectedCsrGraph h =
          GraphBuilder().file_format(FileFormat::Binary).path(tmp + "/u.bin").build_undirected_labeled();
      EXPECT(h.node_count() == 5 && h.edge_count() == g.edge_count());
      EXPECT(labels_of(h) == labels_of(g));
      for (std::uint32_t v = 0; v < 5; ++v) EXPECT(row(h.neighbors(v)) == row(g.neighbors(v)));
      LabelStats a = g.label_stats(), b = h.label_stats();
      EXPECT(a.max_degree == b.max_degree && a.label_count == b.label_count && a.label_frequency == b.label_frequency);
      NeighborLabelFrequencies fa = g.neighbor_label_frequencies(), fb = h.neighbor_label_frequencies();
      EXPECT(fa.offsets == fb.offsets && fa.labels == fb.labels && fa.counts == fb.counts);
      h.serialize_labeled(tmp + "/u2.bin");
      EXPECT(bytes_of(tmp + "/u2.bin") == bytes_of(tmp + "/u.bin"));
      // the unlabelled writer keeps refusing a labelled twin
      EXPECT(status_of([&] { g.serialize(tmp + "/plain.bin"); }) == GB_ERR_UNSUPPORTED);
    }
    // any other source is an error
    EXPECT(status_of([] { GraphBuilder().edges({{0, 1}}).build_directed_labeled(); }) == GB_ERR_INVALID);
    EXPECT(status_of([&] {
             GraphBuilder().file_format(FileFormat::DotGraph).path(dir + "/test.graph").build_undirected_labeled();
           }) == GB_ERR_INVALID);
    EXPECT(status_of([&] {
             GraphBuilder().file_format(FileFormat::EdgeList).path(dir + "/test.el").build_directed_labeled();
           }) == GB_ERR_INVALID);
    // a width the file does not have, and an unlabelled file
    EXPECT(status_of([&] {
             GraphBuilder().file_format(FileFormat::Binary).path(dir + "/binary_labeled_directed_u32.bin")
                 .build_directed_labeled(8);
           }) == GB_ERR_INVALID);
    EXPECT(status_of([&] {
             GraphBuilder().file_format(FileFormat::Binary).path(dir + "/binary_labeled_directed_u32.bin")
                 .build_directed_labeled(2);
           }) == GB_ERR_INVALID);
    EXPECT(status_of([&] {
             GraphBuilder().file_format(FileFormat::Binary).path(dir + "/binary_undirected_u32.bin")
                 .build_undirected_labeled();
           }) == GB_ERR_INVALID);
    // an unlabelled twin cannot be saved as a labelled one
    DirectedCsrGraph plain = GraphBuilder().edges({{0, 1}}).build_directed();
    EXPECT(status_of([&] { plain.serialize_labeled(tmp + "/none.bin"); }) == GB_ERR_UNSUPPORTED);
  } catch (const graph::Error& e) {
    std::printf("graph::Error %d: %s\n", (int)e.status, e.what());
    return (int)e.status;
  }
  std::printf("labeled_binary ok\n");
  return 0;
}
