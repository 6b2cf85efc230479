// graph::prelude::wcc_file through include/graph_b200.hpp: the labels of wcc_afforest on the graph GraphBuilder loads
// from the same file, for every format, and graph::Error where the load fails.  argv[1] is tests/golden.  Exits 0 and
// prints "wcc_file ok" when every check passes; prints the first failure otherwise.
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

int main(int argc, char** argv) {
  if (argc < 2) {
    std::printf("usage: %s <tests/golden>\n", argv[0]);
    return 64;
  }
  const std::string dir = argv[1];
  const struct {
    const char* name;
    FileFormat format;
  } files[] = {{"scale_8.graph500", FileFormat::Graph500},
               {"example.el", FileFormat::EdgeList},
               {"test.wel", FileFormat::EdgeList},
               {"test.graph", FileFormat::DotGraph},
               {"binary_directed_u32.bin", FileFormat::Binary},
               {"binary_directed_usize_values.bin", FileFormat::Binary}};
  for (const auto& f : files) {
    const std::string path = dir + "/" + f.name;
    const DirectedCsrGraph g = GraphBuilder().file_format(f.format).path(path).build_directed();
    const Components want = wcc_afforest(g);
    const Components got = wcc_file(path, f.format, WccConfig{});
    EXPECT(got.to_vec().size() == g.node_count());
    EXPECT(got.to_vec() == want.to_vec());
  }
  // an undirected binary file is not a directed graph: the load's error
  int status = GB_OK;
  std::string message;
  try {
    wcc_file(dir + "/binary_undirected_u32.bin", FileFormat::Binary);
  } catch (const graph::Error& e) {
    status = e.status;
    message = e.what();
  }
  EXPECT(status == GB_ERR_INVALID);
  EXPECT(message == "binary graph file holds an undirected graph, not a directed one");
  std::printf("wcc_file ok\n");
  return 0;
}
