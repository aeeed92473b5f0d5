// Fast text parsers for the applications' data files (reference apps/mf/io.h:38-352 MatrixMarket readers,
// apps/knowledge_graph_embeddings.cc triple files): one pass over the file buffer, no per-line allocations.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace adapm {

// Whitespace-separated integer triples "s r o", one per line; returns 3*n values.
std::vector<int64_t> read_triples_file(const std::string& path);

struct CooMatrix {
  int64_t rows = 0, cols = 0;
  std::vector<int64_t> i, j;   // 0-based
  std::vector<float> x;
};
// MatrixMarket "matrix coordinate real general" (1-based indices on disk).
CooMatrix read_matrix_market_coo_file(const std::string& path);

struct EdgeList {
  std::vector<int64_t> src, dst;   // node labels 0 .. ids.size() - 1
  std::vector<double> weight;      // empty when the lines have no weight column
  std::vector<int64_t> ids;        // ids[label] = the node's id in the file, ascending
};
// SNAP-style edge list: "src dst [weight]" per line, ids non-negative integers, blank lines and lines starting with
// '#' skipped. Every data line has the field count of the first one. A malformed line throws with its line number.
EdgeList read_edge_list_file(const std::string& path);

}  // namespace adapm
