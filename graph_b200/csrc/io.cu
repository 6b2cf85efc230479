// io.cu — native host-side readers of the reference's two input formats (no device code).
//
//   Graph500 packed edges   crates/builder/src/input/graph500.rs:63-127
//   text edge lists         crates/builder/src/input/edgelist.rs:181-279
//   DotGraph (.graph)       crates/builder/src/input/dotgraph.rs:136-203 (one thread: the device loader
//                           takes every file it is worth splitting)
//
// Like the reference the work is split into one contiguous chunk per hardware thread (edgelist.rs:
// 186-212 cuts at line boundaries); unlike it the chunks are written at prefix offsets, so the edge
// order is the file order on every run (the reference appends chunks in completion order).
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "binary_format.h"
#include "common.cuh"
#include "edgelist_line.h"

namespace gb {

static unsigned io_threads(uint64_t work_items) {
  unsigned hw = std::thread::hardware_concurrency();
  if (hw == 0) hw = 4;  // DEFAULT_PARALLELISM, crates/algos/src/lib.rs:152
  const uint64_t by_work = std::max<uint64_t>(1, work_items / (1u << 16));
  return (unsigned)std::min<uint64_t>(hw, by_work);
}

template <typename F>
static void parallel_chunks(unsigned threads, F&& body) {
  if (threads <= 1) {
    body(0u);
    return;
  }
  std::vector<std::thread> pool;
  pool.reserve(threads);
  for (unsigned t = 0; t < threads; ++t) pool.emplace_back([&body, t] { body(t); });
  for (auto& th : pool) th.join();
}

// the end of the line that starts at p: the position of its '\n', or len
static uint64_t line_end(const char* text, uint64_t p, uint64_t len) {
  const void* nl = std::memchr(text + p, '\n', len - p);
  return nl ? (uint64_t)(static_cast<const char*>(nl) - text) : len;
}

gb_status dot_fail(uint32_t code, uint64_t line, const DotHeader& h, uint64_t have) {
  if (code == DOT_MISSING) {
    if (have == 0) return fail(GB_ERR_INVALID, "DotGraph file is empty: the header line \"t N M\" is missing");
    return fail(GB_ERR_INVALID, "DotGraph file ends after %llu lines; its header declares 1 + %u node + %u edge lines",
                (unsigned long long)have, h.nodes, h.edges);
  }
  return fail(GB_ERR_INVALID, "DotGraph line %llu: %s", (unsigned long long)line, dot_error_text(code));
}

gb_status dot_read_header(const char* text, uint64_t len, DotHeader* h) {
  if (len == 0) return dot_fail(DOT_MISSING, 0, *h, 0);
  const uint64_t eol = line_end(text, 0, len);
  uint32_t v[2];
  if (const uint32_t code = dot_line(text, 0, eol, 2, v)) return dot_fail(code, 1, *h, 0);
  h->nodes = v[0];
  h->edges = v[1];
  h->lines = 1 + (uint64_t)v[0] + v[1];
  h->body = eol < len ? eol + 1 : len;
  return GB_OK;
}

gb_status dot_read_host(const char* text, uint64_t len, const DotHeader& h, uint32_t* labels, uint32_t* src,
                        uint32_t* dst) {
  uint64_t p = h.body;
  for (uint64_t line = 1; line < h.lines; ++line) {  // 0-based: the header is line 0
    if (p >= len) return dot_fail(DOT_MISSING, 0, h, line);
    const uint64_t eol = line_end(text, p, len);
    uint32_t v[3];
    const bool node = line <= h.nodes;
    if (const uint32_t code = dot_line(text, p, eol, node ? 3 : 2, v)) return dot_fail(code, line + 1, h, 0);
    if (node) {
      if (labels) labels[line - 1] = v[1];
    } else if (src) {
      src[line - 1 - h.nodes] = v[0];
      dst[line - 1 - h.nodes] = v[1];
    }
    p = eol < len ? eol + 1 : len;
  }
  return GB_OK;
}

}  // namespace gb

extern "C" {

// PackedEdge{v0_low, v1_low, high}: src = v0_low | (high & 0xFFFF) << 32, dst = v1_low | (high >> 16) << 32
// (graph500.rs:111-127); node_count = edge_count / 16 (graph500.rs:74).
gb_status gb_graph500_decode(const void* bytes, uint64_t len, uint32_t* src, uint32_t* dst, uint64_t* edge_count,
                             uint32_t* node_count) {
  GB_REQUIRE(edge_count && node_count, "NULL argument");
  const uint64_t m = len / 12;
  *edge_count = m;
  *node_count = (uint32_t)std::min<uint64_t>(m / 16, 0xFFFFFFFFull);
  if (m == 0) return GB_OK;
  GB_REQUIRE(bytes && src && dst, "NULL argument");
  const unsigned T = gb::io_threads(m);
  std::vector<int> bad(T, 0);
  const uint8_t* base = static_cast<const uint8_t*>(bytes);
  gb::parallel_chunks(T, [&](unsigned t) {
    const uint64_t b = m * t / T, e = m * (t + 1) / T;
    for (uint64_t i = b; i < e; ++i) {
      uint32_t rec[3];
      std::memcpy(rec, base + 12 * i, 12);
      if (rec[2] != 0) bad[t] = 1;  // an id above 32 bits: Idx::new asserts (index.rs:51-54)
      src[i] = rec[0];
      dst[i] = rec[1];
    }
  });
  for (int b : bad) GB_REQUIRE(b == 0, "Graph500 node id does not fit 32 bits");
  return GB_OK;
}

// The inverse: edges -> packed 12-byte records (high word 0 for 32-bit ids), the file format the
// reference's CLI reads with `-f graph500 --use-32-bit` (crates/app/src/runner.rs:104-133).
gb_status gb_graph500_encode(const uint32_t* src, const uint32_t* dst, uint64_t edge_count, void* bytes) {
  if (edge_count == 0) return GB_OK;
  GB_REQUIRE(src && dst && bytes, "NULL argument");
  const unsigned T = gb::io_threads(edge_count);
  uint8_t* base = static_cast<uint8_t*>(bytes);
  gb::parallel_chunks(T, [&](unsigned t) {
    const uint64_t b = edge_count * t / T, e = edge_count * (t + 1) / T;
    for (uint64_t i = b; i < e; ++i) {
      const uint32_t rec[3] = {src[i], dst[i], 0u};
      std::memcpy(base + 12 * i, rec, 12);
    }
  });
  return GB_OK;
}

// Two-phase use: call with src == NULL to obtain *edge_count, allocate, call again to fill.
// values may be NULL.  Ids above 32 bits are an error.
gb_status gb_edge_list_parse(const char* text, uint64_t len, uint32_t* src, uint32_t* dst, float* values,
                             uint64_t* edge_count) {
  GB_REQUIRE(edge_count, "NULL argument");
  *edge_count = 0;
  if (len == 0) return GB_OK;
  GB_REQUIRE(text != nullptr, "NULL text");
  // new_line_bytes, edgelist.rs:271-279
  uint64_t nl = 1;
  if (const void* first = std::memchr(text, '\n', len)) {
    const uint64_t i = (uint64_t)(static_cast<const char*>(first) - text);
    if (i > 0 && text[i - 1] == '\r') nl = 2;
  }
  // chunk boundaries moved forward to the next line start (edgelist.rs:193-212)
  const unsigned T = gb::io_threads(len / 8);
  std::vector<uint64_t> start(T + 1, len);
  start[0] = 0;
  for (unsigned t = 1; t < T; ++t) {
    uint64_t p = len * t / T;
    while (p < len && text[p - 1] != '\n') ++p;
    start[t] = std::max(p, start[t - 1]);
  }
  std::vector<uint64_t> count(T + 1, 0);
  std::vector<int> bad(T, 0);
  gb::parallel_chunks(T, [&](unsigned t) {
    uint64_t c = 0;
    for (uint64_t p = start[t]; p < start[t + 1];) {
      uint64_t s, d;
      float v;
      p = gb::parse_line(text, p, len, nl, &s, &d, &v);
      if (s > 0xFFFFFFFFull || d > 0xFFFFFFFFull) bad[t] = 1;
      ++c;
    }
    count[t + 1] = c;
  });
  for (int b : bad) GB_REQUIRE(b == 0, "edge list node id does not fit 32 bits");
  for (unsigned t = 0; t < T; ++t) count[t + 1] += count[t];
  *edge_count = count[T];
  if (!src) return GB_OK;
  GB_REQUIRE(dst != nullptr, "dst is NULL");
  gb::parallel_chunks(T, [&](unsigned t) {
    uint64_t i = count[t];
    for (uint64_t p = start[t]; p < start[t + 1]; ++i) {
      uint64_t s, d;
      float v;
      p = gb::parse_line(text, p, len, nl, &s, &d, &v);
      src[i] = (uint32_t)s;
      dst[i] = (uint32_t)d;
      if (values) values[i] = v;
    }
  });
  return GB_OK;
}

}  // extern "C"

namespace gb {

// Binary graph files (binary_format.h): the section table from the headers, then the labels (label_bytes != 0),
// the offsets and targets checked and narrowed to u32 on the host.  In-CSR values are never returned (device graphs
// hold none).
static gb_status binary_decode(const void* bytes, uint64_t len, gb_graph_kind kind, uint32_t label_bytes,
                               uint32_t* node_count, uint64_t* entries, int* has_values, uint32_t* labels,
                               uint32_t* out_offsets, uint32_t* out_targets, float* out_values, uint32_t* in_offsets,
                               uint32_t* in_targets) {
  GB_REQUIRE(node_count && entries && has_values, "NULL argument");
  GB_REQUIRE(kind == GB_KIND_DIRECTED || kind == GB_KIND_UNDIRECTED, "unknown graph kind %d", (int)kind);
  GB_REQUIRE(bytes || len == 0, "NULL bytes");
  const uint8_t* base = static_cast<const uint8_t*>(bytes);
  BinLayout l;
  GB_TRY(bin_parse([&](uint64_t pos, void* dst, uint64_t n) { return std::memcpy(dst, base + pos, n), true; }, len,
                   kind, &l, label_bytes));
  *node_count = l.n;
  *entries = l.entries;
  *has_values = l.values ? 1 : 0;
  if (!out_offsets) return GB_OK;
  GB_REQUIRE(labels || label_bytes == 0, "labels is NULL");
  GB_REQUIRE(out_targets || l.entries == 0, "out_targets is NULL");
  GB_REQUIRE(!out_values || l.values, "the file holds no edge values");
  GB_REQUIRE(kind == GB_KIND_UNDIRECTED || (in_offsets && (in_targets || l.entries == 0)), "in-CSR arrays are NULL");
  const uint64_t n = l.n, m = l.entries, w = l.id_bytes, rec = l.rec_bytes;
  for (uint64_t v = 0; v < n && label_bytes; ++v) {  // the labels first: they come first in the file
    uint64_t x = 0;
    std::memcpy(&x, base + BIN_USIZE + v * label_bytes, label_bytes);
    if (x > 0xFFFFFFFFull) return bin_label_wide(v);
    labels[v] = (uint32_t)x;
  }
  for (unsigned c = 0; c < l.ncsr; ++c) {
    const char* what = bin_csr_name(l, c);
    uint32_t* off = c == 0 ? out_offsets : in_offsets;
    uint32_t* tgt = c == 0 ? out_targets : in_targets;
    float* val = c == 0 ? out_values : nullptr;
    bool wide = false;
    auto id_at = [&](uint64_t pos) {
      uint64_t v = 0;
      std::memcpy(&v, base + pos, w);
      wide |= v > 0xFFFFFFFFull;
      return (uint32_t)v;
    };
    uint64_t decreasing = 0, big = 0;
    for (uint64_t v = 0; v <= n; ++v) {
      off[v] = id_at(l.csr[c].off_pos + v * w);
      if (v && off[v] < off[v - 1]) ++decreasing;
    }
    const unsigned T = io_threads(m);
    std::vector<uint64_t> big_t(T, 0);
    std::vector<int> wide_t(T, 0);
    parallel_chunks(T, [&](unsigned t) {
      uint64_t nbig = 0;  // counted in registers: big_t[t] and wide_t[t] of the threads share cache lines
      bool nwide = false;
      for (uint64_t i = m * t / T, e = m * (t + 1) / T; i < e; ++i) {
        const uint8_t* r = base + l.csr[c].rec_pos + i * rec;
        uint64_t v = 0;
        std::memcpy(&v, r, w);
        nwide |= v > 0xFFFFFFFFull;
        nbig += v >= n;
        tgt[i] = (uint32_t)v;
        if (val) std::memcpy(val + i, r + w, 4);
      }
      big_t[t] = nbig;
      wide_t[t] = nwide;
    });
    for (unsigned t = 0; t < T; ++t) big += big_t[t], wide |= wide_t[t] != 0;
    GB_REQUIRE(!wide, "binary graph file: %s holds an id or offset that does not fit 32 bits", what);
    GB_REQUIRE(off[0] == 0, "%s offsets[0] must be 0", what);
    GB_TRY(require_monotone(what, decreasing));
    GB_REQUIRE(off[n] == m, "%s offsets end at %u, not at its %llu entries", what, off[n], (unsigned long long)m);
    GB_TRY(require_ids(what, big, l.n));
  }
  return GB_OK;
}

}  // namespace gb

extern "C" {

gb_status gb_binary_decode(const void* bytes, uint64_t len, gb_graph_kind kind, uint32_t* node_count,
                           uint64_t* entries, int* has_values, uint32_t* out_offsets, uint32_t* out_targets,
                           float* out_values, uint32_t* in_offsets, uint32_t* in_targets) {
  return gb::binary_decode(bytes, len, kind, 0, node_count, entries, has_values, nullptr, out_offsets, out_targets,
                           out_values, in_offsets, in_targets);
}

// the NodeValues payload of label_bytes (4 or 8) per node in front of the CSRs; 8-byte labels are narrowed
gb_status gb_binary_decode_labeled(const void* bytes, uint64_t len, gb_graph_kind kind, uint32_t label_bytes,
                                   uint32_t* node_count, uint64_t* entries, int* has_values, uint32_t* labels,
                                   uint32_t* out_offsets, uint32_t* out_targets, float* out_values,
                                   uint32_t* in_offsets, uint32_t* in_targets) {
  GB_TRY(gb::bin_check_label_bytes(label_bytes));
  return gb::binary_decode(bytes, len, kind, label_bytes, node_count, entries, has_values, labels, out_offsets,
                           out_targets, out_values, in_offsets, in_targets);
}

}  // extern "C"
