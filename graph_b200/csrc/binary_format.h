// binary_format.h — the section table of the reference's binary graph files, shared by the host decoder
// (io.cu), the streamed device loader and the writer (load.cu).
//
// SerializeGraphOp / DeserializeGraphOp (crates/builder/src/graph_ops.rs:232-238) write, little-endian, with
// usize = 8 bytes:
//
//   NodeValues (csr.rs:334-341; NV = (), so no payload)   [usize n]
//   per CSR (directed: csr_out, csr_inc; undirected: csr), Csr::serialize csr.rs:252-266:
//     [usize L][L bytes: type name of NI, "u32" | "u64" | "usize"]
//     [NI node_count][NI entries]                       entries = targets.len() (undirected: 2m)
//     [NI offsets x (node_count + 1)]
//     [Target<NI, EV> x entries]                        #[repr(C)] (graph/mod.rs:6-10): (u32,()) 4 B,
//                                                       (u32,f32) 8 B, (u64,()) 8 B, (u64,f32) 16 B
//
// Nothing is aligned: the offsets of a u32 directed file start at byte 27.  The file does not say whether the
// records carry values; the record size follows from the header counts and the file size.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>

#include "common.cuh"

namespace gb {

constexpr uint64_t BIN_USIZE = 8;
constexpr uint64_t BIN_MAX_NAME = 64;  // longer type names are read only this far, for the message

// one CSR of the file: byte offsets of its parts
struct BinCsr {
  uint64_t header = 0;   // [usize L]
  uint64_t off_pos = 0;  // offsets[0]
  uint64_t rec_pos = 0;  // the first Target record
  uint64_t end = 0;      // one past the last record
};

struct BinLayout {
  gb_graph_kind kind = GB_KIND_DIRECTED;
  uint32_t id_bytes = 4;   // 4: "u32", 8: "u64" / "usize"
  uint32_t rec_bytes = 4;  // id_bytes without values; 8 (u32,f32) or 16 (u64,f32: 4 padding bytes) with
  bool values = false;
  uint32_t n = 0;
  uint64_t entries = 0;  // targets per CSR
  unsigned ncsr = 1;
  BinCsr csr[2];
  uint64_t file_bytes = 0;
  std::string name;  // NI's type name
};

inline uint32_t bin_value_rec_bytes(uint32_t id_bytes) { return id_bytes == 4 ? 8 : 16; }

// the parts of a CSR whose header starts at `header`
inline BinCsr bin_csr_at(uint64_t header, uint64_t name_len, uint32_t id_bytes, uint64_t n, uint64_t entries,
                         uint32_t rec_bytes) {
  BinCsr c;
  c.header = header;
  c.off_pos = header + BIN_USIZE + name_len + 2ull * id_bytes;
  c.rec_pos = c.off_pos + (n + 1) * id_bytes;
  c.end = c.rec_pos + entries * rec_bytes;
  return c;
}

// the file this library writes: NI = u32, records with values when `values`
inline BinLayout bin_layout_u32(gb_graph_kind kind, uint32_t n, uint64_t entries, bool values) {
  BinLayout l;
  l.kind = kind;
  l.id_bytes = 4;
  l.rec_bytes = values ? bin_value_rec_bytes(4) : 4;
  l.values = values;
  l.n = n;
  l.entries = entries;
  l.ncsr = kind == GB_KIND_DIRECTED ? 2 : 1;
  l.name = "u32";
  uint64_t pos = BIN_USIZE;
  for (unsigned c = 0; c < l.ncsr; ++c) {
    l.csr[c] = bin_csr_at(pos, 3, 4, n, entries, l.rec_bytes);
    pos = l.csr[c].end;
  }
  l.file_bytes = pos;
  return l;
}

// the header bytes in front of CSR c's offsets (with the NodeValues count in front of the first)
inline std::string bin_header_bytes(const BinLayout& l, unsigned c) {
  std::string h;
  auto put = [&](uint64_t v, unsigned bytes) { h.append(reinterpret_cast<const char*>(&v), bytes); };
  if (c == 0) put(l.n, BIN_USIZE);
  put(l.name.size(), BIN_USIZE);
  h += l.name;
  put(l.n, l.id_bytes);
  put(l.entries, l.id_bytes);
  return h;
}

inline const char* bin_kind_name(gb_graph_kind k) { return k == GB_KIND_DIRECTED ? "directed" : "undirected"; }
inline const char* bin_csr_name(const BinLayout& l, unsigned c) {
  return l.kind == GB_KIND_UNDIRECTED ? "csr" : (c == 0 ? "csr_out" : "csr_inc");
}

struct BinHeader {
  int err = 0;  // 0: read, 1: the file ends inside it, 2: unknown type name
  uint64_t name_len = 0, n = 0, entries = 0;
  uint32_t id_bytes = 0;
  std::string name;
};

// read(pos, dst, len) -> bool reads len bytes at pos; the callers below never ask past `size`
template <typename Read>
bool bin_get(Read& read, uint64_t size, uint64_t pos, unsigned bytes, uint64_t* v) {
  *v = 0;
  if (pos > size || size - pos < bytes) return false;
  return read(pos, v, bytes);  // little-endian host
}

template <typename Read>
BinHeader bin_read_header(Read& read, uint64_t size, uint64_t pos) {
  BinHeader h;
  if (!bin_get(read, size, pos, BIN_USIZE, &h.name_len) || h.name_len > size - pos - BIN_USIZE) {
    h.err = 1;
    return h;
  }
  h.name.resize(std::min(h.name_len, BIN_MAX_NAME));
  if (!h.name.empty() && !read(pos + BIN_USIZE, &h.name[0], h.name.size())) {
    h.err = 1;
    return h;
  }
  if (h.name == "u32") h.id_bytes = 4;
  else if (h.name == "u64" || h.name == "usize") h.id_bytes = 8;
  if (h.id_bytes == 0 || h.name_len != h.name.size()) {
    h.err = 2;
    return h;
  }
  const uint64_t p = pos + BIN_USIZE + h.name_len;
  if (!bin_get(read, size, p, h.id_bytes, &h.n) || !bin_get(read, size, p + h.id_bytes, h.id_bytes, &h.entries))
    h.err = 1;
  return h;
}

inline gb_status bin_eof() { return fail(GB_ERR_INVALID, "binary graph file: unexpected end of file"); }

inline gb_status bin_header_error(const BinHeader& h) {
  if (h.err == 1) return bin_eof();
  std::string shown;  // Error::InvalidIdType, lib.rs:297-298
  for (char ch : h.name) shown += (ch >= 32 && ch < 127 && ch != '"') ? ch : '?';
  if (h.name_len > h.name.size()) shown += "...";
  return fail(GB_ERR_INVALID, "invalid id size, expected \"u32\" bytes, got \"%s\" bytes", shown.c_str());
}

// Walks the headers of a file of `size` bytes that should hold a graph of kind `want`, and fills the section
// table.  Checks everything the headers decide: type names, the NodeValues count (lib.rs:295), node_count > 0,
// counts that fit 32 bits, equal csr_out / csr_inc counts, the graph kind, and that the sections end exactly
// at the end of the file.  The offsets and targets themselves are checked by the callers.
template <typename Read>
gb_status bin_parse(Read read, uint64_t size, gb_graph_kind want, BinLayout* l) {
  uint64_t nv = 0;
  if (!bin_get(read, size, 0, BIN_USIZE, &nv)) return bin_eof();
  const BinHeader h = bin_read_header(read, size, BIN_USIZE);
  if (h.err) return bin_header_error(h);
  const uint32_t w = h.id_bytes;
  GB_REQUIRE(h.n <= 0xFFFFFFFFull, "binary graph file: node_count %llu does not fit 32 bits",
             (unsigned long long)h.n);
  GB_REQUIRE(nv == h.n, "number of node values must be the same as node count");
  GB_REQUIRE(h.n > 0, "binary graph file: node_count must be > 0");
  GB_REQUIRE(h.entries < 0xFFFFFFFFull, "binary graph file: %llu entries do not fit u32 offsets",
             (unsigned long long)h.entries);
  const uint32_t cand[2] = {w, bin_value_rec_bytes(w)};
  BinCsr first[2];
  for (int i = 0; i < 2; ++i) first[i] = bin_csr_at(BIN_USIZE, h.name_len, w, h.n, h.entries, cand[i]);
  if (first[0].rec_pos > size) return bin_eof();  // inside the header or the offsets

  l->kind = want;
  l->id_bytes = w;
  l->n = (uint32_t)h.n;
  l->entries = h.entries;
  l->name = h.name;
  l->file_bytes = size;
  auto choose = [&](int i) {
    l->rec_bytes = cand[i];
    l->values = i == 1 && h.entries > 0;  // without entries the two record sizes give the same file
    l->csr[0] = first[i];
  };
  // the csr_inc header a directed file has after csr_out's records, for either record size
  BinHeader second[2];
  for (int i = 0; i < 2; ++i) second[i] = bin_read_header(read, size, first[i].end);
  const int undirected_fit = size == first[0].end ? 0 : size == first[1].end ? 1 : -1;

  if (want == GB_KIND_UNDIRECTED) {
    l->ncsr = 1;
    if (undirected_fit >= 0) {
      choose(undirected_fit);
      return GB_OK;
    }
    for (int i = 0; i < 2; ++i) {
      if (second[i].err || second[i].name != h.name || second[i].n != h.n || second[i].entries != h.entries) continue;
      if (bin_csr_at(first[i].end, second[i].name_len, w, h.n, h.entries, cand[i]).end == size)
        return fail(GB_ERR_INVALID, "binary graph file holds a directed graph, not an undirected one");
    }
    if (size < first[0].end) return bin_eof();
    if (size > first[1].end)
      return fail(GB_ERR_INVALID, "binary graph file: %llu trailing bytes after the last CSR",
                  (unsigned long long)(size - first[1].end));
    return fail(GB_ERR_INVALID,
                "binary graph file: the targets end neither with %u- nor with %u-byte records "
                "(unexpected end of file or trailing bytes)", cand[0], cand[1]);
  }

  l->ncsr = 2;
  int pick = second[0].err == 0 ? 0 : second[1].err == 0 ? 1 : -1;
  if (pick < 0) {
    if (undirected_fit >= 0)
      return fail(GB_ERR_INVALID, "binary graph file holds an undirected graph, not a directed one");
    // a csr_inc header with a bad name: its csr_inc, read like csr_out, would end at the end of the file
    for (int i = 0; i < 2 && pick < 0; ++i)
      if (second[i].err == 2 &&
          bin_csr_at(first[i].end, second[i].name_len, w, h.n, h.entries, cand[i]).end == size)
        pick = i;
    if (pick < 0) return bin_eof();
  }
  choose(pick);
  const BinHeader& h2 = second[pick];
  if (h2.err) return bin_header_error(h2);
  GB_REQUIRE(h2.name == h.name, "binary graph file: csr_out and csr_inc differ in id type (%s, %s)",
             h.name.c_str(), h2.name.c_str());
  GB_REQUIRE(h2.n == h.n, "binary graph file: csr_out and csr_inc differ in node_count (%llu, %llu)",
             (unsigned long long)h.n, (unsigned long long)h2.n);
  GB_REQUIRE(h2.entries == h.entries, "binary graph file: csr_out and csr_inc differ in entries (%llu, %llu)",
             (unsigned long long)h.entries, (unsigned long long)h2.entries);
  l->csr[1] = bin_csr_at(first[pick].end, h2.name_len, w, h.n, h.entries, cand[pick]);
  if (size < l->csr[1].end) return bin_eof();
  GB_REQUIRE(size == l->csr[1].end, "binary graph file: %llu trailing bytes after the last CSR",
             (unsigned long long)(size - l->csr[1].end));
  return GB_OK;
}

}  // namespace gb
