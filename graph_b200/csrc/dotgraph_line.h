// dotgraph_line.h — the grammar of one line of a DotGraph (.graph) file, shared by the host reader (io.cu) and
// the device parser (load.cu), so that both accept and reject the same bytes with the same message.
//
// The reader of crates/builder/src/input/dotgraph.rs:136-203 is positional:
//   line 1          "t N M"                  the header
//   lines 2..N+1    "v <id> <label> <degree>" node lines in id order; the id is skipped, the label kept
//   lines N+2..N+M+1 "e <src> <dst>"          edges, in file order
// It skips 2 bytes at the start of every line without looking at them (example.graph tags its nodes `n`), then
// reads leading ASCII digits, skips exactly one byte between numbers, and never reads past line N+M+1.  Where
// the reference would panic or misread, the line is an error here: a number without digits (which includes a
// line too short to hold its numbers), a byte between the last number and the line end (a '\r' included), and a
// number >= 2^32.  The last line may lack its '\n'.
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define GB_HD __host__ __device__ __forceinline__
#else
#define GB_HD inline
#endif

namespace gb {

enum DotError : uint32_t {
  DOT_OK = 0,
  DOT_NO_DIGITS = 1,  // a number has no digits
  DOT_TRAILING = 2,   // bytes between the last number and the end of the line
  DOT_WIDE = 3,       // a number does not fit 32 bits
  DOT_MISSING = 4,    // the file ends before line N+M+1 (only the readers report it, not dot_line)
};

// Parses `count` numbers (2 or 3) of the line [p, eol) of text into v[]; DOT_OK or the line's error.
GB_HD uint32_t dot_line(const char* text, uint64_t p, uint64_t eol, int count, uint32_t* v) {
  p += 2;  // the tag byte and the byte after it, unread
  for (int k = 0; k < count; ++k) {
    if (k) p += 1;  // exactly one separator byte
    if (p >= eol || text[p] < '0' || text[p] > '9') return DOT_NO_DIGITS;
    uint64_t x = 0;
    while (p < eol && text[p] >= '0' && text[p] <= '9') {
      x = x * 10 + (uint64_t)(text[p++] - '0');
      if (x > 0xFFFFFFFFull) return DOT_WIDE;
    }
    v[k] = (uint32_t)x;
  }
  return p == eol ? (uint32_t)DOT_OK : (uint32_t)DOT_TRAILING;
}

// The error of 1-based line `line` as both readers report it; `line` 0 stands for the whole file (DOT_MISSING,
// with `have` lines found of `want`).
inline const char* dot_error_text(uint32_t code) {
  switch (code) {
    case DOT_NO_DIGITS: return "a number has no digits";
    case DOT_TRAILING: return "bytes follow the last number";
    case DOT_WIDE: return "a number does not fit 32 bits";
    default: return "malformed line";
  }
}

// The parsed header.  `lines` = 1 + N + M, the lines the reader reads.
struct DotHeader {
  uint32_t nodes = 0, edges = 0;
  uint64_t lines = 0;
  uint64_t body = 0;  // byte offset of line 2
};

// Whether a file of `len` bytes can hold the lines the header declares: a node line takes at least 7 bytes
// ("v 0 0 0") and an edge line 5 ("e 0 0"), each with a '\n' but the file's last.  The readers size their arrays
// by N and M only then.  Otherwise they parse without storing, which is bound to meet a missing or malformed line,
// so a header such as "t 4294967295 4294967295" costs no allocation and fails with the message it would anyway.
inline bool dot_fits(const DotHeader& h, uint64_t len) {
  return 8 * (uint64_t)h.nodes + 6 * (uint64_t)h.edges <= len - h.body + 1;
}

}  // namespace gb

#undef GB_HD
