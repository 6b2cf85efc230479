// edgelist_line.h — the grammar of one text edge-list line, as the host reader parses it (host only).
//
// This function is the specification of the format: the host reader (io.cu) calls it for every line,
// the device loader (load.cu) calls it for the lines whose value its fast parser declines, and the
// device parser (edgelist_scan.h) is tested against it byte for byte (tests/cpp/edgelist_scan_check.cpp).
#pragma once
#include <charconv>
#include <cstdint>
#include <cstring>

namespace gb {

// one line "<src><1 byte><dst>[ <value>]<newline>"; returns the position after the line.
// Nothing is read at or beyond the line's end (the buffer is a (pointer, length) pair, not a C string):
// the value is parsed by std::from_chars over [p, end of line) — bounded, locale-free, and like the
// reference's fast_float2::parse_partial (edgelist.rs:237-241) it takes the longest valid prefix.
static inline uint64_t parse_line(const char* text, uint64_t p, uint64_t len, uint64_t nl, uint64_t* s, uint64_t* t,
                                  float* v) {
  (void)nl;
  const void* nlp = std::memchr(text + p, '\n', len - p);
  const uint64_t eol = nlp ? (uint64_t)(static_cast<const char*>(nlp) - text) : len;  // position of '\n' (or len)
  uint64_t a = 0, b = 0;
  while (p < eol && text[p] >= '0' && text[p] <= '9') a = a * 10 + (uint64_t)(text[p++] - '0');
  if (p < eol) p += 1;  // exactly one separator byte (edgelist.rs:225)
  while (p < eol && text[p] >= '0' && text[p] <= '9') b = b * 10 + (uint64_t)(text[p++] - '0');
  float val = 0.0f;  // EV::default() when the column is missing (edgelist.rs:237-241)
  if (p < eol && text[p] == ' ') {
    ++p;
    if (p < eol && text[p] == '+') ++p;
    float parsed = 0.0f;
    const auto res = std::from_chars(text + p, text + eol, parsed);
    if (res.ec == std::errc() || res.ec == std::errc::result_out_of_range) val = parsed;
  }
  *s = a;
  *t = b;
  *v = val;
  return eol < len ? eol + 1 : len;
}

}  // namespace gb
