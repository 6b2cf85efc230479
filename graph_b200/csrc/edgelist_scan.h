// edgelist_scan.h — the device loader's parser of one text edge-list line (host and device).
//
// It reads the same grammar as gb::parse_line (edgelist_line.h), which is the specification:
//   - the line ends at the first '\n' or at the end of the buffer; a '\r' before the '\n' stays in the line;
//   - ids are the leading decimal digits, accumulated in uint64_t with wrap-around, and exactly one separator
//     byte of any value follows the source id;
//   - a value is read only when the byte after the target id is ' ', after one optional '+'.
// Ids are parsed exactly as there.  For the value, std::from_chars (longest valid prefix, round to nearest)
// is not available on the device, so scan_value takes a fast path that is exact or declines:
//   [-]digits[.digits][(e|E)[+-]digits] with at most 19 significant digits and |exponent| <= 22 is
//   evaluated as w * 10^q or w / 10^-q in double (10^q is exact; so is w up to 2^53, and above that the
//   double is within one ulp).  The result is within 2 double ulps of the decimal value, so (float)d is the
//   correctly rounded float unless d lies within 16 double ulps of a float rounding midpoint — the only
//   place rounding twice can differ from rounding once — or outside the normal float range.  Those cases,
//   and everything the grammar above does not cover (inf, nan, hex-looking input, "5.", ".5", an
//   incomplete exponent, more digits, larger exponents, an empty value), are declined: the loader re-parses
//   declined lines with gb::parse_line on the host, so every value is bit-identical to the host reader.
#pragma once
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define GB_HD __host__ __device__
#else
#define GB_HD
#endif

namespace gb {

GB_HD inline bool scan_is_digit(char c) { return c >= '0' && c <= '9'; }

// 10^k for 0 <= k <= 22, exact: every factor and partial product is a power of ten below 2^53 * 2^22
GB_HD inline double scan_pow10(int k) {
  double r = 1.0, b = 10.0;
  while (k) {
    if (k & 1) r *= b;
    b *= b;
    k >>= 1;
  }
  return r;
}

// The value over [p, eol): true and *out = the float std::from_chars gives, or false (declined).
GB_HD inline bool scan_value(const char* text, uint64_t p, uint64_t eol, float* out) {
  bool neg = false;
  if (p < eol && text[p] == '-') {
    neg = true;
    ++p;
  }
  if (!(p < eol && scan_is_digit(text[p]))) return false;  // empty, ".5", "inf", "nan", a second sign, ...
  uint64_t w = 0;  // significant digits
  int nd = 0;      // how many (leading zeros are not significant)
  int q = 0;       // decimal exponent of w
  while (p < eol && scan_is_digit(text[p])) {
    const int dg = text[p++] - '0';
    if (nd == 0 && dg == 0) continue;
    if (nd == 19) return false;
    w = w * 10 + (uint64_t)dg;
    ++nd;
  }
  if (p < eol && text[p] == '.') {
    ++p;
    if (!(p < eol && scan_is_digit(text[p]))) return false;  // "5." / "5.e3"
    while (p < eol && scan_is_digit(text[p])) {
      const int dg = text[p++] - '0';
      if (q == -64) return false;
      --q;
      if (nd == 0 && dg == 0) continue;
      if (nd == 19) return false;
      w = w * 10 + (uint64_t)dg;
      ++nd;
    }
  }
  if (p < eol && (text[p] == 'e' || text[p] == 'E')) {
    ++p;
    bool eneg = false;
    if (p < eol && (text[p] == '+' || text[p] == '-')) eneg = text[p++] == '-';
    if (!(p < eol && scan_is_digit(text[p]))) return false;  // incomplete exponent: the prefix ends before 'e'
    int e = 0;
    while (p < eol && scan_is_digit(text[p])) {
      if (e < 1000) e = e * 10 + (text[p] - '0');
      ++p;
    }
    q += eneg ? -e : e;
  }
  // whatever follows ends the number (from_chars stops there); "0x1p3" reads as 0, but decline hex-looking input
  if (p < eol && (text[p] == 'x' || text[p] == 'X')) return false;
  if (w == 0) {
    *out = neg ? -0.0f : 0.0f;
    return true;
  }
  if (q < -22 || q > 22) return false;
  double d = (double)w;
  const double pw = scan_pow10(q < 0 ? -q : q);
  d = q < 0 ? d / pw : d * pw;
  if (!(d >= 0x1p-125 && d <= 0x1p127)) return false;  // normal floats only, with a margin at both ends
  uint64_t bits;
  memcpy(&bits, &d, sizeof bits);
  // the 29 mantissa bits a float drops: 2^28 is exactly half a float ulp
  const int64_t r = (int64_t)(bits & 0x1FFFFFFFull) - (int64_t)(1ull << 28);
  if (r >= -16 && r <= 16) return false;
  const float f = (float)d;
  *out = neg ? -f : f;
  return true;
}

struct ScannedLine {
  uint64_t src, dst;
  float value;    // 0.0f when there is no value column or the value was declined
  bool declined;  // the value must be re-parsed with gb::parse_line
};

// One line starting at p of text[0, len); returns the position after the line, like gb::parse_line.
// want_value = false skips the value column (nothing is declined then).
GB_HD inline uint64_t scan_line(const char* text, uint64_t p, uint64_t len, bool want_value, ScannedLine* out) {
  uint64_t eol = p;
  while (eol < len && text[eol] != '\n') ++eol;
  uint64_t a = 0, b = 0;
  while (p < eol && scan_is_digit(text[p])) a = a * 10 + (uint64_t)(text[p++] - '0');
  if (p < eol) p += 1;
  while (p < eol && scan_is_digit(text[p])) b = b * 10 + (uint64_t)(text[p++] - '0');
  float val = 0.0f;
  bool declined = false;
  if (want_value && p < eol && text[p] == ' ') {
    ++p;
    if (p < eol && text[p] == '+') ++p;
    if (!scan_value(text, p, eol, &val)) {
      val = 0.0f;
      declined = true;
    }
  }
  out->src = a;
  out->dst = b;
  out->value = val;
  out->declined = declined;
  return eol < len ? eol + 1 : len;
}

}  // namespace gb
