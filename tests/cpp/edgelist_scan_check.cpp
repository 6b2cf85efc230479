// The device loader's line parser (graph_b200/csrc/edgelist_scan.h) against the host reader's
// gb::parse_line (edgelist_line.h), on the CPU.  Every line must give the same ids and the same end
// position; every value the fast path accepts must be bit-equal to parse_line's, and on values printed with
// %g, %.6f, %.9g and as the shortest round-trip string of a float32 (Python's repr) it may decline < 1 %.
#include <charconv>
#include <cinttypes>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "edgelist_line.h"
#include "edgelist_scan.h"

static uint64_t g_lines = 0, g_declined = 0, g_failures = 0;

static uint32_t fbits(float f) {
  uint32_t b;
  std::memcpy(&b, &f, 4);
  return b;
}

// parses all of text with both parsers, line by line; returns the number of declined values
static uint64_t compare_text(const std::string& text, bool verbose_fail = true) {
  uint64_t p = 0, declined = 0;
  const uint64_t len = text.size();
  while (p < len) {
    uint64_t s, t;
    float v;
    const uint64_t next = gb::parse_line(text.data(), p, len, 1, &s, &t, &v);
    gb::ScannedLine sl;
    const uint64_t next2 = gb::scan_line(text.data(), p, len, true, &sl);
    gb::ScannedLine ids_only;
    const uint64_t next3 = gb::scan_line(text.data(), p, len, false, &ids_only);
    ++g_lines;
    bool ok = next == next2 && next == next3 && sl.src == s && sl.dst == t && ids_only.src == s &&
              ids_only.dst == t && !ids_only.declined && ids_only.value == 0.0f;
    if (sl.declined) {
      ++declined;
      ok = ok && sl.value == 0.0f;
    } else {
      ok = ok && fbits(sl.value) == fbits(v);
    }
    if (!ok) {
      ++g_failures;
      if (verbose_fail && g_failures <= 20) {
        std::string line = text.substr(p, next - p);
        for (auto& c : line)
          if (c == '\n') c = '|';
        std::printf("MISMATCH line [%s]: host (%" PRIu64 ", %" PRIu64 ", %08x, next %" PRIu64 ") scan (%" PRIu64
                    ", %" PRIu64 ", %08x, declined %d, next %" PRIu64 ")\n",
                    line.c_str(), s, t, fbits(v), next, sl.src, sl.dst, fbits(sl.value), (int)sl.declined, next2);
      }
    }
    p = next;
  }
  g_declined += declined;
  return declined;
}

static std::string fmt(const char* f, double x) {
  char buf[128];
  std::snprintf(buf, sizeof buf, f, x);
  return buf;
}

static std::string shortest(float x) {  // the digits Python's repr prints for float(np.float32(x))
  char buf[64];
  auto r = std::to_chars(buf, buf + sizeof buf, (double)x);
  return std::string(buf, r.ptr);
}

int main() {
  // ---- adversarial corpus --------------------------------------------------------------------------
  const char* corpus[] = {
      "", "\n", "\n\n", "0 1\n", "0 1", "0 1 \n", "0 1 \r\n", "0 1\r\n", "0 1 2.5\r\n", "0 1 2.5\r", "0\n",
      "0 \n", "5", "7 ", "12\t34 1.5\n", "1,2 3\n", "1  2 3\n", "1 2  3\n", "1 2 +3\n", "1 2 ++3\n", "1 2 +-3\n",
      "1 2 -3\n", "1 2 -\n", "1 2 -.5\n", "1 2 .5\n", "1 2 5.\n", "1 2 5.e3\n", "1 2 1e\n", "1 2 1e+\n",
      "1 2 1e-\n", "1 2 1E5\n", "1 2 1e5x\n", "1 2 1.5abc\n", "1 2 1.5 7\n", "1 2 1.2.3\n", "1 2 1e50\n",
      "1 2 -1e50\n", "1 2 1e39\n", "1 2 3.4028235e38\n", "1 2 3.4028234e38\n", "1 2 3.40282357e38\n",
      "1 2 1e-30\n", "1 2 1e-38\n", "1 2 1e-40\n", "1 2 1e-45\n", "1 2 1e-46\n", "1 2 1.17549435e-38\n",
      "1 2 inf\n", "1 2 -inf\n", "1 2 infinity\n", "1 2 nan\n", "1 2 NaN\n", "1 2 nan(123)\n", "1 2 0x1p3\n",
      "1 2 0X10\n", "1 2 0x\n", "1 2 0\n", "1 2 -0\n", "1 2 0.0\n", "1 2 -0.0e5\n", "1 2 000001.5000\n",
      "1 2 0.1\n", "1 2 0.2\n", "1 2 0.3\n", "1 2 16777217\n", "1 2 16777219\n", "1 2 16777218.5\n",
      "1 2 33554435\n", "1 2 1.00000005960464477539\n", "1 2 1.0000000596046447\n", "1 2 1.0000000596046448\n",
      "1 2 1.00000011920928955\n", "1 2 1.000000059604644775390625\n", "1 2 0.100000001490116119384765625\n",
      "1 2 12345678901234567890\n", "1 2 1234567890123456789\n", "1 2 9007199254740993\n",
      "1 2 1e22\n", "1 2 1e23\n", "1 2 1e-22\n", "1 2 1e-23\n", "1 2 123456789e-30\n",
      "123456789012345678901 2\n", "18446744073709551615 18446744073709551616\n", "4294967295 4294967296\n",
      "4294967296 0 1.5\n", "99999999999999999999999 1 1\n", "a b c\n", "1 2 \x01\n", "1 2 1e5\r\n\r\n",
      "\r\n", "1 2 3\n4 5 6", "1 2 1e0000000000000000000000000001\n", "1 2 1.5e-0\n", "1 2 1.5E+00\n",
  };
  for (const char* c : corpus) compare_text(c);
  {
    std::string all;
    for (const char* c : corpus) all += c;
    compare_text(all);
  }
  // exact float midpoints (as shortest / exact decimal strings) and their neighbours
  {
    std::mt19937_64 rng(7);
    std::string text;
    for (int i = 0; i < 200000; ++i) {
      const uint32_t b = (uint32_t)(rng() % 0x7F000000u) + 0x00800000u;
      float f;
      std::memcpy(&f, &b, 4);
      const double mid = (double)f + std::ldexp(1.0, std::ilogb(f) - 24);
      for (double x : {mid, std::nextafter(mid, 0.0), std::nextafter(mid, 1e300)}) {
        text += "3 4 ";
        text += fmt((i & 1) ? "%.17g" : "%.25g", x);
        text += (i & 2) ? "\r\n" : "\n";
      }
    }
    compare_text(text);
  }
  // ---- random tokens ------------------------------------------------------------------------------
  {
    std::mt19937_64 rng(12345);
    const char alphabet[] = "0123456789012345678901234567890123456789.eE+-  \r\nxXinfa\t";
    std::string text;
    uint64_t tokens = 0;
    while (tokens < 10000000) {
      text.clear();
      for (int i = 0; i < 100000; ++i, ++tokens) {
        const int kind = (int)(rng() % 8);
        text += std::to_string(rng() % 100000);
        text += ' ';
        text += std::to_string(rng() % 100000);
        if (kind == 0) {  // garbage of random length
          text += ' ';
          const int n = (int)(rng() % 24);
          for (int k = 0; k < n; ++k) text += alphabet[rng() % (sizeof alphabet - 1)];
        } else if (kind == 1) {  // random bit pattern, every printf form
          const uint32_t b = (uint32_t)rng();
          float f;
          std::memcpy(&f, &b, 4);
          static const char* forms[] = {"%g", "%.6f", "%.9g", "%.17g", "%e", "%.3e", "%a"};
          text += ' ';
          text += fmt(forms[rng() % 7], (double)f);
        } else if (kind == 2) {  // digit strings with a point and an exponent
          text += ' ';
          if (rng() % 4 == 0) text += '-';
          const int n = 1 + (int)(rng() % 24);
          for (int k = 0; k < n; ++k) text += (char)('0' + rng() % 10);
          if (rng() % 2) {
            text += '.';
            const int f = (int)(rng() % 24);
            for (int k = 0; k < f; ++k) text += (char)('0' + rng() % 10);
          }
          if (rng() % 3 == 0) {
            text += (rng() % 2) ? 'e' : 'E';
            const int s = (int)(rng() % 3);
            if (s) text += s == 1 ? '-' : '+';
            text += std::to_string(rng() % 60);
          }
        } else if (kind == 3) {  // huge ids (wrap-around, > 32 bits)
          text += std::to_string(rng());
          text += std::to_string(rng() % 1000);
        } else {  // plain values
          const float f = (float)std::ldexp((double)(rng() >> 11) / 9007199254740992.0, (int)(rng() % 60) - 30);
          text += ' ';
          text += (kind == 4) ? fmt("%g", f) : (kind == 5) ? fmt("%.9g", f) : (kind == 6) ? shortest(f) : fmt("%.6f", f);
        }
        text += (rng() % 5 == 0) ? "\r\n" : "\n";
      }
      compare_text(text);
      if (g_failures) break;
    }
    std::printf("random tokens: %" PRIu64 "\n", tokens);
  }
  // ---- decline rate on printed float32 values -----------------------------------------------------
  // values: half uniform in (0, 1), half log-uniform in [1e-6, 1e6], one in ten negative
  int rate_fail = 0;
  {
    const char* names[] = {"%g", "%.6f", "%.9g", "repr"};
    for (int form = 0; form < 4; ++form) {
      std::mt19937_64 rng(99 + form);
      std::uniform_real_distribution<double> u01(0.0, 1.0);
      std::string text;
      const int N = 1000000;
      for (int i = 0; i < N; ++i) {
        double x = (i & 1) ? u01(rng) : std::pow(10.0, -6.0 + 12.0 * u01(rng));
        if (rng() % 10 == 0) x = -x;
        const float f = (float)x;
        text += "1 2 ";
        text += form == 0 ? fmt("%g", f) : form == 1 ? fmt("%.6f", f) : form == 2 ? fmt("%.9g", f) : shortest(f);
        text += '\n';
      }
      const uint64_t d = compare_text(text);
      const double rate = (double)d / N;
      std::printf("decline rate %-5s %.5f%%\n", names[form], 100.0 * rate);
      if (rate >= 0.01) rate_fail = 1;
    }
  }
  std::printf("lines %" PRIu64 ", declined %" PRIu64 ", mismatches %" PRIu64 "\n", g_lines, g_declined, g_failures);
  if (g_failures || rate_fail) return 1;
  std::printf("edgelist_scan ok\n");
  return 0;
}
