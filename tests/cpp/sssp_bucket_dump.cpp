// Prints gb::sssp_next_bucket (graph_b200/csrc/sssp_bucket.h) for (dmin, delta, old_upper) triples read from
// stdin as f32 bit patterns in hex, one triple per line: "<lower bits> <upper bits> <steps>".  The port of the
// function in tools/sssp_model.py is compared against this output bit for bit.
#include <cstdint>
#include <cstdio>
#include <cstring>

#include "sssp_bucket.h"

static float from_bits(uint32_t u) {
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}

static uint32_t to_bits(float f) {
  uint32_t u;
  std::memcpy(&u, &f, 4);
  return u;
}

int main() {
  unsigned a, b, c;
  while (std::scanf("%x %x %x", &a, &b, &c) == 3) {
    const gb::SsspBucket r = gb::sssp_next_bucket(from_bits(a), from_bits(b), from_bits(c));
    std::printf("%08x %08x %d\n", to_bits(r.lower), to_bits(r.upper), r.steps);
  }
  return 0;
}
