// CPU check of the delta-stepping bucket advance (graph_b200/csrc/sssp_bucket.h): for every positive finite
// delta (subnormal ones included) and every distance from 0 to FLT_MAX the new bucket holds dmin, starts at
// or above the old upper bound, is not empty, and is found in a bounded number of steps.  Where the bucket
// index is small it is the bucket of width delta that sssp.rs:126 uses.
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#include "sssp_bucket.h"

static int failures = 0;
static long checked = 0;

static void fail(const char* what, float dmin, float delta, float old_upper, const gb::SsspBucket& b) {
  if (++failures <= 20)
    std::printf("FAIL %s: dmin %a delta %a old_upper %a -> [%a, %a) steps %d\n", what, dmin, delta, old_upper,
                b.lower, b.upper, b.steps);
}

static gb::SsspBucket check(float dmin, float delta, float old_upper) {
  const gb::SsspBucket b = gb::sssp_next_bucket(dmin, delta, old_upper);
  ++checked;
  if (!(old_upper <= b.lower && b.lower <= dmin && dmin < b.upper)) fail("bounds", dmin, delta, old_upper, b);
  if (!(b.upper > b.lower)) fail("empty", dmin, delta, old_upper, b);
  if (b.steps < 0 || b.steps > 2) fail("steps", dmin, delta, old_upper, b);
  // small index: exactly the bucket [delta k, delta (k + 1)) in f32 that holds dmin
  const float q = dmin / delta;
  if (q < 1048576.0f) {
    const float k0 = std::floor(q);
    for (float k = std::fmax(k0 - 2.0f, 0.0f); k <= k0 + 2.0f; k += 1.0f) {
      const float lo = delta * k, up = delta * (k + 1.0f);
      if (lo <= dmin && dmin < up && lo >= old_upper && (b.lower != lo || b.upper != up))
        fail("index bucket", dmin, delta, old_upper, b);
    }
  }
  return b;
}

static float from_bits(uint32_t u) {
  float f;
  std::memcpy(&f, &u, 4);
  return f;
}

int main() {
  std::vector<float> deltas = {from_bits(1), from_bits(2), from_bits(3), 1e-45f, 1e-44f, 1e-40f, 1e-38f,
                               FLT_MIN, 1e-30f, 1e-20f, 1e-12f, 1e-8f, 1e-3f, 0.05f, 0.3f, 1.0f, 1000.0f,
                               1e20f, 1e30f};
  for (float d = 1e-45f; d < 1e30f; d *= 7.3f) deltas.push_back(d);
  std::vector<float> dmins = {0.0f, from_bits(1), 1e-40f, FLT_MIN, 1e-8f, 0.5f, 1.0f, 3.0f, 5.0f, 1e30f,
                              FLT_MAX, std::nextafter(FLT_MAX, 0.0f)};
  for (float x = 1e-45f; x < 3e38f; x *= 3.1f) dmins.push_back(x);
  uint32_t rng = 12345u;
  for (int i = 0; i < 4000; ++i) {  // random finite non-negative bit patterns
    rng = rng * 1664525u + 1013904223u;
    const float x = from_bits(rng & 0x7FFFFFFFu);
    if (std::isfinite(x)) dmins.push_back(x);
  }
  for (float delta : deltas) {
    for (float dmin : dmins) {
      check(dmin, delta, 0.0f);
      check(dmin, delta, dmin);                     // the pile's minimum sits exactly at the old upper bound
      check(dmin, delta, std::nextafter(dmin, 0.0f));
      const gb::SsspBucket b = check(dmin, delta, 0.0f);
      if (b.upper < INFINITY) check(b.upper, delta, b.upper);  // the next distance just past the bucket
    }
    // a run of bucket advances, each finding its minimum right at the previous upper bound (the most
    // buckets a distance range can take), from the first bucket and from distances 0.5 .. 5
    for (float start : {0.0f, 0.5f, 5.0f}) {
      float upper = start == 0.0f ? delta : start;
      for (int i = 0; i < 2000 && upper < INFINITY; ++i) {
        const gb::SsspBucket b = check(upper, delta, upper);
        if (!(b.upper > upper)) {
          fail("no progress", upper, delta, upper, b);
          break;
        }
        upper = b.upper;
      }
    }
  }
  std::printf("sssp_bucket: %ld cases, %d failures\n", checked, failures);
  if (failures) return 1;
  std::printf("sssp_bucket ok\n");
  return 0;
}
