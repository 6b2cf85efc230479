// sssp_bucket.h — the host-side bucket advance of delta-stepping (sssp.cu), kept free of CUDA so that it
// can be tested on the CPU.
//
// The bounds of bucket k are delta * k and delta * (k + 1), rounded to f32 like sssp.rs:126.  For an index
// below 2^22, f32 holds k and k + 1 exactly and their products with delta are strictly increasing, so the
// bucket that holds dmin is found from floor(dmin / delta) in at most one correction step each way.  Past
// that (a delta tiny against the distances: dmin / delta can even overflow to inf for a subnormal delta)
// consecutive indices no longer give distinct bounds, and the bucket becomes [dmin, next f32 above dmin).
// The kernels stay exact whatever the bucket widths are: f32 `+` is monotone and weights are >= 0, so the
// fixed point dist[t] = min fl(dist[u] + w) is unique (sssp.cu) and only the number of passes depends on
// the bounds.
#pragma once

#include <cmath>

namespace gb {

struct SsspBucket {
  float lower, upper;
  int steps;  // index corrections taken (at most 2)
};

// the next bucket after one whose upper bound was old_upper; dmin (>= old_upper) is the smallest live
// distance left.  Returns old_upper <= lower <= dmin < upper, for every positive finite delta.
inline SsspBucket sssp_next_bucket(float dmin, float delta, float old_upper) {
  SsspBucket b{dmin, std::nextafter(dmin, INFINITY), 0};
  const float q = dmin / delta;           // dest_bin = (nd / delta) as usize, sssp.rs:190
  if (!(q < 4194304.0f)) return b;         // 2^22; also inf
  float k = std::floor(q);
  float lo = delta * k, up = delta * (k + 1.0f);
  if (!(dmin < up)) {
    k += 1.0f;
    lo = up;
    up = delta * (k + 1.0f);
    b.steps = 1;
  } else if (dmin < lo) {
    k -= 1.0f;
    up = lo;
    lo = delta * k;
    b.steps = 1;
  }
  if (old_upper <= lo && lo <= dmin && dmin < up) {
    b.lower = lo;
    b.upper = up;
  }
  return b;
}

}  // namespace gb
