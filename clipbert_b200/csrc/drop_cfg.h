// Dropout configuration passed by value to every mask-drawing kernel (see the RNG helpers in common.cuh).
#pragma once
#include <stdint.h>

namespace cb {

struct DropCfg {
  uint32_t thresh;          // p * 65536 (0 = no dropout, 65536 = drop everything)
  float inv_keep;           // 1 / (1 - p), 0 when p >= 1
  uint64_t seed;
  const uint64_t* offset;   // device word added (times an odd constant) to the seed at run time, or nullptr
};

// process-wide device word bound by cb_dropout_offset_bind (api.cu); nullptr = seeds are used as passed
const uint64_t* drop_offset_ptr();

inline DropCfg make_drop(float p, uint64_t seed) {
  DropCfg d;
  d.seed = seed;
  d.offset = drop_offset_ptr();
  if (p >= 1.0f) {
    // nn.Dropout(p=1) returns zeros. No 16-bit lane reaches 65536, so every element is dropped; the multiplier of a kept
    // element would be 1 / 0 = inf, which turns a kept 0 into NaN.
    d.thresh = 65536u;
    d.inv_keep = 0.0f;
  } else if (p > 0.0f) {
    double t = static_cast<double>(p) * 65536.0 + 0.5;
    d.thresh = t >= 65535.0 ? 65535u : static_cast<uint32_t>(t);
    if (d.thresh == 0) d.thresh = 1;
    d.inv_keep = 1.0f / (1.0f - p);
  } else {
    d.thresh = 0;
    d.inv_keep = 1.0f;
  }
  return d;
}

}  // namespace cb
