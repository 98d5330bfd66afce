// Shared definitions of the attention kernel (attention.cu).
#pragma once

#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include "common.cuh"
#include "host.h"

namespace dk {

constexpr int ATT_BQ = 128;
constexpr int ATT_BKV = 128;

struct AttParams {
  int B, S, heads, split;
  float scale_log2;  // scale * log2(e)
  void* out0;
  long long ld0;
  void* out1;
  long long ld1;
};

// one 128-row Q tile per CTA, K / V ring of KS tiles of 128 keys
template <int D>
struct AttCfg {
  static constexpr int KS = 2;
  static constexpr int TILE_BYTES = 128 * D * 2;
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = TILE_BYTES;
  static constexpr int OFF_V = OFF_K + KS * TILE_BYTES;
  static constexpr int OFF_BAR = OFF_V + KS * TILE_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
};

}  // namespace dk
