// Shared declarations of the spatial-attention kernel (attn_spatial.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

namespace mimo {

constexpr int BKV = 128;                // keys per tile
constexpr int kChunkBytes = 128 * 128;  // one 64-element-wide (128 B) chunk of a 128-row tile

struct AttnArgs {
  int lq, lb, heads, d, dp;  // dp = d rounded up to 16
  int n_self_tiles, n_bank_tiles;
  float scale_log2;
  const int* bank_index;
  void* out;
  long long ld_out;
};

}  // namespace mimo
