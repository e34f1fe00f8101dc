// The weight norm of torch.nn.utils.weight_norm (dim 0), applied when a vocoder's weights are packed (dsx_hifigan.cu,
// dsx_pwg.cu).
#pragma once
#include "dsx_internal.h"

namespace dsx {
namespace {   // every translation unit has its own k_wnorm

// scale[i] = g[i] / ||v[i]|| over the `inner` elements of index i of dim 0 (torch._weight_norm, dim 0); 1 without g
__global__ void k_wnorm(const float* v, const float* g, int inner, float* scale) {
  const int i = blockIdx.x;
  float s = 0.f;
  if (g) {
    for (int e = threadIdx.x; e < inner; e += blockDim.x) {
      const float x = v[static_cast<size_t>(i) * inner + e];
      s = fmaf(x, x, s);
    }
  }
  __shared__ float red[32];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) t += red[w];
    scale[i] = g ? g[i] / sqrtf(t) : 1.f;
  }
}

}  // namespace
}  // namespace dsx
