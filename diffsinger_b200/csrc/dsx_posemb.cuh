// Sinusoidal position embedding of the pitch extractor (dsx_pe.cu) and the FastSpeech2 decoder (dsx_fs2dec.cu):
// the positions are make_positions over channel 0 of the input (utils/__init__.py:145-157, padding_idx 0), the table is
// SinusoidalPositionalEmbedding.get_embedding (modules/commons/common_layers.py:106-122) evaluated in fp32 on the fly, so
// it has no size limit and the reference's regrowth past its initial size (:127-135) needs no counterpart.
#pragma once
#include <math.h>

#include "dsx_internal.h"

namespace dsx {
namespace {   // every translation unit has its own kernels

// pos[b][t] = cumsum(x[b, :, 0] != 0)[t] * (x[b, t, 0] != 0) over contiguous x [B][T][n].  One block per utterance,
// kScanChunk frames per thread per pass.
constexpr int kScanThreads = 1024, kScanChunk = 8;
__global__ void __launch_bounds__(kScanThreads) k_pos_scan(const float* x, int T, int n, int* pos) {
  __shared__ int sh[kScanThreads];
  const int b = blockIdx.x, tid = threadIdx.x;
  const float* xb = x + static_cast<size_t>(b) * T * n;
  int carry = 0;
  for (int base = 0; base < T; base += kScanThreads * kScanChunk) {
    const int t0 = base + tid * kScanChunk, t1 = min(T, t0 + kScanChunk);
    int local = 0;
    for (int t = t0; t < t1; ++t) local += xb[static_cast<size_t>(t) * n] != 0.f;
    sh[tid] = local;
    __syncthreads();
    for (int off = 1; off < kScanThreads; off <<= 1) {
      const int v = tid >= off ? sh[tid - off] : 0;
      __syncthreads();
      sh[tid] += v;
      __syncthreads();
    }
    int s = carry + sh[tid] - local;
    for (int t = t0; t < t1; ++t) {
      const bool nz = xb[static_cast<size_t>(t) * n] != 0.f;
      s += nz;
      pos[static_cast<size_t>(b) * T + t] = nz ? s : 0;
    }
    carry += sh[kScanThreads - 1];
    __syncthreads();
  }
}

// -ln(1e4) / (n / 2 - 1): the frequency exponent step of an n-channel table
inline float pos_neg_emb(int n) { return -static_cast<float>(log(10000.0) / (n / 2 - 1)); }

// table[ps][c] = [sin(ps f_i), cos(ps f_i)], f_i = exp(i * neg_emb), row 0 = 0, with the full-range sinf / cosf
__device__ __forceinline__ float pos_table(int ps, int c, int n, float neg_emb) {
  if (ps == 0) return 0.f;
  const int half = n / 2, fi = c < half ? c : c - half;
  const float arg = static_cast<float>(ps) * expf(static_cast<float>(fi) * neg_emb);
  return c < half ? sinf(arg) : cosf(arg);
}

// out = fp16(x + alpha * table[pos]) (tts_modules.py:228-229)
__global__ void k_pos_add(const float* x, const int* pos, const float* alpha, int total_rows, int n, float neg_emb,
                          __half* out) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<size_t>(total_rows) * n) return;
  const int c = static_cast<int>(i % n);
  out[i] = __float2half_rn(x[i] + alpha[0] * pos_table(pos[i / n], c, n, neg_emb));
}

}  // namespace
}  // namespace dsx
