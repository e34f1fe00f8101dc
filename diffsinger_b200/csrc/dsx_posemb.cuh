// Sinusoidal position embedding of the pitch extractor (dsx_pe.cu), the FastSpeech2 decoder (dsx_fs2dec.cu) and the
// sinusoidal FastSpeech2 encoder (dsx_fs2enc.cu): the positions are make_positions over channel 0 of the input, or over
// the token ids for the encoder (utils/__init__.py:145-157, padding_idx 0), the table is
// SinusoidalPositionalEmbedding.get_embedding (modules/commons/common_layers.py:106-122) evaluated in fp32 on the fly, so
// it has no size limit and the reference's regrowth past its initial size (:127-135) needs no counterpart.
#pragma once
#include <math.h>

#include "dsx_internal.h"

namespace dsx {
namespace {   // every translation unit has its own kernels

// Inclusive prefix sum over t < T of val(t) (type V) by one block of kScanThreads threads, kScanChunk items per thread
// per pass: calls out(t, sum of val(0..t), val(t)) for every t.  sh: kScanThreads V of shared memory.
constexpr int kScanThreads = 1024, kScanChunk = 8;
template <typename V, typename Val, typename Out>
__device__ __forceinline__ void block_scan(V* sh, int T, Val val, Out out) {
  const int tid = threadIdx.x;
  V carry = 0;
  for (int base = 0; base < T; base += kScanThreads * kScanChunk) {
    const int t0 = base + tid * kScanChunk, t1 = min(T, t0 + kScanChunk);
    V local = 0;
    for (int t = t0; t < t1; ++t) local += val(t);
    sh[tid] = local;
    __syncthreads();
    for (int off = 1; off < kScanThreads; off <<= 1) {
      const V v = tid >= off ? sh[tid - off] : V(0);
      __syncthreads();
      sh[tid] += v;
      __syncthreads();
    }
    V s = carry + sh[tid] - local;
    for (int t = t0; t < t1; ++t) {
      const V v = val(t);
      s += v;
      out(t, s, v);
    }
    carry += sh[kScanThreads - 1];
    __syncthreads();
  }
}

// pos[b][t] = cumsum(x[b, :, 0] != 0)[t] * (x[b, t, 0] != 0) over contiguous x [B][T][n].  One block per utterance.
__global__ void __launch_bounds__(kScanThreads) k_pos_scan(const float* x, int T, int n, int* pos) {
  __shared__ int sh[kScanThreads];
  const float* xb = x + static_cast<size_t>(blockIdx.x) * T * n;
  int* pb = pos + static_cast<size_t>(blockIdx.x) * T;
  block_scan<int>(sh, T, [&](int t) { return static_cast<int>(xb[static_cast<size_t>(t) * n] != 0.f); },
                  [&](int t, int s, int nz) { pb[t] = nz ? s : 0; });
}

// The same positions over token ids (make_positions(txt_tokens), padding_idx 0): tok [B][T] int64.
__global__ void __launch_bounds__(kScanThreads) k_pos_scan_tokens(const int64_t* tok, int T, int* pos) {
  __shared__ int sh[kScanThreads];
  const int64_t* tb = tok + static_cast<size_t>(blockIdx.x) * T;
  int* pb = pos + static_cast<size_t>(blockIdx.x) * T;
  block_scan<int>(sh, T, [&](int t) { return static_cast<int>(tb[t] != 0); },
                  [&](int t, int s, int nz) { pb[t] = nz ? s : 0; });
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

// LayerNorm of one row of H = 32 * per channels held by a warp (lane holds channels lane + 32 i, i < per <= 8) ->
// fp16 ar[H]: the first LayerNorm of an FFTBlocks stack, written by the entry kernels of the decoder and the encoder.
__device__ __forceinline__ void warp_row_ln16(const float (&v)[8], int per, int H, float eps, const float* ln_w,
                                              const float* ln_b, __half* ar) {
  const int lane = threadIdx.x & 31;
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (i >= per) break;
    sum += v[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / static_cast<float>(H);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (i >= per) break;
    const float d = v[i] - mean;
    sq += d * d;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
  const float rstd = 1.f / sqrtf(sq / static_cast<float>(H) + eps);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (i >= per) break;
    const int c = lane + 32 * i;
    ar[c] = __float2half_rn((v[i] - mean) * rstd * ln_w[c] + ln_b[c]);
  }
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
