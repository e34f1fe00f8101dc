// Entry and exit kernels of the FFT denoiser (usr/diff/candidate_decoder.py:50-100), shared by the sampler's evaluation
// (dsx_fftdiff.cu) and the training step (dsx_ffttrain.cu): the hi+lo fp16 split of an operand and of a weight block, the
// fold of input_projection into get_decode_inp, the step part of get_decode_inp, the entry GEMM with its pad flags and
// get_mel_out.  See dsx_fftdiff.cu for the arithmetic.
#pragma once
#include "dsx_conv.cuh"
#include "dsx_internal.h"
#include "dsx_ptx.cuh"

namespace dsx {
namespace {   // every translation unit has its own copies, like dsx_conv.cuh

constexpr int kSplit = 3;      // planes of a hi+lo operand along K
constexpr int kOutNT = 128;    // get_mel_out: M = 80 columns in one tile

// x logically [B][C][T] fp32 (strides xs) -> fp16 [B][T][3C] = (hi, lo, hi) of every value
__global__ void k_fft_split(const float* __restrict__ x, dsx_strides xs, int T, int C, __half* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const bool c_fast = xs.c == 1 && xs.t != 1;   // read along the unit-stride axis
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = c_fast ? t0 + i : t0 + threadIdx.x, c = c_fast ? c0 + threadIdx.x : c0 + i;
    const float v = (t < T && c < C) ? x[b * xs.b + c * xs.c + t * xs.t] : 0.f;
    if (c_fast) tile[threadIdx.x][i] = v; else tile[i][threadIdx.x] = v;   // tile[c][t]
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < C) {
      const float v = tile[threadIdx.x][i];
      const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
      __half* o = out + (static_cast<size_t>(b) * T + t) * kSplit * C + c;
      o[0] = hi;
      o[C] = lo;
      o[2 * C] = hi;
    }
  }
}

// w[n][col0 + k] (row stride ldw) -> out [N][3K] = (hi, hi, lo): fp32 values that fp16 holds exactly
__global__ void k_fft_split_w(const float* __restrict__ w, int ldw, int col0, int K, int N, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * K) return;
  const int n = i / K, k = i - n * K;
  const float v = w[static_cast<size_t>(n) * ldw + col0 + k];
  const float hi = __half2float(__float2half_rn(v)), lo = __half2float(__float2half_rn(v - hi));
  float* o = out + static_cast<size_t>(n) * kSplit * K + k;
  o[0] = hi;
  o[K] = hi;
  o[2 * K] = lo;
}

// W' [H][M] = Wd[:, 0:dim] . W_in and b' = Wd[:, 0:dim] . b_in + b_d, summed in double (block h, thread m; m == M: b')
__global__ void k_fft_fold(const float* __restrict__ wd, int ldw, const float* __restrict__ win,
                           const float* __restrict__ bin, const float* __restrict__ bd, int dim, int M,
                           float* __restrict__ wf, float* __restrict__ bf) {
  const int h = blockIdx.x, m = threadIdx.x;
  if (m > M) return;
  double acc = m == M ? static_cast<double>(bd[h]) : 0.0;
  for (int c = 0; c < dim; ++c) {
    const double a = wd[static_cast<size_t>(h) * ldw + c];
    acc += a * (m == M ? bin[c] : win[static_cast<size_t>(c) * M + m]);
  }
  if (m == M) bf[h] = static_cast<float>(acc);
  else wf[static_cast<size_t>(h) * M + m] = static_cast<float>(acc);
}

// TTAB[row][h] = Wd[h][col0:col0 + dim] . EMB[row] in fp32, one warp per (row, h)
__global__ void k_fft_tproj(const float* __restrict__ emb, const float* __restrict__ wd, int ldw, int col0, int dim,
                            int H, int rows, float* __restrict__ ttab) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows * H) return;
  const int row = warp / H, h = warp - row * H;
  const float* w = wd + static_cast<size_t>(h) * ldw + col0;
  const float* v = emb + static_cast<size_t>(row) * dim;
  float acc = 0.f;
  for (int k = lane; k < dim; k += 32) acc = fmaf(w[k], v[k], acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) ttab[warp] = acc;
}

struct FftInArgs {
  ConvGemm g;
  const __half* a;             // [B][T][g.cin] split operand
  int T;
  float* out;                  // [B][T][n] fp32
  const float* cp;             // non-null (entry): CONDPART [B][T][n]; null: out = the product alone (the cond part)
  const float* ttab;           // [rows][n]
  int row0, row_per_b;
  uint8_t* pad;                // [B][T]
};

// One 64-row tile of utterance blockIdx.y; one column tile holds all n <= 256 columns, so the pad flag of a row is
// decided here.
template <int NT>
__global__ void __launch_bounds__(128 * (NT > 128 ? 2 : 1)) k_fft_in(const FftInArgs p) {
  constexpr int WG = NT > 128 ? 2 : 1, NH = NT / WG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ int nonzero[kConvRows];
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, b = blockIdx.y, m0 = blockIdx.x * kConvRows;
  if (tid < kConvRows) nonzero[tid] = 0;   // published by the K loop's barriers
  float acc[NH / 2];
  conv_k_loop<NT, WG>(p.g, p.a, p.T, p.T, b, m0, 0, smem, acc);

  const int n = p.g.n, c0 = wg * NH, r0 = acc_row(wtid, 0);
  const size_t rbase = static_cast<size_t>(b) * p.T;
  const float* tt = p.cp ? p.ttab + static_cast<size_t>(p.row0 + b * p.row_per_b) * n : nullptr;
  bool any[2] = {false, false};
#pragma unroll
  for (int e = 0; e < NH / 2; e += 2) {
    const int col = c0 + acc_col(wtid, e), r = (e >> 1) & 1, m = m0 + r0 + 8 * r;
    if (col >= n || m >= p.T) continue;
    const size_t idx = (rbase + m) * n + col;
    float v0 = acc[e], v1 = acc[e + 1];
    if (p.cp) {
      const float2 c = *reinterpret_cast<const float2*>(p.cp + idx);
      v0 = ((v0 + __ldg(p.g.b + col)) + c.x) + __ldg(tt + col);
      v1 = ((v1 + __ldg(p.g.b + col + 1)) + c.y) + __ldg(tt + col + 1);
      any[r] = any[r] || v0 != 0.f || v1 != 0.f;
    }
    *reinterpret_cast<float2*>(p.out + idx) = make_float2(v0, v1);
  }
  if (!p.cp) return;
  if (any[0]) nonzero[r0] = 1;
  if (any[1]) nonzero[r0 + 8] = 1;
  __syncthreads();
  if (tid < kConvRows && m0 + tid < p.T) p.pad[rbase + m0 + tid] = nonzero[tid] ? 0 : 1;
}

// eps[b][0][col][m] = A[b][m] . mel_out_w[col] + bias[col], contiguous [B][1][n][T]
__global__ void __launch_bounds__(128) k_fft_out(const ConvGemm g, const __half* __restrict__ a, int T,
                                                 float* __restrict__ eps) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, b = blockIdx.y, m0 = blockIdx.x * kConvRows;
  float acc[kOutNT / 2];
  conv_k_loop<kOutNT, 1>(g, a, T, T, b, m0, 0, smem, acc);
  const int n = g.n, r0 = acc_row(tid, 0);
#pragma unroll
  for (int e = 0; e < kOutNT / 2; e += 2) {
    const int col = acc_col(tid, e), m = m0 + r0 + 8 * ((e >> 1) & 1);
    if (col >= n || m >= T) continue;
    float* o = eps + (static_cast<size_t>(b) * n + col) * T + m;
    o[0] = acc[e] + __ldg(g.b + col);
    o[T] = acc[e + 1] + __ldg(g.b + col + 1);
  }
}

int fft_in_run(const FftInArgs& p, int B, cudaStream_t s) {
  const dim3 grid((p.T + kConvRows - 1) / kConvRows, B, 1);
  return conv_dispatch<256>(p.g.nt, [&](auto c) {
    constexpr int NT = decltype(c)::value;
    k_fft_in<NT><<<grid, 128 * (NT > 128 ? 2 : 1), conv_smem<NT>(), s>>>(p);
    return launch_check("k_fft_in");
  });
}

}  // namespace
}  // namespace dsx
