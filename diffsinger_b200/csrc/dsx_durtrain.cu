// Duration predictor training step on sm_90a: DurationPredictor._forward in training mode (modules/fastspeech/
// tts_modules.py:106-120, dur_loss 'mse') with what the backward needs saved to a caller-owned tape, and the exact backward
// to every parameter and to the input xs.  P = chans, F = B T tokens, layer i: conv_i (k taps from tap0), ReLU, LayerNorm
// (eps 1e-12), dropout site i, * !mask; then the head Linear(P, 1), * !mask.
//
// Forward (1 + 1 + 2 L launches and 2 copies): k_dpt_hdr copies the mask and writes the header, durpred_train_pack refills
// a dsx_durpred handle's fp16 packs (one k_pack_conv per layer), and durpred_train_run runs the eval kernel k_pe_conv in
// its training form (dsx_pe.cu): each layer's fp16 input operand, its LayerNorm input (fp32) and the head's input (fp32)
// go to the tape.  Masks come from Philox keyed by (seed, site, frame, channel) (dsx_rng.cuh) and are drawn again in the
// backward, not stored.
//
// Backward, with GU the fp16 gradient at conv_i's output (before the ReLU), scaled by S:
//   k_dpt_amax, k_scale    S from amax |d_xs * !mask| (S amax in [2^5, 2^6)), NaN when the tape is of another (B, T)
//   k_pack_conv x L        conv_i^T (taps reversed), the data-gradient packs of this backward's weights
//   k_dpt_head             per token: the head's backward (d linear partials), then layer L - 1's dropout, LayerNorm and
//                          ReLU backward -> GU
//   per layer i = L - 1 .. 0:
//     k_wgrad + k_wgrad_sum     d conv_i (taps as shifted B tiles, four per launch) and its bias (the A column sums)
//     k_dpt_dgrad               conv_i's stride-1 transposed conv of GU on conv_k_loop (a whole row of chans <= 256
//                               columns in one CTA), with layer i - 1's * !mask, dropout, LayerNorm and ReLU backward in
//                               the epilogue -> the next GU; at layer 0, d_x = the transposed conv / S
//   k_dpt_lnreduce         LayerNorm affine and head gradients: the per-CTA partials of k_dpt_head and k_dpt_dgrad (fixed
//                          grids) summed in order, / S
// 4 + 4 L launches for k <= 4.  No atomics touch a result, so two backwards of one tape are bitwise equal; every gradient
// written is a fixed-order fp32 sum times 1 / S, so 2^k d_xs gives exactly 2^k times every gradient.
//
// The backward (dpt_backward) also serves the pitch predictor's step (dsx_pitchtrain.cu): there the mask is NULL and
// the head has od <= 16 outputs, d_out [F][od] instead of d_xs.
#include <math.h>

#include <algorithm>
#include <vector>

#include "dsx_conv.cuh"
#include "dsx_internal.h"
#include "dsx_ptx.cuh"
#include "dsx_wgrad.cuh"

namespace dsx {
namespace {

constexpr int kDpMaxLayers = 16;
constexpr int kHeadBlocks = 256;    // CTAs of k_dpt_head: fixed, so its partial sums have a fixed order
constexpr float kLnEps = 1e-12f;    // LayerNorm of tts_modules.py (not the 1e-5 of the FFT blocks)

using TapeHdr = Fs2TapeHdr;

// a scaled gradient operand as fp16: a value beyond fp16's range saturates at +-65504 instead of becoming inf (NaN stays
// NaN).  S keeps d_xs's largest value 2^10 below that (oracle/precision_study_durtrain.py measures 2^10 to 2^12 of
// headroom at every layer), but a row whose ReLU output is nearly constant has a LayerNorm rstd up to 1e6 (eps 1e-12).
__device__ __forceinline__ __half sat_half(float v) {
  return __float2half_rn(fabsf(v) > 65504.f ? copysignf(65504.f, v) : v);
}

// the tape's header (block 0) and its copy of the mask
__global__ void k_dpt_hdr(TapeHdr* h, uint64_t seed, float p, int B, int T, const uint8_t* mask, uint8_t* pad) {
  const size_t F = static_cast<size_t>(B) * T;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < F;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    pad[i] = mask[i];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    h->seed = seed;
    h->p = p;
    h->B = B;
    h->T = T;
  }
}

// amax |d_out| over the od columns of the non-padding tokens (pad NULL: every token), one CTA (F is a few thousand
// tokens, tens of thousands of frames for the pitch predictor)
__global__ void __launch_bounds__(1024) k_dpt_amax(const float* g, const uint8_t* pad, size_t F, int od,
                                                   unsigned* amax_bits) {
  __shared__ float red[32];
  float m = 0.f;
  for (size_t i = threadIdx.x; i < F * od; i += blockDim.x) m = fmaxf(m, pad && pad[i / od] ? 0.f : fabsf(g[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < static_cast<int>(blockDim.x >> 5); ++w) m = fmaxf(m, red[w]);
    *amax_bits = __float_as_uint(m);
  }
}

// ---- the head and layer L - 1: one warp per token ---------------------------------------------------------------------
struct DpHeadArgs {
  const float* dxs;            // [F][od] d_out, unscaled
  const uint8_t* pad;          // [F] or NULL (no mask)
  const float* hin;            // the head's input [F][P] (tape)
  const float* r;              // layer L - 1's LayerNorm input [F][P] (tape)
  const float* wl;             // linear.weight [od][P]
  const float* gamma;          // layer L - 1's LayerNorm weight [P]
  const TapeHdr* hdr;
  int site;                    // L - 1
  const float* scal;
  __half* gu;                  // [F][P]
  float* part;                 // [kHeadBlocks][head_part_floats]: d gamma, d beta, d linear.weight, d linear.bias
  int F, P, od;
};

// floats of one CTA's k_dpt_head partials: d gamma [P], d beta [P], d linear.weight [od][P], d linear.bias [od]
__host__ __device__ inline int head_part_floats(int P, int od) { return (2 + od) * P + od; }

// OD >= od outputs of the head (the duration predictor's 1, the pitch predictor's up to 16); the warps' partials are
// added into the CTA's sums in warp order, so OD = 1 sums exactly as a per-warp table summed in order would
template <int OD>
__global__ void __launch_bounds__(256) k_dpt_head(const DpHeadArgs p) {
  __shared__ float tot[(2 + OD) * 256 + OD];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, P = p.P, od = p.od;
  const float S = p.scal[0], inv_p = 1.f / static_cast<float>(P);
  const Fs2Drop drop = hdr_drop(p.hdr, p.site);
  float dgam[8], dbet[8], dwl[OD][8], dbl[OD];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    dgam[i] = dbet[i] = 0.f;
#pragma unroll
    for (int o = 0; o < OD; ++o) dwl[o][i] = 0.f;
  }
#pragma unroll
  for (int o = 0; o < OD; ++o) dbl[o] = 0.f;
  for (int f = blockIdx.x * 8 + warp; f < p.F; f += gridDim.x * 8) {
    const size_t rb = static_cast<size_t>(f) * P;
    const bool padded = p.pad && p.pad[f];
    float gx[OD];
#pragma unroll
    for (int o = 0; o < OD; ++o) gx[o] = padded || o >= od ? 0.f : S * p.dxs[static_cast<size_t>(f) * od + o];
    if (lane == 0) {
#pragma unroll
      for (int o = 0; o < OD; ++o) dbl[o] += gx[o];
    }
    float rv[8], gy[8], sum = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = lane + 32 * i;
      rv[i] = gy[i] = 0.f;
      if (c >= P) continue;
      const float h = p.hin[rb + c];
      float g = gx[0] * p.wl[c];
#pragma unroll
      for (int o = 0; o < OD; ++o) {
        dwl[o][i] += gx[o] * h;
        if (o > 0 && o < od) g += gx[o] * p.wl[o * P + c];
      }
      gy[i] = g * dropout_scale(drop, f, c);
      rv[i] = p.r[rb + c];
      sum += rv[i];
    }
    const float mean = warp_sum(sum) * inv_p;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float d = rv[i] - mean;
      sq += lane + 32 * i < P ? d * d : 0.f;
    }
    const float rstd = 1.f / sqrtf(warp_sum(sq) * inv_p + kLnEps);
    float s1 = 0.f, s2 = 0.f, xh[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = lane + 32 * i;
      xh[i] = (rv[i] - mean) * rstd;
      if (c >= P) continue;
      dgam[i] += gy[i] * xh[i];
      dbet[i] += gy[i];
      const float gg = gy[i] * p.gamma[c];
      gy[i] = gg;
      s1 += gg;
      s2 += gg * xh[i];
    }
    const float m1 = warp_sum(s1) * inv_p, m2 = warp_sum(s2) * inv_p;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = lane + 32 * i;
      if (c >= P) continue;
      const float v = rv[i] > 0.f ? rstd * (gy[i] - m1 - xh[i] * m2) : 0.f;
      p.gu[rb + c] = sat_half(v);
    }
  }
  const int W = head_part_floats(P, od);
  for (int t = threadIdx.x; t < W; t += blockDim.x) tot[t] = 0.f;
  for (int w = 0; w < 8; ++w) {
    __syncthreads();
    if (warp != w) continue;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int c = lane + 32 * i;
      if (c >= P) continue;
      tot[c] += dgam[i];
      tot[P + c] += dbet[i];
#pragma unroll
      for (int o = 0; o < OD; ++o)
        if (o < od) tot[(2 + o) * P + c] += dwl[o][i];
    }
    if (lane == 0) {
#pragma unroll
      for (int o = 0; o < OD; ++o)
        if (o < od) tot[(2 + od) * P + o] += dbl[o];
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < W; t += blockDim.x) p.part[static_cast<size_t>(blockIdx.x) * W + t] = tot[t];
}

// ---- data gradient of conv i, with layer i - 1's backward in the epilogue ---------------------------------------------
struct DgradArgs {
  ConvGemm g;                  // conv_i^T: g.cin = P (GU's channels), g.n = conv_i's input channels
  const __half* x;             // GU of layer i [F][P]
  int T;
  float* dx;                   // layer 0: d_x [F][g.n] = the transposed conv / S
  const float* r;              // else layer i - 1's LayerNorm input [F][g.n] (tape)
  const float* gamma;          // layer i - 1's LayerNorm weight
  const uint8_t* pad;          // [F] or NULL (no mask)
  const TapeHdr* hdr;
  int site;                    // i - 1
  __half* gu;                  // GU of layer i - 1 [F][g.n]
  float* part;                 // [B * mtiles][2 g.n]: d gamma, d beta of this CTA's 64 rows
  const float* scal;
};

template <int NT>
struct DgShape {
  static constexpr int WG = NT > 128 ? 2 : 1;      // warpgroups per CTA, each with NT / WG columns of the same 64 rows
};

template <int NT>
__global__ void __launch_bounds__(128 * DgShape<NT>::WG) k_dpt_dgrad(const DgradArgs p) {
  constexpr int WG = DgShape<NT>::WG, NH = NT / WG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ float xrow[WG][kConvRows];
  __shared__ float colsum[2][4 * WG][NH];
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, warp = wtid >> 5, lane = tid & 31;
  const int b = blockIdx.y, m0 = blockIdx.x * kConvRows, T = p.T;
  float acc[NH / 2];
  conv_k_loop<NT, WG>(p.g, p.x, T, T, b, m0, 0, smem, acc);

  const int n = p.g.n, c0 = wg * NH, r0 = acc_row(wtid, 0);
  const size_t rbase = static_cast<size_t>(b) * T;
  const int mrow[2] = {m0 + r0, m0 + r0 + 8};
  if (p.dx) {
    const float is = p.scal[1];
#pragma unroll
    for (int e = 0; e < NH / 2; e += 2) {
      const int col = c0 + acc_col(wtid, e), m = mrow[(e >> 1) & 1];
      if (col < n && m < T)
        *reinterpret_cast<float2*>(p.dx + (rbase + m) * n + col) = make_float2(acc[e] * is, acc[e + 1] * is);
    }
    return;
  }
  auto row_sum = [&](float& s0, float& s1) {
    s0 = quad_sum(s0);
    s1 = quad_sum(s1);
    if (WG > 1) {
      if ((wtid & 3) == 0) {
        xrow[wg][r0] = s0;
        xrow[wg][r0 + 8] = s1;
      }
      __syncthreads();
      s0 = xrow[0][r0] + xrow[1][r0];
      s1 = xrow[0][r0 + 8] + xrow[1][r0 + 8];
      __syncthreads();
    }
  };
  const Fs2Drop drop = hdr_drop(p.hdr, p.site);
  bool keep[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) keep[r] = mrow[r] < T && !(p.pad && p.pad[rbase + mrow[r]]);
  // g = the gradient at layer i - 1's LayerNorm output (in acc); its input r, then xhat, in the spent operand stages
  // (thread-private slots: NT / 2 floats per thread fit in conv_smem<NT>())
  float* rv = reinterpret_cast<float*>(smem) + tid;
  constexpr int kStride = 128 * WG;
  float s[2] = {0.f, 0.f};
#pragma unroll
  for (int e = 0; e < NH / 2; e += 2) {
    const int col = c0 + acc_col(wtid, e), r = (e >> 1) & 1, m = mrow[r];
    float2 x = make_float2(0.f, 0.f);
    if (col < n && m < T) x = *reinterpret_cast<const float2*>(p.r + (rbase + m) * n + col);
    rv[e * kStride] = x.x;
    rv[(e + 1) * kStride] = x.y;
    s[r] += x.x + x.y;
    const float2 ds = keep[r] && col < n ? dropout_scale2(drop, rbase + m, col) : make_float2(0.f, 0.f);
    acc[e] *= ds.x;
    acc[e + 1] *= ds.y;
  }
  const float inv_n = 1.f / static_cast<float>(n);
  row_sum(s[0], s[1]);
  const float mean[2] = {s[0] * inv_n, s[1] * inv_n};
  float q[2] = {0.f, 0.f};
#pragma unroll
  for (int e = 0; e < NH / 2; ++e) {
    const int col = c0 + acc_col(wtid, e), r = (e >> 1) & 1;
    const float d = rv[e * kStride] - mean[r];
    q[r] += col < n ? d * d : 0.f;
  }
  row_sum(q[0], q[1]);
  const float rstd[2] = {1.f / sqrtf(q[0] * inv_n + kLnEps), 1.f / sqrtf(q[1] * inv_n + kLnEps)};
  // column partials of d gamma = g xhat and d beta = g over this CTA's rows, and the row sums of the LayerNorm backward
  float t1[2] = {0.f, 0.f}, t2[2] = {0.f, 0.f};
  uint64_t pos = 0;   // bit e: r > 0 (the ReLU's gradient)
#pragma unroll
  for (int e = 0; e < NH / 2; ++e) {
    const int col = c0 + acc_col(wtid, e), r = (e >> 1) & 1;
    const float x = rv[e * kStride];
    if (x > 0.f) pos |= 1ull << e;
    const float xh = col < n ? (x - mean[r]) * rstd[r] : 0.f;
    rv[e * kStride] = xh;
    const float gg = col < n ? acc[e] * __ldg(p.gamma + col) : 0.f;
    t1[r] += gg;
    t2[r] += gg * xh;
  }
#pragma unroll
  for (int e = 0; e < NH / 2; ++e) {   // rows r0 and r0 + 8 of a column, then the warp's 16 rows, in a fixed order
    if (e & 2) continue;
    float cg = acc[e] * rv[e * kStride] + acc[e + 2] * rv[(e + 2) * kStride], cb = acc[e] + acc[e + 2];
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) {
      cg += __shfl_xor_sync(0xffffffffu, cg, o);
      cb += __shfl_xor_sync(0xffffffffu, cb, o);
    }
    if (lane < 4) {
      const int lc = acc_col(wtid, e);
      colsum[0][wg * 4 + warp][lc] = cg;
      colsum[1][wg * 4 + warp][lc] = cb;
    }
  }
  row_sum(t1[0], t1[1]);
  row_sum(t2[0], t2[1]);
#pragma unroll
  for (int e = 0; e < NH / 2; e += 2) {
    const int col = c0 + acc_col(wtid, e), r = (e >> 1) & 1, m = mrow[r];
    if (col >= n || m >= T) continue;
    float v[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float gg = acc[e + i] * __ldg(p.gamma + col + i);
      v[i] = ((pos >> (e + i)) & 1) ? rstd[r] * (gg - t1[r] * inv_n - rv[(e + i) * kStride] * t2[r] * inv_n) : 0.f;
    }
    *reinterpret_cast<__half2*>(p.gu + (rbase + m) * n + col) = __halves2half2(sat_half(v[0]), sat_half(v[1]));
  }
  __syncthreads();
  float* part = p.part + (static_cast<size_t>(b) * gridDim.x + blockIdx.x) * 2 * n;
  for (int t = tid; t < 2 * n; t += 128 * WG) {
    const int which = t >= n, col = t - which * n, w = col / NH, lc = col - w * NH;
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < 4; ++k) v += colsum[which][w * 4 + k][lc];
    part[t] = v;
  }
}

// ---- reductions ---------------------------------------------------------------------------------------------------------
// every LayerNorm affine gradient and the head's: layer l's partials part[l] (blocks[l] rows of stride[l] floats, d gamma
// then d beta), the head's (d linear.weight [od][P], then d linear.bias [od]) from column 2 P of the last layer's rows,
// summed in row order, / S
struct LnRedArgs {
  const float* part[kDpMaxLayers];
  int blocks[kDpMaxLayers], stride[kDpMaxLayers];
  float* dgamma[kDpMaxLayers];
  float* dbeta[kDpMaxLayers];
  float* dwl;
  float* dbl;
  int L, P, od;
  const float* scal;
};

__global__ void k_dpt_lnreduce(const LnRedArgs p) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, P = p.P;
  if (t >= 2 * p.L * P + p.od * (P + 1)) return;
  const int l = t < 2 * p.L * P ? t / (2 * P) : p.L - 1, c = t < 2 * p.L * P ? t % (2 * P) : t - 2 * p.L * P + 2 * P;
  float s = 0.f;
  for (int k = 0; k < p.blocks[l]; ++k) s += p.part[l][static_cast<size_t>(k) * p.stride[l] + c];
  s *= p.scal[1];
  if (t >= 2 * p.L * P) {
    if (c < (2 + p.od) * P) p.dwl[c - 2 * P] = s;
    else p.dbl[c - (2 + p.od) * P] = s;
  } else if (c < P) {
    p.dgamma[l][c] = s;
  } else {
    p.dbeta[l][c - P] = s;
  }
}

// ---- tape and workspace -------------------------------------------------------------------------------------------------
using Tape = DurTape;

// every region of the tape for (config, B, T), in order; bytes of the whole tape
size_t tape_carve(const dsx_durpred_config& c, int B, int T, uint8_t* base, Tape* t) {
  const size_t F = static_cast<size_t>(B) * T, P = c.chans;
  const int L = c.layers;
  size_t n = 0;
  auto take = [&](size_t bytes) {
    uint8_t* q = base ? base + n : nullptr;
    n += align256(bytes);
    return q;
  };
  Tape dummy;
  Tape& tp = t ? *t : dummy;
  tp.hdr = reinterpret_cast<TapeHdr*>(take(sizeof(TapeHdr)));
  tp.pad = take(F);
  tp.tr.a.resize(L);
  tp.tr.r.resize(L);
  tp.tr.a[0] = reinterpret_cast<__half*>(take(2 * F * c.idim));
  for (int l = 0; l < L; ++l) tp.tr.r[l] = reinterpret_cast<float*>(take(4 * F * P));
  for (int l = 1; l < L; ++l) tp.tr.a[l] = reinterpret_cast<__half*>(take(2 * F * P));
  tp.tr.hin = reinterpret_cast<float*>(take(4 * F * P));
  return n;
}

}  // namespace
}  // namespace dsx

struct dsx_durpred_train {
  int device = 0;
  dsx_durpred_config cfg{};
  dsx_durpred* fwd = nullptr;                  // the forward's packs (refilled by every forward) and kernels
  dsx::ConvGemm dgrad[dsx::kDpMaxLayers];      // conv_i^T, refilled by every backward
  dsx::DevAllocs mem;
};

namespace dsx {
namespace {

int tap0_of(const dsx_durpred_config& c) { return c.padding ? -(c.kernel - 1) : -(c.kernel - 1) / 2; }

struct Ws {
  unsigned* amax;   // the scale's words, then the gradient operands and partial sums of dpt_backward
  float* scal;
  __half* gu[2];
  float* hpart;
  float* lnp;                  // (L - 1) regions of [B * mtiles][2 P]
  size_t lnp_stride;           // floats between them
  float* wpart;
};

// the backward's workspace (the forward uses none) for a head of od outputs; bytes of it
size_t ws_carve(const dsx_durpred_train* h, int B, int T, int od, uint8_t* base, Ws* w) {
  const dsx_durpred_config& c = h->cfg;
  const size_t F = static_cast<size_t>(B) * T, P = c.chans, mt = (T + kConvRows - 1) / kConvRows;
  size_t n = 0;
  auto take = [&](size_t bytes) {
    uint8_t* q = base ? base + n : nullptr;
    n += align256(bytes);
    return q;
  };
  Ws dummy;
  Ws& ws = w ? *w : dummy;
  ws.amax = reinterpret_cast<unsigned*>(take(256));
  ws.scal = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(ws.amax) + 16);
  ws.gu[0] = reinterpret_cast<__half*>(take(2 * F * P));
  ws.gu[1] = reinterpret_cast<__half*>(take(2 * F * P));
  ws.hpart = reinterpret_cast<float*>(take(4 * static_cast<size_t>(kHeadBlocks) * head_part_floats(c.chans, od)));
  ws.lnp_stride = align256(4 * B * mt * 2 * P) / 4;
  ws.lnp = reinterpret_cast<float*>(take(4 * ws.lnp_stride * (c.layers - 1)));
  std::vector<std::pair<int, int>> shapes;   // (m tiles, n tiles) of the weight gradients: ntl <= 4 taps a launch
  for (int ntl = 1; ntl <= std::min(c.kernel, 4); ++ntl) shapes.push_back({(c.chans + 63) / 64, ntl});
  ws.wpart = reinterpret_cast<float*>(take(4 * wgrad_part_floats(static_cast<int>(F), shapes, h->device)));
  return n;
}

int check_geom(const dsx_durpred_train* h, int B, int T) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(B <= 65535, DSX_E_INVALID, "B = %d utterances per call is above the 65535 the launch grid holds", B);
  const long long Tp = (T + kConvRows - 1) / kConvRows * kConvRows;
  DSX_CHECK(static_cast<long long>(B) * Tp * std::max(h->cfg.idim, h->cfg.chans) < (1ll << 31), DSX_E_INVALID,
            "B * T = %lld tokens is too large", static_cast<long long>(B) * T);
  return DSX_OK;
}

int check_params(const dsx_durpred_train* h, const dsx_durpred_params* p, const char* what) {
  DSX_CHECK(p, DSX_E_INVALID, "%s is NULL", what);
  DSX_CHECK(p->conv_w && p->conv_b && p->ln_w && p->ln_b && p->linear_w && p->linear_b, DSX_E_INVALID,
            "a pointer of %s is NULL", what);
  for (int l = 0; l < h->cfg.layers; ++l)
    DSX_CHECK(p->conv_w[l] && p->conv_b[l] && p->ln_w[l] && p->ln_b[l], DSX_E_INVALID,
              "a pointer of layer %d of %s is NULL", l, what);
  return DSX_OK;
}

template <int NT>
int run_dgrad(DgradArgs a, const ConvGemm& g, int B, int T, cudaStream_t s) {
  a.g = g;
  a.T = T;
  k_dpt_dgrad<NT><<<dim3((T + kConvRows - 1) / kConvRows, B), 128 * DgShape<NT>::WG, conv_smem<NT>(), s>>>(a);
  return launch_check("k_dpt_dgrad");
}

}  // namespace
}  // namespace dsx

namespace dsx {

dsx_durpred* dpt_forward_handle(dsx_durpred_train* h) { return h->fwd; }

size_t dpt_workspace_bytes(const dsx_durpred_train* h, int B, int T, int od) {
  return ws_carve(h, B, T, od, nullptr, nullptr);
}

int dpt_backward(dsx_durpred_train* h, const dsx_durpred_params* w, const DurTape& tp, const float* d_out, int od,
                 const dsx_durpred_params* grads, float* d_x, int B, int T, void* workspace, cudaStream_t s) {
  const dsx_durpred_config& c = h->cfg;
  const int P = c.chans, L = c.layers, k = c.kernel, F = B * T, mtiles = (T + kConvRows - 1) / kConvRows;
  Ws ws;
  ws_carve(h, B, T, od, static_cast<uint8_t*>(workspace), &ws);
  auto gp = [](const float* q) { return const_cast<float*>(q); };

  k_dpt_amax<<<1, 1024, 0, s>>>(d_out, tp.pad, static_cast<size_t>(F), od, ws.amax);
  DSX_TRY(launch_check("k_dpt_amax"));
  k_scale<<<1, 1, 0, s>>>(ws.amax, ws.scal, tp.hdr, B, T);
  DSX_TRY(launch_check("k_scale"));
  for (int i = (d_x ? 0 : 1); i < L; ++i) {
    const ConvGemm& g = h->dgrad[i];
    DSX_TRY(conv_repack(g, PackArgs{w->conv_w[i], nullptr, nullptr, g.cin, g.n, g.n, k, 1, 1}, s));
  }

  DpHeadArgs ha{};
  ha.dxs = d_out;
  ha.pad = tp.pad;
  ha.hin = tp.tr.hin;
  ha.r = tp.tr.r[L - 1];
  ha.wl = w->linear_w;
  ha.gamma = w->ln_w[L - 1];
  ha.hdr = tp.hdr;
  ha.site = L - 1;
  ha.scal = ws.scal;
  ha.gu = ws.gu[0];
  ha.part = ws.hpart;
  ha.F = F;
  ha.P = P;
  ha.od = od;
  if (od == 1) k_dpt_head<1><<<kHeadBlocks, 256, 0, s>>>(ha);
  else if (od == 2) k_dpt_head<2><<<kHeadBlocks, 256, 0, s>>>(ha);
  else if (od <= 4) k_dpt_head<4><<<kHeadBlocks, 256, 0, s>>>(ha);
  else if (od <= 8) k_dpt_head<8><<<kHeadBlocks, 256, 0, s>>>(ha);
  else k_dpt_head<16><<<kHeadBlocks, 256, 0, s>>>(ha);
  DSX_TRY(launch_check("k_dpt_head"));

  int cur = 0;
  for (int i = L - 1; i >= 0; --i) {
    const int cin = i ? P : c.idim;
    // d conv_i [P][cin][k]: tap j is sum_f GU[f] (x) a_i[f + tap0 + j], four taps a launch
    for (int j0 = 0; j0 < k; j0 += 4) {
      WgradArgs t{};
      const int ntl = std::min(4, k - j0);
      WgradDst o{};
      for (int jj = 0; jj < ntl; ++jj) {
        t.b[jj] = tp.tr.a[i];
        t.ldb[jj] = cin;
        t.bn[jj] = cin;
        t.shift[jj] = tap0_of(c) + j0 + jj;
        o.dst[jj] = gp(grads->conv_w[i]) + j0 + jj;
        o.ms[jj] = cin * k;
        o.cs[jj] = k;
      }
      o.db = j0 == 0 ? gp(grads->conv_b[i]) : nullptr;
      t.a = ws.gu[cur];
      t.lda = P;
      t.am = P;
      t.F = F;
      t.T = T;
      DSX_TRY(run_wgrad(t, ntl, o, ws.wpart, ws.scal, h->device, s));
    }
    if (i == 0 && !d_x) break;
    DgradArgs a{};
    a.x = ws.gu[cur];
    a.pad = tp.pad;
    a.hdr = tp.hdr;
    a.scal = ws.scal;
    if (i == 0) {
      a.dx = d_x;
    } else {
      a.r = tp.tr.r[i - 1];
      a.gamma = w->ln_w[i - 1];
      a.site = i - 1;
      a.gu = ws.gu[cur ^ 1];
      a.part = ws.lnp + static_cast<size_t>(i - 1) * ws.lnp_stride;
    }
    const ConvGemm& g = h->dgrad[i];
    DSX_TRY(conv_dispatch<256>(g.nt, [&](auto kk) { return run_dgrad<decltype(kk)::value>(a, g, B, T, s); }));
    cur ^= 1;
  }

  LnRedArgs lr{};
  for (int l = 0; l < L; ++l) {
    const bool last = l == L - 1;
    lr.part[l] = last ? ws.hpart : ws.lnp + static_cast<size_t>(l) * ws.lnp_stride;
    lr.blocks[l] = last ? kHeadBlocks : B * mtiles;
    lr.stride[l] = last ? head_part_floats(P, od) : 2 * P;
    lr.dgamma[l] = gp(grads->ln_w[l]);
    lr.dbeta[l] = gp(grads->ln_b[l]);
  }
  lr.dwl = gp(grads->linear_w);
  lr.dbl = gp(grads->linear_b);
  lr.L = L;
  lr.P = P;
  lr.od = od;
  lr.scal = ws.scal;
  const int nout = 2 * L * P + od * (P + 1);
  k_dpt_lnreduce<<<(nout + 255) / 256, 256, 0, s>>>(lr);
  return launch_check("k_dpt_lnreduce");
}

}  // namespace dsx

using namespace dsx;

extern "C" {

int dsx_durpred_train_create(int device, const dsx_durpred_config* cfg, dsx_durpred_train** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  dsx_durpred* fwd = nullptr;
  DSX_TRY(dsx_durpred_create(device, cfg, &fwd));   // validates the configuration and selects the device
  dsx_durpred_train* h = new dsx_durpred_train();
  h->device = device;
  h->cfg = *cfg;
  h->fwd = fwd;
  int rc = [&]() -> int {
    DSX_TRY(durpred_train_alloc(fwd));
    DSX_TRY(conv_opt_in<256>([](auto k) { return k_dpt_dgrad<decltype(k)::value>; }));
    DSX_CUDA(cudaFuncSetAttribute(k_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmem));
    const int P = cfg->chans;
    for (int i = 0; i < cfg->layers; ++i) {   // gx[t] = sum_j W_j^T GU[t - tap0 - j]
      ConvGemm& g = h->dgrad[i];
      g.cin = P;
      g.n = i ? P : cfg->idim;
      g.taps = cfg->kernel;
      g.tap0 = -tap0_of(*cfg);
      g.tstep = -1;
      DSX_TRY(conv_alloc(h->mem, g, 256));
    }
    return DSX_OK;
  }();
  if (rc != DSX_OK) {
    dsx_durpred_train_destroy(h);
    return rc;
  }
  *out = h;
  return DSX_OK;
}

void dsx_durpred_train_destroy(dsx_durpred_train* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  h->mem.free_all();
  dsx_durpred_destroy(h->fwd);
  delete h;
}

int dsx_durpred_train_tape_bytes(dsx_durpred_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  DSX_TRY(check_geom(h, B, T));
  *out = tape_carve(h->cfg, B, T, nullptr, nullptr);
  return DSX_OK;
}

int dsx_durpred_train_workspace_bytes(dsx_durpred_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  DSX_TRY(check_geom(h, B, T));
  *out = ws_carve(h, B, T, 1, nullptr, nullptr);
  return DSX_OK;
}

int dsx_durpred_train_forward(dsx_durpred_train* h, const dsx_durpred_params* w, const float* x, dsx_strides xs_,
                              const uint8_t* mask, int B, int T, float p_drop, uint64_t seed, void* tape,
                              size_t tape_bytes, void* workspace, size_t workspace_bytes, float* xs, void* stream) {
  (void)workspace;   // the forward writes only the tape and xs
  (void)workspace_bytes;
  DSX_TRY(check_geom(h, B, T));
  DSX_TRY(check_params(h, w, "the parameters"));
  DSX_CHECK(x && mask && tape && xs, DSX_E_INVALID, "x, mask, tape and xs must not be NULL");
  DSX_CHECK(p_drop >= 0.f && p_drop < 1.f, DSX_E_INVALID, "dropout p = %g is outside [0, 1)", static_cast<double>(p_drop));
  const size_t need = tape_carve(h->cfg, B, T, nullptr, nullptr);
  DSX_CHECK(tape_bytes >= need, DSX_E_INVALID, "tape of %zu bytes is below the %zu this (B, T) needs", tape_bytes, need);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Tape tp;
  tape_carve(h->cfg, B, T, static_cast<uint8_t*>(tape), &tp);
  tp.tr.seed = seed;
  tp.tr.p = p_drop;
  const size_t F = static_cast<size_t>(B) * T;
  k_dpt_hdr<<<static_cast<unsigned>(std::min<size_t>((F + 255) / 256, 1024)), 256, 0, s>>>(tp.hdr, seed, p_drop, B, T,
                                                                                          mask, tp.pad);
  DSX_TRY(launch_check("k_dpt_hdr"));
  DSX_TRY(durpred_train_pack(h->fwd, w, s));
  return durpred_train_run(h->fwd, x, xs_, tp.pad, B, T, tp.tr, xs, s);
}

int dsx_durpred_train_backward(dsx_durpred_train* h, const dsx_durpred_params* w, const void* tape, const float* d_xs,
                               const dsx_durpred_params* grads, float* d_x, int B, int T, void* workspace,
                               size_t workspace_bytes, void* stream) {
  DSX_TRY(check_geom(h, B, T));
  DSX_TRY(check_params(h, w, "the parameters"));
  DSX_TRY(check_params(h, grads, "the gradients"));
  DSX_CHECK(tape && d_xs && workspace, DSX_E_INVALID, "tape, d_xs and workspace must not be NULL");
  const size_t wneed = ws_carve(h, B, T, 1, nullptr, nullptr);
  DSX_CHECK(workspace_bytes >= wneed, DSX_E_INVALID, "workspace of %zu bytes is below the %zu this (B, T) needs",
            workspace_bytes, wneed);
  DSX_CUDA(cudaSetDevice(h->device));
  Tape tp;
  tape_carve(h->cfg, B, T, static_cast<uint8_t*>(const_cast<void*>(tape)), &tp);
  return dpt_backward(h, w, tp, d_xs, 1, grads, d_x, B, T, workspace, static_cast<cudaStream_t>(stream));
}

int dsx_durpred_train_masks(dsx_durpred_train* h, uint64_t seed, float p_drop, int B, int T, uint8_t* const* out,
                            void* stream) {
  DSX_TRY(check_geom(h, B, T));
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  DSX_CHECK(p_drop >= 0.f && p_drop < 1.f, DSX_E_INVALID, "dropout p = %g is outside [0, 1)", static_cast<double>(p_drop));
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t F = static_cast<size_t>(B) * T, n = h->cfg.chans;
  for (int site = 0; site < h->cfg.layers; ++site) {
    DSX_CHECK(out[site], DSX_E_INVALID, "mask %d is NULL", site);
    k_drop_masks<<<static_cast<unsigned>(std::min<size_t>((F * n + 255) / 256, 4096)), 256, 0, s>>>(
        make_drop(seed, p_drop, site), F, static_cast<int>(n), out[site]);
    DSX_TRY(launch_check("k_drop_masks"));
  }
  return DSX_OK;
}

}  // extern "C"
