// FastSpeech2 decoder on sm_90a: decoder_inp [B, T, H] -> [B, T, H] (modules/fastspeech/tts_modules.py:251-357,
// FFTBlocks with EncSALayer of modules/commons/common_layers.py:542-588), in eval mode.
//
// Per call, 3 + 5 L launches over frames-major buffers:
//   k_fs2_pack    x (any strides) -> fp32 X and the pad flags (a frame whose H channels are all exactly 0)
//   k_pos_scan    positions over channel 0 (dsx_posemb.cuh)
//   k_fs2_embed   X = (X + alpha * table[pos]) * !pad, and LN1 of layer 0 -> fp16 A
//   per layer:
//     k_fs2_conv<F2_QKV>   A . in_proj^T: Q (scaled by D^-0.5 in fp32), K as fp16 [B][head][T][D], V transposed
//                          [B][head][D][Tp] (Tp = T rounded up to 64, zero past T)
//     k_fs2_attn<D>        softmax(Q K^T + key mask) V per head, flash style -> fp16 O [B][T][H]
//     k_fs2_conv<F2_RES>   O . out_proj^T + X, * !pad -> X; LN2 -> fp16 A
//     k_fs2_conv<F2_FFN1>  k-tap conv of A (+ bias) * k^-0.5, GELU or ReLU -> fp16 F [B][T][4H]
//     k_fs2_conv<F2_RES>   F . ffn_2^T + bias + X, * !pad -> X; LN1 of the next layer -> A, or after the last layer
//                          the final LayerNorm * !pad -> the fp32 output
// GEMMs use the implicit-GEMM core of dsx_conv.cuh (fp16 operands, fp32 accumulation).  The residual stream, LayerNorm
// statistics and the softmax state are fp32.  Everything after k_fs2_pack is fs2_stack_run, which the FFT diffusion
// denoiser (dsx_fftdiff.cu) runs on its own buffers; its layers (fs2_layers_run) are also the FastSpeech2 encoder's
// (dsx_fs2enc.cu), after an entry of its own.
//
// Padded rows: a padding frame is 0 after each mask, but LN2(0) = beta2 is what the FFN conv's taps read from it, as in
// the reference, so LN2 is written for every row < T; only rows at or past T read as the conv's zero padding.
#include <math.h>
#include <stdio.h>

#include <algorithm>

#include "dsx_conv.cuh"
#include "dsx_internal.h"
#include "dsx_posemb.cuh"
#include "dsx_ptx.cuh"

namespace dsx {
namespace {

constexpr float kFs2LnEps = 1e-5f;   // common_layers.LayerNorm, nn.LayerNorm defaults
constexpr int kFs2MaxLayers = 64;

enum { F2_QKV = 0, F2_FFN1 = 1, F2_RES = 2 };

struct Fs2ConvArgs {
  ConvGemm g;
  const __half* x;             // [B][T][g.cin]
  int T, Tp, mode;
  // F2_QKV
  int H, heads, D;
  float qscale;                // head_dim^-0.5
  __half* q;                   // [B][heads][T][D]
  __half* k;                   // [B][heads][T][D]
  __half* vt;                  // [B][heads][D][Tp]
  // F2_FFN1
  float ffn_scale;             // kernel_size^-0.5
  int relu;                    // 0 GELU (erf), 1 ReLU
  __half* o16;                 // [B][T][n]
  // F2_RES
  const uint8_t* pad;          // [B][T]
  float* xres;                 // [B][T][n] residual stream, updated in place
  const float* ln_w;           // LayerNorm applied after the residual update
  const float* ln_b;
  __half* ln16;                // [B][T][n] LayerNorm output, every row < T
  float* out;                  // non-null: LayerNorm * !pad -> out [B][T][n] fp32 instead of ln16
  int mask16;                  // with ln16: LayerNorm * !pad (the FFT denoiser's get_mel_out operand)
  // training forward (Fs2Train); drop.site < 0 and null pointers otherwise
  Fs2Drop drop;                // F2_FFN1: dropout after the activation; F2_RES: dropout of the GEMM output + bias
  __half* vrow;                // F2_QKV: V as [B][heads][T][D] as well
  __half* z16;                 // F2_FFN1: the activation's input [B][T][n]
  float* xsave;                // F2_RES: a copy of the updated residual stream [B][T][n]
};

template <int NT>
struct Fs2Shape {
  static constexpr int WG = NT > 128 ? 2 : 1;      // warpgroups per CTA; each owns NH columns of the same 64 rows
  static constexpr int NH = NT / WG;
};

// One 64-row x NT-column tile (column tile blockIdx.z) of utterance blockIdx.y.
template <int NT>
__global__ void __launch_bounds__(128 * Fs2Shape<NT>::WG) k_fs2_conv(const Fs2ConvArgs p) {
  constexpr int NH = Fs2Shape<NT>::NH, WG = Fs2Shape<NT>::WG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ float xrow[WG][kConvRows];
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, b = blockIdx.y, m0 = blockIdx.x * kConvRows;
  const int tile = blockIdx.z, T = p.T;

  float acc[NH / 2];
  conv_k_loop<NT, WG>(p.g, p.x, T, T, b, m0, tile, smem, acc);

  const int n = p.g.n, c0 = tile * NT + wg * NH;
  const int r0 = acc_row(wtid, 0);
  const int mrow[2] = {m0 + r0, m0 + r0 + 8};
  const size_t rbase = static_cast<size_t>(b) * T;

  if (p.mode == F2_QKV) {
    // column col: part col / H (q, k, v), head, d; rows in [T, Tp) are 0 (zero A rows, no bias) and written to V only
#pragma unroll
    for (int e = 0; e < NH / 2; e += 2) {
      const int col = c0 + acc_col(wtid, e), m = mrow[(e >> 1) & 1];
      if (col >= n) continue;
      const int part = col / p.H, w = col - part * p.H, hd = w / p.D, d = w - hd * p.D;
      const size_t bh = static_cast<size_t>(b) * p.heads + hd;
      if (part == 2) {
        if (m >= p.Tp) continue;
        __half* v = p.vt + (bh * p.D + d) * p.Tp + m;
        v[0] = __float2half_rn(acc[e]);
        v[p.Tp] = __float2half_rn(acc[e + 1]);
        if (p.vrow && m < T)
          *reinterpret_cast<__half2*>(p.vrow + (bh * T + m) * p.D + d) = __floats2half2_rn(acc[e], acc[e + 1]);
      } else {
        if (m >= T) continue;
        const float s = part == 0 ? p.qscale : 1.f;
        __half* dst = (part == 0 ? p.q : p.k) + (bh * T + m) * p.D + d;
        *reinterpret_cast<__half2*>(dst) = __floats2half2_rn(acc[e] * s, acc[e + 1] * s);
      }
    }
    return;
  }

  if (p.mode == F2_FFN1) {
#pragma unroll
    for (int e = 0; e < NH / 2; e += 2) {
      const int col = c0 + acc_col(wtid, e), m = mrow[(e >> 1) & 1];
      if (col >= n || m >= T) continue;
      float v[2], y[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        y[i] = (acc[e + i] + __ldg(p.g.b + col + i)) * p.ffn_scale;
        v[i] = p.relu ? fmaxf(y[i], 0.f) : 0.5f * y[i] * (1.f + erff(y[i] * 0.70710678118654752f));
      }
      if (p.z16) {
        *reinterpret_cast<__half2*>(p.z16 + (rbase + m) * n + col) = __floats2half2_rn(y[0], y[1]);
        const float2 ds = dropout_scale2(p.drop, rbase + m, col);
        v[0] *= ds.x;
        v[1] *= ds.y;
      }
      *reinterpret_cast<__half2*>(p.o16 + (rbase + m) * n + col) = __floats2half2_rn(v[0], v[1]);
    }
    return;
  }

  // F2_RES: one column tile holds the whole row (NT >= n).  x = (x + acc + bias) * !pad, then the LayerNorm of the row.
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
  const bool keep[2] = {mrow[0] < T && !p.pad[rbase + min(mrow[0], T - 1)],
                        mrow[1] < T && !p.pad[rbase + min(mrow[1], T - 1)]};
#pragma unroll
  for (int e = 0; e < NH / 2; e += 2) {
    const int col = c0 + acc_col(wtid, e), r = (e >> 1) & 1, m = mrow[r];
    float v0 = 0.f, v1 = 0.f;
    if (col < n && keep[r]) {
      float* xp = p.xres + (rbase + m) * n + col;
      const float2 xo = *reinterpret_cast<const float2*>(xp);
      if (p.drop.site >= 0) {
        const float2 ds = dropout_scale2(p.drop, rbase + m, col);
        v0 = xo.x + (acc[e] + __ldg(p.g.b + col)) * ds.x;
        v1 = xo.y + (acc[e + 1] + __ldg(p.g.b + col + 1)) * ds.y;
      } else {
        v0 = xo.x + (acc[e] + __ldg(p.g.b + col));
        v1 = xo.y + (acc[e + 1] + __ldg(p.g.b + col + 1));
      }
    }
    if (col < n && m < T) {
      *reinterpret_cast<float2*>(p.xres + (rbase + m) * n + col) = make_float2(v0, v1);
      if (p.xsave) *reinterpret_cast<float2*>(p.xsave + (rbase + m) * n + col) = make_float2(v0, v1);
    }
    acc[e] = v0;
    acc[e + 1] = v1;
  }
  const float inv_n = 1.f / static_cast<float>(n);
  float s[2] = {0.f, 0.f};
#pragma unroll
  for (int e = 0; e < NH / 2; ++e) s[(e >> 1) & 1] += acc[e];
  row_sum(s[0], s[1]);
  const float mean0 = s[0] * inv_n, mean1 = s[1] * inv_n;
  float q[2] = {0.f, 0.f};
#pragma unroll
  for (int e = 0; e < NH / 2; ++e) {
    const int col = c0 + acc_col(wtid, e);
    const float d = acc[e] - ((e & 2) ? mean1 : mean0);
    q[(e >> 1) & 1] += col < n ? d * d : 0.f;
  }
  row_sum(q[0], q[1]);
  const float rstd[2] = {1.f / sqrtf(q[0] * inv_n + kFs2LnEps), 1.f / sqrtf(q[1] * inv_n + kFs2LnEps)};
  const float mean[2] = {mean0, mean1};
#pragma unroll
  for (int e = 0; e < NH / 2; e += 2) {
    const int col = c0 + acc_col(wtid, e), r = (e >> 1) & 1, m = mrow[r];
    if (col >= n || m >= T) continue;
    const float y0 = (acc[e] - mean[r]) * rstd[r] * __ldg(p.ln_w + col) + __ldg(p.ln_b + col);
    const float y1 = (acc[e + 1] - mean[r]) * rstd[r] * __ldg(p.ln_w + col + 1) + __ldg(p.ln_b + col + 1);
    const size_t idx = (rbase + m) * n + col;
    if (p.out) {
      *reinterpret_cast<float2*>(p.out + idx) = keep[r] ? make_float2(y0, y1) : make_float2(0.f, 0.f);
    } else if (p.mask16 && !keep[r]) {
      *reinterpret_cast<__half2*>(p.ln16 + idx) = __floats2half2_rn(0.f, 0.f);
    } else {
      *reinterpret_cast<__half2*>(p.ln16 + idx) = __floats2half2_rn(y0, y1);
    }
  }
}

// ---- attention -----------------------------------------------------------------------------------
// One warpgroup per 64 query rows of one head of one utterance.  Key blocks of 64 (K [64][D] and V^T [D][64]) stream
// through two cp.async stages in the 128-byte-swizzled layout; S = Q K^T and O += P V run on wgmma with both operands in
// shared memory (P rounded to fp16 through a swizzled tile).  Padding keys and keys at or past T get -inf; the softmax
// state (running max and sum per row) is fp32.  A row whose keys are all padding has sum 0 and is written as 0 (the
// reference's 0 / 0 gives NaN there).  With lse (the training forward), the row's log-sum-exp max + log(sum) goes to
// lse [B][heads][T], +inf for a row with no valid key.
template <int D>
constexpr int attn_smem() { return 64 * D * 2 * 3 + D * 64 * 2 * 2 + 64 * 64 * 2 + 1024; }

template <int D>
__global__ void __launch_bounds__(128) k_fs2_attn(const __half* __restrict__ q, const __half* __restrict__ k,
                                                 const __half* __restrict__ vt, const uint8_t* __restrict__ pad, int T,
                                                 int Tp, int heads, __half* __restrict__ o, float* __restrict__ lse) {
  constexpr int kQ = 64 * D * 2, kV = D * 64 * 2;   // bytes of a 64 x D tile (Q, K) and of a D x 64 tile (V^T)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kQ;          // 2 stages
  uint8_t* sV = sK + 2 * kQ;      // 2 stages
  uint8_t* sP = sV + 2 * kV;
  __shared__ float kbias[2][64];  // 0 or -inf per key of a stage
  const int tid = threadIdx.x, m0 = blockIdx.x * 64, hd = blockIdx.y, b = blockIdx.z;
  const size_t bh = static_cast<size_t>(b) * heads + hd;
  const __half* qg = q + bh * T * D;
  const __half* kg = k + bh * T * D;
  const __half* vg = vt + bh * D * Tp;
  const uint8_t* pb = pad + static_cast<size_t>(b) * T;

  // 64 rows x D of a [T][D] array from row0, zero past T: D / 64 swizzled 64 x 64 tiles, 8 KB apart
  auto load_rows = [&](uint8_t* dst, const __half* src, int row0) {
#pragma unroll
    for (int it = 0; it < D / 16; ++it) {
      const int i = tid + it * 128, r = i / (D / 8), cc = i % (D / 8), row = row0 + r;
      const bool ok = row < T;
      cp16(smem_u32(dst + (cc >> 3) * 8192) + sw128(r, cc & 7), src + static_cast<size_t>(ok ? row : 0) * D + cc * 8, ok);
    }
  };
  auto load_kv = [&](int j, int st) {
    load_rows(sK + st * kQ, kg, j * 64);
#pragma unroll
    for (int it = 0; it < D / 16; ++it) {        // V^T rows d, keys j * 64 .. + 63 (inside Tp)
      const int i = tid + it * 128, r = i >> 3, c = i & 7;
      cp16(smem_u32(sV + st * kV) + sw128(r, c), vg + static_cast<size_t>(r) * Tp + j * 64 + c * 8, true);
    }
    if (tid < 64) {
      const int key = j * 64 + tid;
      kbias[st][tid] = (key < T && !pb[key]) ? 0.f : -INFINITY;
    }
  };

  load_rows(sQ, qg, m0);
  load_kv(0, 0);
  cp_commit();

  float oacc[D / 2];
#pragma unroll
  for (int e = 0; e < D / 2; ++e) oacc[e] = 0.f;
  float mrun[2] = {-INFINITY, -INFINITY}, lrun[2] = {0.f, 0.f};
  const int nblk = (T + 63) / 64;
#pragma unroll 1
  for (int j = 0; j < nblk; ++j) {
    const int st = j & 1;
    if (j + 1 < nblk) {
      load_kv(j + 1, st ^ 1);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();

    float s[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) s[e] = 0.f;
    wg_fence();
#pragma unroll
    for (int c = 0; c < D / 64; ++c) {
      const uint64_t da = wg_desc(smem_u32(sQ + c * 8192)), db = wg_desc(smem_u32(sK + st * kQ + c * 8192));
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) wgmma_f16<64>(s, da + 2 * k4, db + 2 * k4, 1);
    }
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < 32; ++e) asm volatile("" : "+f"(s[e])::"memory");

    // online softmax: each thread holds rows r0 (e & 2 == 0) and r0 + 8 of the tile, 16 keys each
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int e = 0; e < 32; ++e) {
      s[e] += kbias[st][acc_col(tid, e)];
      mx[(e >> 1) & 1] = fmaxf(mx[(e >> 1) & 1], s[e]);
    }
    float base[2], alpha[2], ls[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      const float mnew = fmaxf(mrun[r], mx[r]);
      base[r] = mnew == -INFINITY ? 0.f : mnew;   // no valid key yet: every p is exp(-inf) = 0
      alpha[r] = __expf(mrun[r] - base[r]);
      mrun[r] = mnew;
    }
#pragma unroll
    for (int e = 0; e < 32; e += 2) {
      const int r = (e >> 1) & 1;
      const float p0 = __expf(s[e] - base[r]), p1 = __expf(s[e + 1] - base[r]);
      ls[r] += p0 + p1;
      const int row = acc_row(tid, e), col = acc_col(tid, e);
      *reinterpret_cast<__half2*>(sP + sw128(row, col >> 3) + (col & 7) * 2) = __floats2half2_rn(p0, p1);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) lrun[r] = lrun[r] * alpha[r] + quad_sum(ls[r]);
#pragma unroll
    for (int e = 0; e < D / 2; ++e) oacc[e] *= alpha[(e >> 1) & 1];
    fence_proxy_async_smem();
    __syncthreads();

    wg_fence();
    {
      const uint64_t da = wg_desc(smem_u32(sP)), db = wg_desc(smem_u32(sV + st * kV));
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) wgmma_f16<D>(oacc, da + 2 * k4, db + 2 * k4, 1);
    }
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < D / 2; ++e) asm volatile("" : "+f"(oacc[e])::"memory");
    __syncthreads();   // stage st and P are free for the next block
  }

  const int H = heads * D;
  if (lse && (tid & 3) == 0) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int m = m0 + acc_row(tid, 2 * r);
      if (m < T) lse[bh * T + m] = lrun[r] > 0.f ? mrun[r] + logf(lrun[r]) : INFINITY;
    }
  }
#pragma unroll
  for (int e = 0; e < D / 2; e += 2) {
    const int r = (e >> 1) & 1, m = m0 + acc_row(tid, e);
    if (m >= T) continue;
    const float inv = lrun[r] > 0.f ? 1.f / lrun[r] : 0.f;
    *reinterpret_cast<__half2*>(o + (static_cast<size_t>(b) * T + m) * H + hd * D + acc_col(tid, e)) =
        __floats2half2_rn(oacc[e] * inv, oacc[e + 1] * inv);
  }
}

// ---- entry -------------------------------------------------------------------------------------------
// x logically [B, T, H] (any strides: b, c = channel, t) -> contiguous fp32 X and pad[b][t] = all H channels exactly 0
// (tts_modules.py:288, decided before the positions are added).  One warp per frame.
__global__ void k_fs2_pack(const float* x, dsx_strides xs, int B, int T, int H, float* X, uint8_t* pad) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * T) return;
  const int b = warp / T, t = warp - b * T;
  const float* src = x + b * xs.b + t * xs.t;
  bool nz = false;
  for (int c = lane; c < H; c += 32) {
    const float v = src[c * xs.c];
    nz |= v != 0.f;
    X[static_cast<size_t>(warp) * H + c] = v;
  }
  const unsigned any = __ballot_sync(0xffffffffu, nz);
  if (lane == 0) pad[warp] = any ? 0 : 1;
}

// X = (X + alpha * table[pos]) * !pad (tts_modules.py:290-295), then LayerNorm (layer 0's layer_norm1) -> fp16 A.
// One warp per frame, H / 32 <= 8 channels per lane.  Training: dropout (site `drop`) before the mask, and X copied to
// xsave.
__global__ void k_fs2_embed(float* X, const int* pos, const uint8_t* pad, const float* alpha, int rows, int H,
                            float neg_emb, const float* ln_w, const float* ln_b, __half* A, Fs2Drop drop,
                            float* xsave) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int ps = pos[warp], per = H / 32;
  const bool keep = !pad[warp];
  float* xr = X + static_cast<size_t>(warp) * H;
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (i >= per) break;
    const int c = lane + 32 * i;
    float y = xr[c] + alpha[0] * pos_table(ps, c, H, neg_emb);
    if (drop.site >= 0) y *= dropout_scale(drop, warp, c);
    v[i] = keep ? y : 0.f;
    xr[c] = v[i];
    if (xsave) xsave[static_cast<size_t>(warp) * H + c] = v[i];
  }
  warp_row_ln16(v, per, H, kFs2LnEps, ln_w, ln_b, A + static_cast<size_t>(warp) * H);
}

}  // namespace
}  // namespace dsx

using namespace dsx;

struct dsx_fs2dec {
  struct Layer {
    ConvGemm qkv, out, ffn1, ffn2;
    float *ln1_w = nullptr, *ln1_b = nullptr, *ln2_w = nullptr, *ln2_b = nullptr;
  };
  int device = 0;
  dsx_fs2dec_config cfg{};
  bool loaded = false;
  std::vector<Layer> layers;
  float* lnf_w = nullptr;      // layer_norm
  float* lnf_b = nullptr;
  float* alpha = nullptr;      // pos_embed_alpha [1]
  DevAllocs mem;               // the packs above
  GrowBuffer ws;               // workspace of a forward call
};

namespace {

int f2_copy(dsx_fs2dec* h, float** dst, const float* src, int n, const char* what, int layer, cudaStream_t s) {
  DSX_CHECK(src, DSX_E_INVALID, "missing %s of layer %d", what, layer);
  DSX_TRY(h->mem.alloc(dst, static_cast<size_t>(n) * sizeof(float)));
  DSX_CUDA(cudaMemcpyAsync(*dst, src, static_cast<size_t>(n) * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return DSX_OK;
}

// pack a conv (k taps from tap0) or linear (k = 1) of cin -> n channels into column tiles of up to 256
int f2_pack(dsx_fs2dec* h, ConvGemm& g, const float* w, const float* b, int cin, int n, int k, int tap0,
            const char* what, int layer, cudaStream_t s) {
  DSX_CHECK(w, DSX_E_INVALID, "missing %s weight of layer %d", what, layer);
  g.cin = cin;
  g.n = n;
  g.taps = k;
  g.tap0 = tap0;
  return conv_pack(h->mem, g, 256, PackArgs{w, nullptr, b, cin, n, n, k, 1, 0}, s);
}

int f2_run(const ConvGemm& g, Fs2ConvArgs a, int B, cudaStream_t s) {
  a.g = g;
  const dim3 grid((a.T + kConvRows - 1) / kConvRows, B, g.ntiles);
  return conv_dispatch<256>(g.nt, [&](auto c) {
    constexpr int NT = decltype(c)::value;
    k_fs2_conv<NT><<<grid, 128 * Fs2Shape<NT>::WG, conv_smem<NT>(), s>>>(a);
    return launch_check("k_fs2_conv");
  });
}

int f2_validate(const dsx_fs2dec_config* c) {
  DSX_CHECK(c, DSX_E_INVALID, "config is NULL");
  DSX_CHECK(c->hidden >= 64 && c->hidden <= 256 && c->hidden % 64 == 0, DSX_E_INVALID,
            "unsupported hidden %d: a multiple of 64 in [64, 256]", c->hidden);
  DSX_CHECK(c->layers >= 1 && c->layers <= kFs2MaxLayers, DSX_E_INVALID, "unsupported layers %d: 1..%d", c->layers,
            kFs2MaxLayers);
  DSX_CHECK(c->heads >= 1 && c->hidden % c->heads == 0 &&
                (c->hidden / c->heads == 64 || c->hidden / c->heads == 128),
            DSX_E_INVALID, "unsupported heads %d: hidden / heads must be 64 or 128", c->heads);
  DSX_CHECK(c->padding == 0 || c->padding == 1, DSX_E_INVALID, "unsupported padding %d: 0 (SAME) or 1 (LEFT)",
            c->padding);
  DSX_CHECK(c->kernel >= 1 && c->kernel <= 255 && (c->padding == 1 || c->kernel % 2 == 1), DSX_E_INVALID,
            "unsupported ffn kernel %d: in [1, 255], odd for SAME", c->kernel);
  DSX_CHECK(c->act == 0 || c->act == 1, DSX_E_INVALID, "unsupported act %d: 0 (gelu) or 1 (relu)", c->act);
  return DSX_OK;
}

template <int D>
int attn_opt_in() {
  DSX_CUDA(cudaFuncSetAttribute(k_fs2_attn<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, attn_smem<D>()));
  return DSX_OK;
}

}  // namespace

namespace dsx {

// fp32 X, fp16 A (LayerNorm outputs), O (attention), Q, K, F (FFN hidden), V^T, pad flags, positions
size_t fs2_workspace_bytes(const dsx_fs2dec* h, int B, int T) {
  const int H = h->cfg.hidden, Tp = (T + kConvRows - 1) / kConvRows * kConvRows;
  const size_t frames = static_cast<size_t>(B) * T;
  return align256(frames * H * 4) + 4 * align256(frames * H * 2) + align256(frames * 4 * H * 2) +
         align256(static_cast<size_t>(B) * Tp * H * 2) + align256(frames) + align256(frames * 4);
}

Fs2Bufs fs2_carve(const dsx_fs2dec* h, void* base, int B, int T) {
  const int H = h->cfg.hidden, Tp = (T + kConvRows - 1) / kConvRows * kConvRows;
  const size_t frames = static_cast<size_t>(B) * T;
  Bump ws{static_cast<uint8_t*>(base)};
  Fs2Bufs w;
  w.X = ws.take<float>(frames * H * 4);
  w.A = ws.take<__half>(frames * H * 2);
  w.O = ws.take<__half>(frames * H * 2);
  w.Q = ws.take<__half>(frames * H * 2);
  w.K = ws.take<__half>(frames * H * 2);
  w.F = ws.take<__half>(frames * 4 * H * 2);
  w.VT = ws.take<__half>(static_cast<size_t>(B) * Tp * H * 2);
  w.PAD = ws.take<uint8_t>(frames);
  w.POS = ws.take<int>(frames * 4);
  return w;
}

int fs2_layers(const dsx_fs2dec* h) { return h->cfg.layers; }

int fs2_stack_run(const dsx_fs2dec* h, const Fs2Bufs& w, int B, int T, float* out, __half* out16, cudaStream_t s,
                  const Fs2Train* tr) {
  const int H = h->cfg.hidden;
  const size_t frames = static_cast<size_t>(B) * T;
  const unsigned row_blocks = static_cast<unsigned>((frames * 32 + 255) / 256);
  k_pos_scan<<<B, kScanThreads, 0, s>>>(w.X, T, H, w.POS);
  DSX_TRY(launch_check("k_pos_scan"));
  k_fs2_embed<<<row_blocks, 256, 0, s>>>(w.X, w.POS, w.PAD, h->alpha, static_cast<int>(frames), H, pos_neg_emb(H),
                                         h->layers[0].ln1_w, h->layers[0].ln1_b, tr ? tr->a1[0] : w.A,
                                         tr ? tr->drop(0) : Fs2Drop{}, tr ? tr->xin[0] : nullptr);
  DSX_TRY(launch_check("k_fs2_embed"));
  return fs2_layers_run(h, w, B, T, out, out16, s, tr);
}

void fs2_first_ln(const dsx_fs2dec* h, const float** w, const float** b) {
  *w = h->layers[0].ln1_w;
  *b = h->layers[0].ln1_b;
}

int fs2_layers_run(const dsx_fs2dec* h, const Fs2Bufs& w, int B, int T, float* out, __half* out16, cudaStream_t s,
                   const Fs2Train* tr) {
  const dsx_fs2dec_config& c = h->cfg;
  const int H = c.hidden, L = c.layers, heads = c.heads, D = H / heads;
  const int mtiles = (T + kConvRows - 1) / kConvRows, Tp = mtiles * kConvRows;

  Fs2ConvArgs base{};
  base.T = T;
  base.Tp = Tp;
  base.H = H;
  base.heads = heads;
  base.D = D;
  base.pad = w.PAD;
  base.xres = w.X;
  for (int i = 0; i < L; ++i) {
    const dsx_fs2dec::Layer& l = h->layers[i];
    // the training forward keeps the GEMM operands on its tape; evaluation reuses the workspace's
    __half* A1 = tr ? tr->a1[i] : w.A;
    __half* A2 = tr ? tr->a2[i] : w.A;
    __half* Q = tr ? tr->q[i] : w.Q;
    __half* K = tr ? tr->k[i] : w.K;
    __half* O = tr ? tr->o[i] : w.O;
    __half* Fh = tr ? tr->hd[i] : w.F;
    float* lse = tr ? tr->lse[i] : nullptr;
    // self-attention block (common_layers.py:569-580): x = (x + out_proj(MHA(LN1(x)))) * !pad
    Fs2ConvArgs a = base;
    a.x = A1;
    a.mode = F2_QKV;
    a.qscale = static_cast<float>(sqrt(1.0 / D));   // math.sqrt(1 / head_dim) of F.multi_head_attention_forward
    a.q = Q;
    a.k = K;
    a.vt = w.VT;
    if (tr) a.vrow = tr->v[i];
    DSX_TRY(f2_run(l.qkv, a, B, s));
    const dim3 agrid(mtiles, heads, B);
    if (D == 64) {
      k_fs2_attn<64><<<agrid, 128, attn_smem<64>(), s>>>(Q, K, w.VT, w.PAD, T, Tp, heads, O, lse);
    } else {
      k_fs2_attn<128><<<agrid, 128, attn_smem<128>(), s>>>(Q, K, w.VT, w.PAD, T, Tp, heads, O, lse);
    }
    DSX_TRY(launch_check("k_fs2_attn"));
    a = base;
    a.x = O;
    a.mode = F2_RES;
    a.ln_w = l.ln2_w;
    a.ln_b = l.ln2_b;
    a.ln16 = A2;
    if (tr) {
      a.drop = tr->drop(1 + 3 * i);
      a.xsave = tr->xin[2 * i + 1];
    }
    DSX_TRY(f2_run(l.out, a, B, s));
    // FFN block (:582-587, TransformerFFNLayer :503-522): x = (x + ffn_2(act(ffn_1(LN2(x)) * k^-0.5))) * !pad
    a = base;
    a.x = A2;
    a.mode = F2_FFN1;
    a.ffn_scale = static_cast<float>(pow(static_cast<double>(c.kernel), -0.5));
    a.relu = c.act;
    a.o16 = Fh;
    if (tr) {
      a.drop = tr->drop(2 + 3 * i);
      a.z16 = tr->z[i];
    }
    DSX_TRY(f2_run(l.ffn1, a, B, s));
    a = base;
    a.x = Fh;
    a.mode = F2_RES;
    if (tr) {
      a.drop = tr->drop(3 + 3 * i);
      a.xsave = tr->xin[2 * i + 2];
    }
    if (i + 1 < L) {
      a.ln_w = h->layers[i + 1].ln1_w;
      a.ln_b = h->layers[i + 1].ln1_b;
      a.ln16 = tr ? tr->a1[i + 1] : w.A;
    } else {   // tts_modules.py:300-301: layer_norm(x) * !pad
      a.ln_w = h->lnf_w;
      a.ln_b = h->lnf_b;
      a.out = out;
      a.ln16 = out16;
      a.mask16 = out16 != nullptr;
    }
    DSX_TRY(f2_run(l.ffn2, a, B, s));
  }
  return DSX_OK;
}

}  // namespace dsx

extern "C" {

int dsx_fs2dec_create(int device, const dsx_fs2dec_config* cfg, dsx_fs2dec** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_TRY(f2_validate(cfg));
  DSX_TRY(select_sm90_device(device, "FastSpeech2 decoder"));
  DSX_TRY(conv_opt_in<256>([](auto c) { return k_fs2_conv<decltype(c)::value>; }));
  DSX_TRY(attn_opt_in<64>());
  DSX_TRY(attn_opt_in<128>());
  dsx_fs2dec* h = new dsx_fs2dec();
  h->device = device;
  h->cfg = *cfg;
  *out = h;
  return DSX_OK;
}

void dsx_fs2dec_destroy(dsx_fs2dec* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  h->mem.free_all();
  h->ws.release();
  delete h;
}

int dsx_fs2dec_load(dsx_fs2dec* h, const dsx_fs2dec_params* p, void* stream) {
  DSX_CHECK(h && p, DSX_E_INVALID, "null handle or params");
  DSX_CHECK(p->pos_embed_alpha, DSX_E_INVALID, "missing layer_norm or pos_embed_alpha");
  return fs2_load(h, p, stream);
}

}  // extern "C"

namespace dsx {

// dsx_fs2dec_load without pos_embed_alpha, which the encoder's stack does not have (h->alpha stays NULL without it)
int fs2_load(dsx_fs2dec* h, const dsx_fs2dec_params* p, void* stream) {
  DSX_CHECK(h && p, DSX_E_INVALID, "null handle or params");
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const dsx_fs2dec_config& c = h->cfg;
  const int H = c.hidden, L = c.layers, k = c.kernel;
  DSX_CHECK(p->ln1_w && p->ln1_b && p->in_proj_w && p->out_proj_w && p->ln2_w && p->ln2_b && p->ffn1_w && p->ffn1_b &&
                p->ffn2_w && p->ffn2_b,
            DSX_E_INVALID, "missing per-layer arrays");
  DSX_CHECK(p->ln_w && p->ln_b, DSX_E_INVALID, "missing layer_norm");
  DSX_CUDA(cudaStreamSynchronize(s));   // the old packs may still be read by queued work
  h->mem.free_all();
  h->loaded = false;
  h->layers.assign(L, dsx_fs2dec::Layer{});
  const int tap0 = c.padding ? -(k - 1) : -(k / 2);   // ConstantPad1d (k - 1, 0) or padding = k // 2
  for (int i = 0; i < L; ++i) {
    dsx_fs2dec::Layer& l = h->layers[i];
    DSX_TRY(f2_copy(h, &l.ln1_w, p->ln1_w[i], H, "layer_norm1.weight", i, s));
    DSX_TRY(f2_copy(h, &l.ln1_b, p->ln1_b[i], H, "layer_norm1.bias", i, s));
    DSX_TRY(f2_copy(h, &l.ln2_w, p->ln2_w[i], H, "layer_norm2.weight", i, s));
    DSX_TRY(f2_copy(h, &l.ln2_b, p->ln2_b[i], H, "layer_norm2.bias", i, s));
    DSX_TRY(f2_pack(h, l.qkv, p->in_proj_w[i], nullptr, H, 3 * H, 1, 0, "self_attn.in_proj", i, s));
    DSX_TRY(f2_pack(h, l.out, p->out_proj_w[i], nullptr, H, H, 1, 0, "self_attn.out_proj", i, s));
    DSX_CHECK(p->ffn1_b[i] && p->ffn2_b[i], DSX_E_INVALID, "missing ffn bias of layer %d", i);
    DSX_TRY(f2_pack(h, l.ffn1, p->ffn1_w[i], p->ffn1_b[i], H, 4 * H, k, tap0, "ffn.ffn_1", i, s));
    DSX_TRY(f2_pack(h, l.ffn2, p->ffn2_w[i], p->ffn2_b[i], 4 * H, H, 1, 0, "ffn.ffn_2", i, s));
  }
  DSX_TRY(f2_copy(h, &h->lnf_w, p->ln_w, H, "layer_norm.weight", L, s));
  DSX_TRY(f2_copy(h, &h->lnf_b, p->ln_b, H, "layer_norm.bias", L, s));
  h->alpha = nullptr;
  if (p->pos_embed_alpha) DSX_TRY(f2_copy(h, &h->alpha, p->pos_embed_alpha, 1, "pos_embed_alpha", L, s));
  h->loaded = true;
  return DSX_OK;
}

int fs2_forward_run(const dsx_fs2dec* h, const float* x, dsx_strides xs, int B, int T, const Fs2Bufs& w, float* out,
                    cudaStream_t s, const Fs2Train* tr) {
  const size_t frames = static_cast<size_t>(B) * T;
  k_fs2_pack<<<static_cast<unsigned>((frames * 32 + 255) / 256), 256, 0, s>>>(x, xs, B, T, h->cfg.hidden, w.X, w.PAD);
  DSX_TRY(launch_check("k_fs2_pack"));
  return fs2_stack_run(h, w, B, T, out, nullptr, s, tr);
}

const dsx_fs2dec_config& fs2_config(const dsx_fs2dec* h) { return h->cfg; }

namespace {
// g's tile shape as f2_pack gives it, with its packs allocated but not filled
int f2_alloc(dsx_fs2dec* h, ConvGemm& g, int cin, int n, int k, int tap0) {
  g.cin = cin;
  g.n = n;
  g.taps = k;
  g.tap0 = tap0;
  g.nt = conv_nt(n, 256);
  g.ntiles = (n + g.nt - 1) / g.nt;
  g.kc = (k * cin + 63) / 64;
  DSX_TRY(h->mem.alloc(&g.w, static_cast<size_t>(g.ntiles) * g.kc * g.nt * 64 * sizeof(__half)));
  return h->mem.alloc(&g.b, static_cast<size_t>(g.ntiles) * g.nt * sizeof(float));
}

int f2_refill(const ConvGemm& g, const float* w, const float* b, int k, const char* what, int layer, cudaStream_t s) {
  DSX_CHECK(w, DSX_E_INVALID, "missing %s weight of layer %d", what, layer);
  const size_t nw = static_cast<size_t>(g.ntiles) * g.kc * g.nt * 64;
  k_pack_conv<<<static_cast<unsigned>(std::min<size_t>((nw + 255) / 256, 4096)), 256, 0, s>>>(
      g, PackArgs{w, nullptr, b, g.cin, g.n, g.n, k, 1, 0});
  return launch_check("k_pack_conv");
}
}  // namespace

int fs2_train_alloc(dsx_fs2dec* h) {
  const dsx_fs2dec_config& c = h->cfg;
  const int H = c.hidden, L = c.layers, k = c.kernel;
  const int tap0 = c.padding ? -(k - 1) : -(k / 2);
  h->layers.assign(L, dsx_fs2dec::Layer{});
  for (int i = 0; i < L; ++i) {
    dsx_fs2dec::Layer& l = h->layers[i];
    DSX_TRY(f2_alloc(h, l.qkv, H, 3 * H, 1, 0));
    DSX_TRY(f2_alloc(h, l.out, H, H, 1, 0));
    DSX_TRY(f2_alloc(h, l.ffn1, H, 4 * H, k, tap0));
    DSX_TRY(f2_alloc(h, l.ffn2, 4 * H, H, 1, 0));
  }
  return DSX_OK;
}

int fs2_train_pack(dsx_fs2dec* h, const dsx_fs2dec_params* p, cudaStream_t s) {
  const dsx_fs2dec_config& c = h->cfg;
  const int L = c.layers;
  for (int i = 0; i < L; ++i) {
    dsx_fs2dec::Layer& l = h->layers[i];
    DSX_TRY(f2_refill(l.qkv, p->in_proj_w[i], nullptr, 1, "self_attn.in_proj", i, s));
    DSX_TRY(f2_refill(l.out, p->out_proj_w[i], nullptr, 1, "self_attn.out_proj", i, s));
    DSX_TRY(f2_refill(l.ffn1, p->ffn1_w[i], p->ffn1_b[i], c.kernel, "ffn.ffn_1", i, s));
    DSX_TRY(f2_refill(l.ffn2, p->ffn2_w[i], p->ffn2_b[i], 1, "ffn.ffn_2", i, s));
    l.ln1_w = const_cast<float*>(p->ln1_w[i]);
    l.ln1_b = const_cast<float*>(p->ln1_b[i]);
    l.ln2_w = const_cast<float*>(p->ln2_w[i]);
    l.ln2_b = const_cast<float*>(p->ln2_b[i]);
  }
  h->lnf_w = const_cast<float*>(p->ln_w);
  h->lnf_b = const_cast<float*>(p->ln_b);
  h->alpha = const_cast<float*>(p->pos_embed_alpha);
  h->loaded = true;
  return DSX_OK;
}

}  // namespace dsx

extern "C" {

int dsx_fs2dec_forward(dsx_fs2dec* h, const float* x, dsx_strides xs, int B, int T, float* out, void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(h->loaded, DSX_E_STATE, "dsx_fs2dec_load has not been called");
  DSX_CHECK(x && out, DSX_E_INVALID, "x and out must not be NULL");
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(B <= 65535, DSX_E_INVALID, "B = %d utterances per call is above the 65535 the launch grid holds", B);
  const int H = h->cfg.hidden;
  const int Tp = (T + kConvRows - 1) / kConvRows * kConvRows;
  DSX_CHECK(static_cast<long long>(B) * Tp * 4 * H < (1ll << 31), DSX_E_INVALID, "B * T = %lld frames is too large",
            static_cast<long long>(B) * T);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_TRY(h->ws.reserve(fs2_workspace_bytes(h, B, T), s));
  return fs2_forward_run(h, x, xs, B, T, fs2_carve(h, h->ws.ptr, B, T), out, s);
}

}  // extern "C"
