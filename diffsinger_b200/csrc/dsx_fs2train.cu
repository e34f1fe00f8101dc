// FastSpeech2 decoder training step on sm_90a: FFTBlocks.forward in training mode (modules/fastspeech/tts_modules.py:
// 282-307 with EncSALayer, modules/commons/common_layers.py:486-588), with what the backward needs saved to a
// caller-owned tape, and the exact backward to every decoder parameter and to decoder_inp.
//
// Forward: the eval decoder's kernels (dsx_fs2dec.cu) in their training form (Fs2Train): dropout in the entry and the
// epilogues, and on the tape the LayerNorm inputs (fp32), the GEMM operands (fp16), ffn_1's output before the activation
// (fp16) and the attention's log-sum-exp per (row, head) (fp32).  Dropout masks come from Philox keyed by (seed, site,
// frame, channel) (dsx_rng.cuh) and are not stored: the backward draws the same bits again, which costs 10 Philox rounds
// per 4 elements in epilogues that already read the element, instead of 1 + 3 L masks on the tape.
//
// Backward, per layer in reverse, with G the fp32 gradient of the residual stream [F][H]:
//   k_f2b_gemm B_GC    gY2 . ffn_2 -> * dropout(2 + 3 i) * act'(z) * k^-0.5 -> gC fp16 [F][4H]
//   k_f2b_gemm B_F32   ffn_1's stride-1 transposed conv of gC (taps reversed) -> gA fp32
//   k_f2b_ln           G += LN2 backward(gA), * !pad; gY = G * dropout(1 + 3 i) -> fp16
//   k_f2b_gemm B_F16   gY . out_proj -> dO fp16 [F][H]
//   k_attn_delta       D = rowsum(dO o O) per (row, head)
//   k_attn_bwd_kv<D>   per 64 keys: P = exp(Q K^T - lse) (fp16), dP = dO V^T, dS = P (dP - D); dK = dS^T Q,
//                      dV = P^T dO
//   k_attn_bwd_q<D>    per 64 queries: dQ = dS K * D^-0.5 (a pass of its own, so nothing is accumulated atomically)
//   k_f2b_gemm B_F32   [dQ | dK | dV] . in_proj -> gA
//   k_f2b_ln           G += LN1 backward(gA), * !pad; the operand of the layer below (dropout 3 + 3 (i - 1)), or at
//                      layer 0 the entry: d_x = G * dropout(0) and d alpha = sum d_x . table[pos]
// The attention backward runs on wgmma (P and dS go through shared memory as fp16 tiles); nothing of size T^2 reaches
// global memory.  Weight gradients use run_wgrad (dsx_wgrad.cuh): k_wgrad splits the frames over CTAs, k_wgrad_sum sums
// the partials in a fixed order.
// LayerNorm affine gradients and d alpha are per-CTA partials of k_f2b_ln (a fixed grid) summed in order.  No atomics
// touch a result, so two backwards of one tape are bitwise equal.
//
// Gradient operands are fp16 scaled by S, a power of two chosen on the device so that S amax |d_out| lies in [2^5, 2^6);
// every gradient written is multiplied by 1 / S, which is exact, so d_out * 2^k gives exactly 2^k times the gradients.
#include <math.h>

#include <algorithm>
#include <vector>

#include "dsx_conv.cuh"
#include "dsx_internal.h"
#include "dsx_posemb.cuh"
#include "dsx_ptx.cuh"
#include "dsx_wgrad.cuh"

namespace dsx {
namespace {

constexpr int kNT = 256;            // columns per CTA of the data-gradient GEMMs (two warpgroups)
constexpr int kLnBlocks = 256;      // CTAs of k_f2b_ln: fixed, so its partial sums have a fixed order
constexpr float kLnEps = 1e-5f;

enum { B_GC, B_F32, B_F16 };

using TapeHdr = Fs2TapeHdr;

struct BwdGemmArgs {
  ConvGemm g;
  const __half* x;             // A operand [B][T][g.cin]
  int T, mode;
  float* o32;                  // B_F32: [F][g.n]
  __half* o16;                 // B_GC, B_F16: [F][g.n]
  const __half* z;             // B_GC: ffn_1 output * k^-0.5 before the activation [F][g.n]
  const TapeHdr* hdr;          // B_GC: the dropout after the activation, site `site` of the tape's seed and p
  int site;
  int relu;
  float kscale;                // kernel_size^-0.5
};

// d act(z) / dz: GELU (erf form) or ReLU
__device__ __forceinline__ float act_grad(float z, int relu) {
  if (relu) return z > 0.f ? 1.f : 0.f;
  return 0.5f * (1.f + erff(z * 0.70710678118654752f)) + z * 0.39894228040143268f * expf(-0.5f * z * z);
}

template <int NT>
__global__ void __launch_bounds__(256) k_f2b_gemm(const BwdGemmArgs p) {
  constexpr int WG = 2, NH = NT / WG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, b = blockIdx.y, m0 = blockIdx.x * kConvRows;
  const int tile = blockIdx.z, T = p.T;
  float acc[NH / 2];
  conv_k_loop<NT, WG>(p.g, p.x, T, T, b, m0, tile, smem, acc);
  const int n = p.g.n, c0 = tile * NT + wg * NH, r0 = acc_row(wtid, 0);
#pragma unroll
  for (int e = 0; e < NH / 2; e += 2) {
    const int col = c0 + acc_col(wtid, e), m = m0 + r0 + ((e & 2) ? 8 : 0);
    if (col >= n || m >= T) continue;
    const size_t f = static_cast<size_t>(b) * T + m, idx = f * n + col;
    if (p.mode == B_F32) {
      *reinterpret_cast<float2*>(p.o32 + idx) = make_float2(acc[e], acc[e + 1]);
    } else if (p.mode == B_F16) {
      *reinterpret_cast<__half2*>(p.o16 + idx) = __floats2half2_rn(acc[e], acc[e + 1]);
    } else {
      const float2 z = __half22float2(*reinterpret_cast<const __half2*>(p.z + idx));
      const float2 ds = dropout_scale2(hdr_drop(p.hdr, p.site), f, col);
      *reinterpret_cast<__half2*>(p.o16 + idx) =
          __floats2half2_rn(acc[e] * ds.x * act_grad(z.x, p.relu) * p.kscale,
                            acc[e + 1] * ds.y * act_grad(z.y, p.relu) * p.kscale);
    }
  }
}

// ---- LayerNorm backward and the gradient stream; one warp per frame --------------------------------------------------
struct LnArgs {
  const float* gin;            // gradient at the LayerNorm output [F][H], scaled by S; from_dout: d_out (unscaled)
  int from_dout;               // gin = d_out: scale it by S and apply the output's * !pad
  const float* x;              // the LayerNorm input (tape)
  const float* gamma;
  const uint8_t* pad;
  float* G;                    // G = (G if accumulate) + LayerNorm backward, then * !pad
  int accumulate;
  __half* o16;                 // G * dropout(drop) -> fp16 [F][H], or null
  int entry;                   // layer 0: d_x = G * dropout(drop) / S and the d alpha partials
  float* dx;                   // entry: [F][H] fp32, or null
  const int* pos;              // entry: the positions of d alpha, or null (no d alpha)
  float neg_emb;
  const TapeHdr* hdr;          // the dropout of o16 or of the entry: site `site` of the tape's seed and p
  int site;
  float* part;                 // [gridDim.x][2 H + 1]: d gamma, d beta, d alpha of this CTA
  const float* scal;           // S, 1 / S
  int F, H;
};

__global__ void __launch_bounds__(256) k_f2b_ln(const LnArgs p) {
  __shared__ float red[8][2 * 256 + 1];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, H = p.H, per = H / 32;
  const float S = p.scal[0], is = p.scal[1], inv_h = 1.f / static_cast<float>(H);
  const Fs2Drop drop = hdr_drop(p.hdr, p.site);
  float dgam[8], dbet[8], dal = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) dgam[i] = dbet[i] = 0.f;
  for (int f = blockIdx.x * 8 + warp; f < p.F; f += gridDim.x * 8) {
    const size_t rb = static_cast<size_t>(f) * H;
    const bool keep = !p.pad[f];
    float xv[8], gv[8], sum = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i >= per) break;
      xv[i] = p.x[rb + lane + 32 * i];
      sum += xv[i];
    }
    const float mean = warp_sum(sum) * inv_h;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i >= per) break;
      const float d = xv[i] - mean;
      sq += d * d;
    }
    const float rstd = 1.f / sqrtf(warp_sum(sq) * inv_h + kLnEps);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i >= per) break;
      const int c = lane + 32 * i;
      float g = p.gin[rb + c];
      if (p.from_dout) g = keep ? g * S : 0.f;
      const float xh = (xv[i] - mean) * rstd;
      dgam[i] += g * xh;
      dbet[i] += g;
      const float gg = g * p.gamma[c];
      gv[i] = gg;
      xv[i] = xh;
      s1 += gg;
      s2 += gg * xh;
    }
    const float m1 = warp_sum(s1) * inv_h, m2 = warp_sum(s2) * inv_h;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      if (i >= per) break;
      const int c = lane + 32 * i;
      float v = rstd * (gv[i] - m1 - xv[i] * m2);
      if (p.accumulate) v += p.G[rb + c];
      v = keep ? v : 0.f;
      p.G[rb + c] = v;
      if (p.o16) p.o16[rb + c] = __float2half_rn(v * dropout_scale(drop, f, c));
      if (p.entry) {
        const float d = v * dropout_scale(drop, f, c);
        if (p.dx) p.dx[rb + c] = d * is;
        if (p.pos) dal += d * pos_table(p.pos[f], c, H, p.neg_emb);
      }
    }
  }
  dal = warp_sum(dal);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (i >= per) break;
    red[warp][lane + 32 * i] = dgam[i];
    red[warp][H + lane + 32 * i] = dbet[i];
  }
  if (lane == 0) red[warp][2 * H] = dal;
  __syncthreads();
  for (int t = threadIdx.x; t < 2 * H + 1; t += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w][t];
    p.part[static_cast<size_t>(blockIdx.x) * (2 * H + 1) + t] = s;
  }
}

// the partials of k_f2b_ln in CTA order, * 1 / S -> d gamma [H], d beta [H], d alpha (if non-null)
__global__ void k_f2b_ln_reduce(const float* part, int blocks, int H, const float* scal, float* dgamma, float* dbeta,
                                float* dalpha) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= 2 * H + 1) return;
  float s = 0.f;
  for (int k = 0; k < blocks; ++k) s += part[static_cast<size_t>(k) * (2 * H + 1) + t];
  s *= scal[1];
  if (t < H) dgamma[t] = s;
  else if (t < 2 * H) dbeta[t - H] = s;
  else if (dalpha) dalpha[0] = s;
}

// ---- attention backward -----------------------------------------------------------------------------------------------
// D[b][head][t] = sum_d dO o O over the head's D channels; one thread per (frame, head)
__global__ void k_attn_delta(const __half* go, const __half* o, int F, int T, int heads, int D, float* delta) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F * heads) return;
  const int f = i / heads, hd = i - f * heads, b = f / T, t = f - b * T;
  const size_t off = static_cast<size_t>(f) * heads * D + hd * D;
  const __half2* g2 = reinterpret_cast<const __half2*>(go + off);
  const __half2* o2 = reinterpret_cast<const __half2*>(o + off);
  float s = 0.f;
  for (int d = 0; d < D / 2; ++d) {
    const float2 a = __half22float2(g2[d]), c = __half22float2(o2[d]);
    s += a.x * c.x + a.y * c.y;
  }
  delta[(static_cast<size_t>(b) * heads + hd) * T + t] = s;
}

struct AttnBwdArgs {
  const __half *q, *k, *v;     // [B][heads][T][D]; q scaled by D^-0.5
  const __half* go;            // dO [F][H]
  const float* lse;            // [B][heads][T]
  const float* delta;          // [B][heads][T]
  const uint8_t* pad;
  int T, heads;
  float qscale;
  __half* gqkv;                // [F][3H]: d of in_proj's output, columns q | k | v
};

template <int D>
constexpr int abwd_smem() { return 6 * 64 * D * 2 + 2 * 64 * 64 * 2 + 1024; }

// 64 rows x D of a [rows][stride] fp16 array from row0 (zero at or past T): D / 64 swizzled 64 x 64 tiles, 8 KB apart
template <int D>
__device__ __forceinline__ void load_tile(uint8_t* dst, const __half* src, size_t stride, int row0, int T) {
  const int tid = threadIdx.x;
#pragma unroll 1
  for (int it = 0; it < D / 16; ++it) {   // not unrolled: hoisted addresses would crowd out the accumulators
    const int i = tid + it * 128, r = i / (D / 8), cc = i % (D / 8), row = row0 + r;
    const bool ok = row < T;
    cp16(smem_u32(dst + (cc >> 3) * 8192) + sw128(r, cc & 7), src + static_cast<size_t>(ok ? row : 0) * stride + cc * 8, ok);
  }
}

__device__ __forceinline__ void put_half2(uint8_t* tile, int row, int col, float a, float b) {
  *reinterpret_cast<__half2*>(tile + sw128(row, col >> 3) + (col & 7) * 2) = __floats2half2_rn(a, b);
}

// s (+)= A . B^T over D for two [64][D] tiles in shared memory, m64n64
template <int D>
__device__ __forceinline__ void qk_product(float (&s)[32], const uint8_t* a, const uint8_t* b) {
#pragma unroll
  for (int c = 0; c < D / 64; ++c) {
    const uint64_t da = wg_desc(smem_u32(a + c * 8192)), db = wg_desc(smem_u32(b + c * 8192));
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) wgmma_f16<64>(s, da + 2 * k4, db + 2 * k4, 1);
  }
}

// One warpgroup per 64 keys of one head of one utterance; query blocks stream through two cp.async stages.
template <int D>
__global__ void __launch_bounds__(128) k_attn_bwd_kv(const AttnBwdArgs p) {
  constexpr int kT = 64 * D * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem;
  uint8_t* sV = sK + kT;
  uint8_t* sQ = sV + kT;          // 2 stages
  uint8_t* sG = sQ + 2 * kT;      // 2 stages
  uint8_t* sP = sG + 2 * kT;
  uint8_t* sS = sP + 8192;
  __shared__ float slse[2][64], sdel[2][64], kok[64];   // kok: 1 for a valid key of this block, else 0
  const int tid = threadIdx.x, n0 = blockIdx.x * 64, hd = blockIdx.y, b = blockIdx.z, T = p.T, H = p.heads * D;
  const size_t bh = static_cast<size_t>(b) * p.heads + hd;
  const __half* qg = p.q + bh * T * D;
  const __half* gg = p.go + static_cast<size_t>(b) * T * H + hd * D;

  load_tile<D>(sK, p.k + bh * T * D, D, n0, T);
  load_tile<D>(sV, p.v + bh * T * D, D, n0, T);
  auto load_q = [&](int i, int st) {
    load_tile<D>(sQ + st * kT, qg, D, i * 64, T);
    load_tile<D>(sG + st * kT, gg, H, i * 64, T);
    if (tid < 64) {
      const int row = i * 64 + tid;
      slse[st][tid] = row < T ? p.lse[bh * T + row] : INFINITY;
      sdel[st][tid] = row < T ? p.delta[bh * T + row] : 0.f;
    }
  };
  load_q(0, 0);
  cp_commit();
  if (tid < 64) kok[tid] = (n0 + tid < T && !p.pad[static_cast<size_t>(b) * T + n0 + tid]) ? 1.f : 0.f;

  float dk[D / 2], dv[D / 2];
#pragma unroll
  for (int e = 0; e < D / 2; ++e) dk[e] = dv[e] = 0.f;
  const int nblk = (T + 63) / 64;
#pragma unroll 1
  for (int i = 0; i < nblk; ++i) {
    const int st = i & 1;
    if (i + 1 < nblk) {
      load_q(i + 1, st ^ 1);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();

    // S^T, then P^T (fp16 tile), then dP^T and dS^T = P^T (dP^T - D) with P^T read back as stored: one 32-register
    // product live at a time next to the dK and dV accumulators
    float s[32];   // rows: keys, columns: queries
#pragma unroll
    for (int e = 0; e < 32; ++e) s[e] = 0.f;
    wg_fence();
    qk_product<D>(s, sK, sQ + st * kT);
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < 32; ++e) asm volatile("" : "+f"(s[e])::"memory");
#pragma unroll
    for (int e = 0; e < 32; e += 2) {
      const int row = acc_row(tid, e), col = acc_col(tid, e);
      const bool ok = kok[row] != 0.f;
      put_half2(sP, row, col, ok ? __expf(s[e] - slse[st][col]) : 0.f, ok ? __expf(s[e + 1] - slse[st][col + 1]) : 0.f);
    }
#pragma unroll
    for (int e = 0; e < 32; ++e) s[e] = 0.f;
    wg_fence();
    qk_product<D>(s, sV, sG + st * kT);
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < 32; ++e) asm volatile("" : "+f"(s[e])::"memory");
#pragma unroll
    for (int e = 0; e < 32; e += 2) {
      const int row = acc_row(tid, e), col = acc_col(tid, e);
      const float2 pt = __half22float2(*reinterpret_cast<const __half2*>(sP + sw128(row, col >> 3) + (col & 7) * 2));
      put_half2(sS, row, col, pt.x * (s[e] - sdel[st][col]), pt.y * (s[e + 1] - sdel[st][col + 1]));
    }
    fence_proxy_async_smem();
    __syncthreads();

    wg_fence();
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      wgmma_f16_bmn<D>(dv, wg_desc(smem_u32(sP)) + 2 * k4, wg_desc_mn(smem_u32(sG + st * kT) + k4 * 2048, 8192), 1);
      wgmma_f16_bmn<D>(dk, wg_desc(smem_u32(sS)) + 2 * k4, wg_desc_mn(smem_u32(sQ + st * kT) + k4 * 2048, 8192), 1);
    }
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < D / 2; ++e) asm volatile("" : "+f"(dk[e]), "+f"(dv[e])::"memory");
    __syncthreads();   // stage st, P and dS are free for the next block
  }

#pragma unroll
  for (int e = 0; e < D / 2; e += 2) {
    const int key = n0 + acc_row(tid, e);
    if (key >= T) continue;
    __half* dst = p.gqkv + (static_cast<size_t>(b) * T + key) * 3 * H + hd * D + acc_col(tid, e);
    *reinterpret_cast<__half2*>(dst + H) = __floats2half2_rn(dk[e], dk[e + 1]);
    *reinterpret_cast<__half2*>(dst + 2 * H) = __floats2half2_rn(dv[e], dv[e + 1]);
  }
}

// One warpgroup per 64 queries of one head of one utterance; key blocks stream through two cp.async stages.
template <int D>
__global__ void __launch_bounds__(128) k_attn_bwd_q(const AttnBwdArgs p) {
  constexpr int kT = 64 * D * 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sG = sQ + kT;
  uint8_t* sK = sG + kT;          // 2 stages
  uint8_t* sV = sK + 2 * kT;      // 2 stages
  uint8_t* sS = sV + 2 * kT;
  __shared__ float kok[2][64];    // 1 for a valid key of the stage, else 0
  const int tid = threadIdx.x, m0 = blockIdx.x * 64, hd = blockIdx.y, b = blockIdx.z, T = p.T, H = p.heads * D;
  const size_t bh = static_cast<size_t>(b) * p.heads + hd;
  const __half* kg = p.k + bh * T * D;
  const __half* vg = p.v + bh * T * D;

  load_tile<D>(sQ, p.q + bh * T * D, D, m0, T);
  load_tile<D>(sG, p.go + static_cast<size_t>(b) * T * H + hd * D, H, m0, T);
  auto load_kv = [&](int j, int st) {
    load_tile<D>(sK + st * kT, kg, D, j * 64, T);
    load_tile<D>(sV + st * kT, vg, D, j * 64, T);
    if (tid < 64) {
      const int key = j * 64 + tid;
      kok[st][tid] = (key < T && !p.pad[static_cast<size_t>(b) * T + key]) ? 1.f : 0.f;
    }
  };
  load_kv(0, 0);
  cp_commit();
  float lse[2], del[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int m = m0 + acc_row(tid, 2 * r);
    lse[r] = m < T ? p.lse[bh * T + m] : INFINITY;
    del[r] = m < T ? p.delta[bh * T + m] : 0.f;
  }

  float dq[D / 2];
#pragma unroll
  for (int e = 0; e < D / 2; ++e) dq[e] = 0.f;
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

    float s[32], dp[32];   // rows: queries, columns: keys
#pragma unroll
    for (int e = 0; e < 32; ++e) s[e] = dp[e] = 0.f;
    wg_fence();
    qk_product<D>(s, sQ, sK + st * kT);
    qk_product<D>(dp, sG, sV + st * kT);
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < 32; ++e) asm volatile("" : "+f"(s[e]), "+f"(dp[e])::"memory");

#pragma unroll
    for (int e = 0; e < 32; e += 2) {
      const int r = (e >> 1) & 1, row = acc_row(tid, e), col = acc_col(tid, e);
      float ds[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float pt = kok[st][col + i] != 0.f ? __expf(s[e + i] - lse[r]) : 0.f;
        ds[i] = pt * (dp[e + i] - del[r]);
      }
      put_half2(sS, row, col, ds[0], ds[1]);
    }
    fence_proxy_async_smem();
    __syncthreads();

    wg_fence();
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4)
      wgmma_f16_bmn<D>(dq, wg_desc(smem_u32(sS)) + 2 * k4, wg_desc_mn(smem_u32(sK + st * kT) + k4 * 2048, 8192), 1);
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < D / 2; ++e) asm volatile("" : "+f"(dq[e])::"memory");
    __syncthreads();
  }

#pragma unroll
  for (int e = 0; e < D / 2; e += 2) {
    const int m = m0 + acc_row(tid, e);
    if (m >= T) continue;
    *reinterpret_cast<__half2*>(p.gqkv + (static_cast<size_t>(b) * T + m) * 3 * H + hd * D + acc_col(tid, e)) =
        __floats2half2_rn(dq[e] * p.qscale, dq[e + 1] * p.qscale);
  }
}

// ---- tape -------------------------------------------------------------------------------------------------------------
using Tape = Fs2TrainTape;

// every region of the tape for (config, B, T), in order; bytes of the whole tape
size_t tape_carve(const dsx_fs2dec_config& c, int B, int T, uint8_t* base, Tape* t) {
  const size_t F = static_cast<size_t>(B) * T, H = c.hidden;
  const int L = c.layers;
  size_t n = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? base + n : nullptr;
    n += align256(bytes);
    return p;
  };
  Tape dummy;
  Tape& tp = t ? *t : dummy;
  tp.hdr = reinterpret_cast<TapeHdr*>(take(sizeof(TapeHdr)));
  tp.pad = take(F);
  tp.pos = reinterpret_cast<int*>(take(F * 4));
  tp.tr.xin.resize(2 * L + 1);
  for (auto& x : tp.tr.xin) x = reinterpret_cast<float*>(take(F * H * 4));
  for (auto* v : {&tp.tr.a1, &tp.tr.a2, &tp.tr.q, &tp.tr.k, &tp.tr.v, &tp.tr.o, &tp.tr.z, &tp.tr.hd}) v->resize(L);
  tp.tr.lse.resize(L);
  for (int l = 0; l < L; ++l) {
    for (auto* v : {&tp.tr.a1, &tp.tr.a2, &tp.tr.q, &tp.tr.k, &tp.tr.v, &tp.tr.o})
      (*v)[l] = reinterpret_cast<__half*>(take(F * H * 2));
    tp.tr.lse[l] = reinterpret_cast<float*>(take(F * c.heads * 4));
    tp.tr.z[l] = reinterpret_cast<__half*>(take(F * 4 * H * 2));
    tp.tr.hd[l] = reinterpret_cast<__half*>(take(F * 4 * H * 2));
  }
  return n;
}

}  // namespace
}  // namespace dsx

struct dsx_fs2dec_train {
  struct Packs {
    dsx::ConvGemm in_t, out_t, ffn1_t, ffn2_t;   // the transposed packs of the data-gradient GEMMs
  };
  int device = 0;
  dsx_fs2dec_config cfg{};
  dsx_fs2dec* dec = nullptr;   // the forward's packs (refilled by every forward) and kernels
  std::vector<Packs> layers;
  dsx::DevAllocs mem;
};

namespace dsx {
namespace {

int gemm_alloc(DevAllocs& mem, ConvGemm& g, int cin, int n, int taps) {
  g.cin = cin;
  g.n = n;
  g.taps = taps;
  g.nt = kNT;
  g.ntiles = (n + kNT - 1) / kNT;
  g.kc = (taps * cin + 63) / 64;
  DSX_TRY(mem.alloc(&g.w, static_cast<size_t>(g.ntiles) * g.kc * g.nt * 64 * sizeof(__half)));
  return mem.alloc(&g.b, static_cast<size_t>(g.ntiles) * g.nt * sizeof(float));
}

// W^T of a Linear or Conv1d weight [cout][cin][k] packed as the GEMM g (g.cin = cout, g.n = cin)
int pack_t(const ConvGemm& g, const float* w, int k, cudaStream_t s) {
  const size_t nw = static_cast<size_t>(g.ntiles) * g.kc * g.nt * 64;
  k_pack_conv<<<static_cast<unsigned>(std::min<size_t>((nw + 255) / 256, 4096)), 256, 0, s>>>(
      g, PackArgs{w, nullptr, nullptr, g.cin, g.n, g.n, k, 1, 1});
  return launch_check("k_pack_conv");
}

int run_bwd_gemm(BwdGemmArgs a, const ConvGemm& g, int B, int T, cudaStream_t s) {
  a.g = g;
  a.T = T;
  const dim3 grid((T + kConvRows - 1) / kConvRows, B, g.ntiles);
  k_f2b_gemm<kNT><<<grid, 256, conv_smem<kNT>(), s>>>(a);
  return launch_check("k_f2b_gemm");
}

int tap0_of(const dsx_fs2dec_config& c) { return c.padding ? -(c.kernel - 1) : -(c.kernel / 2); }

// the backward's workspace: scalars, G, gA (fp32 [F][H]), gY (fp16 [F][H]), gC (fp16 [F][4H]), dO (fp16 [F][H]),
// d in_proj output (fp16 [F][3H]), D of the attention, LayerNorm partials, weight-gradient partials
constexpr int kBwdRegions = 10;
void bwd_sizes(const dsx_fs2dec_config& c, int B, int T, int device, size_t (&sz)[kBwdRegions]) {
  const size_t F = static_cast<size_t>(B) * T, H = c.hidden;
  // (m tiles, n tiles) of the weight-gradient GEMMs: ffn_2, ffn_1 (4 taps a launch), out_proj, in_proj
  const int h = c.hidden;
  const size_t part = wgrad_part_floats(static_cast<int>(F),
                                        {{h / 64, 4 * h / 256}, {4 * h / 64, std::min(c.kernel, 4)}, {h / 64, 1},
                                         {3 * h / 64, 1}},
                                        device);
  const size_t v[kBwdRegions] = {256,       F * H * 4, F * H * 4,
                                 F * H * 2, F * 4 * H * 2, F * H * 2,
                                 F * 3 * H * 2, F * c.heads * 4, static_cast<size_t>(kLnBlocks) * (2 * H + 1) * 4,
                                 part * 4};
  for (int i = 0; i < kBwdRegions; ++i) sz[i] = v[i];
}

size_t ws_bytes(const dsx_fs2dec_train* h, int B, int T) {
  size_t sz[kBwdRegions], n = 0;
  bwd_sizes(h->cfg, B, T, h->device, sz);
  for (size_t z : sz) n += align256(z);
  return std::max(n, fs2_workspace_bytes(h->dec, B, T));
}

int check_geom(const dsx_fs2dec_train* h, int B, int T) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(B <= 65535, DSX_E_INVALID, "B = %d utterances per call is above the 65535 the launch grid holds", B);
  const long long Tp = (T + kConvRows - 1) / kConvRows * kConvRows;
  DSX_CHECK(static_cast<long long>(B) * Tp * 4 * h->cfg.hidden < (1ll << 31), DSX_E_INVALID,
            "B * T = %lld frames is too large", static_cast<long long>(B) * T);
  return DSX_OK;
}

template <int D>
int abwd_opt_in() {
  DSX_CUDA(cudaFuncSetAttribute(k_attn_bwd_kv<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, abwd_smem<D>()));
  DSX_CUDA(cudaFuncSetAttribute(k_attn_bwd_q<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, abwd_smem<D>()));
  return DSX_OK;
}

}  // namespace
}  // namespace dsx

namespace dsx {

dsx_fs2dec* fs2t_stack(dsx_fs2dec_train* h) { return h->dec; }

size_t fs2t_tape_carve(const dsx_fs2dec_train* h, int B, int T, void* base, Fs2TrainTape* t) {
  return tape_carve(h->cfg, B, T, static_cast<uint8_t*>(base), t);
}

int fs2t_check_params(const dsx_fs2dec_params* p, int L, int alpha, const char* what) {
  DSX_CHECK(p, DSX_E_INVALID, "%s is NULL", what);
  DSX_CHECK(p->ln1_w && p->ln1_b && p->in_proj_w && p->out_proj_w && p->ln2_w && p->ln2_b && p->ffn1_w && p->ffn1_b &&
                p->ffn2_w && p->ffn2_b && p->ln_w && p->ln_b && (p->pos_embed_alpha || !alpha),
            DSX_E_INVALID, "a pointer of %s is NULL", what);
  for (int l = 0; l < L; ++l)
    DSX_CHECK(p->ln1_w[l] && p->ln1_b[l] && p->in_proj_w[l] && p->out_proj_w[l] && p->ln2_w[l] && p->ln2_b[l] &&
                  p->ffn1_w[l] && p->ffn1_b[l] && p->ffn2_w[l] && p->ffn2_b[l],
              DSX_E_INVALID, "a pointer of layer %d of %s is NULL", l, what);
  return DSX_OK;
}

int fs2t_begin(dsx_fs2dec_train* h, const dsx_fs2dec_params* w, int B, int T, float p_drop, uint64_t seed, void* tape,
               cudaStream_t s, Fs2TrainTape* tp) {
  const dsx_fs2dec_config& c = h->cfg;
  // round-to-nearest fp16 packs of this step's weights, and the transposed packs of the backward
  DSX_TRY(fs2_train_pack(h->dec, w, s));
  for (int l = 0; l < c.layers; ++l) {
    const dsx_fs2dec_train::Packs& pk = h->layers[l];
    DSX_TRY(pack_t(pk.in_t, w->in_proj_w[l], 1, s));
    DSX_TRY(pack_t(pk.out_t, w->out_proj_w[l], 1, s));
    DSX_TRY(pack_t(pk.ffn1_t, w->ffn1_w[l], c.kernel, s));
    DSX_TRY(pack_t(pk.ffn2_t, w->ffn2_w[l], 1, s));
  }
  tape_carve(c, B, T, static_cast<uint8_t*>(tape), tp);
  tp->tr.seed = seed;
  tp->tr.p = p_drop;
  k_tape_hdr<<<1, 1, 0, s>>>(tp->hdr, seed, p_drop, B, T);
  return launch_check("k_tape_hdr");
}

int fs2t_backward(dsx_fs2dec_train* h, const dsx_fs2dec_params* w, const void* tape, const float* d_out,
                  const dsx_fs2dec_params* grads, float* d_x, float* d_alpha, int B, int T, void* workspace,
                  cudaStream_t s) {
  const dsx_fs2dec_config& c = h->cfg;
  const int H = c.hidden, L = c.layers, heads = c.heads, D = H / heads, k = c.kernel, F = B * T;
  const int mtiles = (T + kConvRows - 1) / kConvRows;
  Tape tp;
  tape_carve(c, B, T, static_cast<uint8_t*>(const_cast<void*>(tape)), &tp);
  const Fs2Train& tr = tp.tr;

  size_t sizes[kBwdRegions];
  bwd_sizes(c, B, T, h->device, sizes);
  Bump bump{static_cast<uint8_t*>(workspace)};
  unsigned* amax = bump.take<unsigned>(sizes[0]);
  float* scal = reinterpret_cast<float*>(amax + 4);
  float* G = bump.take<float>(sizes[1]);
  float* GA = bump.take<float>(sizes[2]);
  __half* GY = bump.take<__half>(sizes[3]);
  __half* GC = bump.take<__half>(sizes[4]);
  __half* GO = bump.take<__half>(sizes[5]);
  __half* GQKV = bump.take<__half>(sizes[6]);
  float* DELTA = bump.take<float>(sizes[7]);
  float* LNP = bump.take<float>(sizes[8]);
  float* PART = bump.take<float>(sizes[9]);
  auto gp = [](const float* p) { return const_cast<float*>(p); };

  DSX_TRY(run_scale(d_out, static_cast<size_t>(F) * H, amax, scal, tp.hdr, B, T, s));

  // LayerNorm backward into G, then its affine gradients
  auto ln = [&](const float* gin, int from_dout, const float* x, const float* gamma, int accumulate, __half* o16,
                int site, int entry, float* dgamma, float* dbeta, float* dalpha) -> int {
    LnArgs a{};
    a.gin = gin;
    a.from_dout = from_dout;
    a.x = x;
    a.gamma = gamma;
    a.pad = tp.pad;
    a.G = G;
    a.accumulate = accumulate;
    a.o16 = o16;
    a.entry = entry;
    a.dx = d_x;
    a.pos = dalpha ? tp.pos : nullptr;
    a.neg_emb = pos_neg_emb(H);
    a.hdr = tp.hdr;
    a.site = site;
    a.part = LNP;
    a.scal = scal;
    a.F = F;
    a.H = H;
    k_f2b_ln<<<kLnBlocks, 256, 0, s>>>(a);
    DSX_TRY(launch_check("k_f2b_ln"));
    k_f2b_ln_reduce<<<(2 * H + 1 + 255) / 256, 256, 0, s>>>(LNP, kLnBlocks, H, scal, dgamma, dbeta, dalpha);
    return launch_check("k_f2b_ln_reduce");
  };
  // weight gradient sum_f A[f][m] B_jj[f + shift_jj][c] of ntiles B tiles into o
  auto wgrad = [&](const __half* A, int lda, int am, WgradArgs t, int ntiles, const WgradDst& o) -> int {
    t.a = A;
    t.lda = lda;
    t.am = am;
    t.F = F;
    t.T = T;
    return run_wgrad(t, ntiles, o, PART, scal, h->device, s);
  };
  // tile jj to dst[m * ms + c * cs + jj * js]
  auto rows = [](float* dst, int ms, int cs, int js, float* db) {
    WgradDst o{};
    for (int jj = 0; jj < 4; ++jj) {
      o.dst[jj] = dst + jj * js;
      o.ms[jj] = ms;
      o.cs[jj] = cs;
    }
    o.db = db;
    return o;
  };
  auto single = [](const __half* b, int ldb, int bn) {
    WgradArgs t{};
    t.b[0] = b;
    t.ldb[0] = ldb;
    t.bn[0] = bn;
    return t;
  };

  // final LayerNorm * !pad (tts_modules.py:300-301)
  DSX_TRY(ln(d_out, 1, tr.xin[2 * L], w->ln_w, 0, GY, 3 + 3 * (L - 1), 0, gp(grads->ln_w), gp(grads->ln_b),
             nullptr));
  for (int i = L - 1; i >= 0; --i) {
    const dsx_fs2dec_train::Packs& pk = h->layers[i];
    // FFN block: x = (x + dropout(ffn_2(dropout(act(ffn_1(LN2(x)) * k^-0.5))))) * !pad
    BwdGemmArgs a{};
    a.mode = B_GC;
    a.x = GY;
    a.o16 = GC;
    a.z = tr.z[i];
    a.hdr = tp.hdr;
    a.site = 2 + 3 * i;
    a.relu = c.act;
    a.kscale = static_cast<float>(pow(static_cast<double>(k), -0.5));
    DSX_TRY(run_bwd_gemm(a, pk.ffn2_t, B, T, s));
    {
      WgradArgs t{};
      const int nt = 4 * H / 256;
      for (int j = 0; j < nt; ++j) {
        t.b[j] = tr.hd[i] + j * 256;
        t.ldb[j] = 4 * H;
        t.bn[j] = 256;
      }
      DSX_TRY(wgrad(GY, H, H, t, nt, rows(gp(grads->ffn2_w[i]), 4 * H, 1, 256, gp(grads->ffn2_b[i]))));
    }
    a = BwdGemmArgs{};
    a.mode = B_F32;
    a.x = GC;
    a.o32 = GA;
    DSX_TRY(run_bwd_gemm(a, pk.ffn1_t, B, T, s));
    for (int j0 = 0; j0 < k; j0 += 4) {   // ffn_1's weight [4H][H][k]: taps j0 .. j0 + 3, each a shifted copy of LN2
      WgradArgs t{};
      const int nt = std::min(4, k - j0);
      for (int jj = 0; jj < nt; ++jj) {
        t.b[jj] = tr.a2[i];
        t.ldb[jj] = H;
        t.bn[jj] = H;
        t.shift[jj] = tap0_of(c) + j0 + jj;
      }
      DSX_TRY(wgrad(GC, 4 * H, 4 * H, t, nt,
                    rows(gp(grads->ffn1_w[i]) + j0, H * k, k, 1, j0 == 0 ? gp(grads->ffn1_b[i]) : nullptr)));
    }
    DSX_TRY(ln(GA, 0, tr.xin[2 * i + 1], w->ln2_w[i], 1, GY, 1 + 3 * i, 0, gp(grads->ln2_w[i]), gp(grads->ln2_b[i]),
               nullptr));
    // self-attention block: x = (x + dropout(out_proj(MHA(LN1(x))))) * !pad
    a = BwdGemmArgs{};
    a.mode = B_F16;
    a.x = GY;
    a.o16 = GO;
    DSX_TRY(run_bwd_gemm(a, pk.out_t, B, T, s));
    DSX_TRY(wgrad(GY, H, H, single(tr.o[i], H, H), 1, rows(gp(grads->out_proj_w[i]), H, 1, 0, nullptr)));
    k_attn_delta<<<(F * heads + 255) / 256, 256, 0, s>>>(GO, tr.o[i], F, T, heads, D, DELTA);
    DSX_TRY(launch_check("k_attn_delta"));
    AttnBwdArgs ab{};
    ab.q = tr.q[i];
    ab.k = tr.k[i];
    ab.v = tr.v[i];
    ab.go = GO;
    ab.lse = tr.lse[i];
    ab.delta = DELTA;
    ab.pad = tp.pad;
    ab.T = T;
    ab.heads = heads;
    ab.qscale = static_cast<float>(sqrt(1.0 / D));
    ab.gqkv = GQKV;
    const dim3 agrid(mtiles, heads, B);
    if (D == 64) {
      k_attn_bwd_kv<64><<<agrid, 128, abwd_smem<64>(), s>>>(ab);
      DSX_TRY(launch_check("k_attn_bwd_kv"));
      k_attn_bwd_q<64><<<agrid, 128, abwd_smem<64>(), s>>>(ab);
    } else {
      k_attn_bwd_kv<128><<<agrid, 128, abwd_smem<128>(), s>>>(ab);
      DSX_TRY(launch_check("k_attn_bwd_kv"));
      k_attn_bwd_q<128><<<agrid, 128, abwd_smem<128>(), s>>>(ab);
    }
    DSX_TRY(launch_check("k_attn_bwd_q"));
    a = BwdGemmArgs{};
    a.mode = B_F32;
    a.x = GQKV;
    a.o32 = GA;
    DSX_TRY(run_bwd_gemm(a, pk.in_t, B, T, s));
    DSX_TRY(wgrad(GQKV, 3 * H, 3 * H, single(tr.a1[i], H, H), 1, rows(gp(grads->in_proj_w[i]), H, 1, 0, nullptr)));
    // LN1, then the operand of the layer below, or the entry: x + alpha * table[pos] -> dropout -> * !pad
    DSX_TRY(ln(GA, 0, tr.xin[2 * i], w->ln1_w[i], 1, i > 0 ? GY : nullptr, i > 0 ? 3 * i : 0, i == 0,
               gp(grads->ln1_w[i]), gp(grads->ln1_b[i]), i == 0 ? d_alpha : nullptr));
  }
  return DSX_OK;
}

}  // namespace dsx

using namespace dsx;

extern "C" {

int dsx_fs2dec_train_create(int device, const dsx_fs2dec_config* cfg, dsx_fs2dec_train** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  dsx_fs2dec* dec = nullptr;
  DSX_TRY(dsx_fs2dec_create(device, cfg, &dec));   // validates the configuration and selects the device
  dsx_fs2dec_train* h = new dsx_fs2dec_train();
  h->device = device;
  h->cfg = *cfg;
  h->dec = dec;
  auto fail = [&](int rc) {
    dsx_fs2dec_train_destroy(h);
    return rc;
  };
  int rc = DSX_OK;
  if ((rc = fs2_train_alloc(dec))) return fail(rc);
  if ((rc = []() -> int {
         DSX_CUDA(cudaFuncSetAttribute(k_f2b_gemm<kNT>, cudaFuncAttributeMaxDynamicSharedMemorySize, conv_smem<kNT>()));
         DSX_CUDA(cudaFuncSetAttribute(k_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmem));
         DSX_TRY(abwd_opt_in<64>());
         return abwd_opt_in<128>();
       }()))
    return fail(rc);
  const int H = cfg->hidden, k = cfg->kernel;
  h->layers.resize(cfg->layers);
  for (auto& l : h->layers) {
    if ((rc = gemm_alloc(h->mem, l.in_t, 3 * H, H, 1)) || (rc = gemm_alloc(h->mem, l.out_t, H, H, 1)) ||
        (rc = gemm_alloc(h->mem, l.ffn1_t, 4 * H, H, k)) || (rc = gemm_alloc(h->mem, l.ffn2_t, H, 4 * H, 1)))
      return fail(rc);
    l.ffn1_t.tap0 = -tap0_of(*cfg);   // gA[t] = sum_j W_j^T gC[t - tap0 - j]
    l.ffn1_t.tstep = -1;
  }
  *out = h;
  return DSX_OK;
}

void dsx_fs2dec_train_destroy(dsx_fs2dec_train* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  h->mem.free_all();
  dsx_fs2dec_destroy(h->dec);
  delete h;
}

int dsx_fs2dec_train_tape_bytes(dsx_fs2dec_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  DSX_TRY(check_geom(h, B, T));
  *out = tape_carve(h->cfg, B, T, nullptr, nullptr);
  return DSX_OK;
}

int dsx_fs2dec_train_workspace_bytes(dsx_fs2dec_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  DSX_TRY(check_geom(h, B, T));
  *out = ws_bytes(h, B, T);
  return DSX_OK;
}

int dsx_fs2dec_train_forward(dsx_fs2dec_train* h, const dsx_fs2dec_params* w, const float* x, dsx_strides xs, int B,
                             int T, float p_drop, uint64_t seed, void* tape, size_t tape_bytes, void* workspace,
                             size_t workspace_bytes, float* out, void* stream) {
  DSX_TRY(check_geom(h, B, T));
  const dsx_fs2dec_config& c = h->cfg;
  DSX_TRY(fs2t_check_params(w, c.layers, 1, "the parameters"));
  DSX_CHECK(x && tape && workspace && out, DSX_E_INVALID, "x, tape, workspace and out must not be NULL");
  DSX_CHECK(p_drop >= 0.f && p_drop < 1.f, DSX_E_INVALID, "dropout p = %g is outside [0, 1)", static_cast<double>(p_drop));
  const size_t need = tape_carve(c, B, T, nullptr, nullptr);
  DSX_CHECK(tape_bytes >= need, DSX_E_INVALID, "tape of %zu bytes is below the %zu this (B, T) needs", tape_bytes, need);
  const size_t wneed = ws_bytes(h, B, T);
  DSX_CHECK(workspace_bytes >= wneed, DSX_E_INVALID, "workspace of %zu bytes is below the %zu this (B, T) needs",
            workspace_bytes, wneed);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  Tape tp;
  DSX_TRY(fs2t_begin(h, w, B, T, p_drop, seed, tape, s, &tp));
  Fs2Bufs fb = fs2_carve(h->dec, workspace, B, T);
  fb.PAD = tp.pad;
  fb.POS = tp.pos;
  return fs2_forward_run(h->dec, x, xs, B, T, fb, out, s, &tp.tr);
}

int dsx_fs2dec_train_backward(dsx_fs2dec_train* h, const dsx_fs2dec_params* w, const void* tape, const float* d_out,
                              const dsx_fs2dec_params* grads, float* d_x, int B, int T, void* workspace,
                              size_t workspace_bytes, void* stream) {
  DSX_TRY(check_geom(h, B, T));
  const dsx_fs2dec_config& c = h->cfg;
  DSX_TRY(fs2t_check_params(w, c.layers, 1, "the parameters"));
  DSX_TRY(fs2t_check_params(grads, c.layers, 1, "the gradients"));
  DSX_CHECK(tape && d_out && workspace, DSX_E_INVALID, "tape, d_out and workspace must not be NULL");
  const size_t wneed = ws_bytes(h, B, T);
  DSX_CHECK(workspace_bytes >= wneed, DSX_E_INVALID, "workspace of %zu bytes is below the %zu this (B, T) needs",
            workspace_bytes, wneed);
  DSX_CUDA(cudaSetDevice(h->device));
  return fs2t_backward(h, w, tape, d_out, grads, d_x, const_cast<float*>(grads->pos_embed_alpha), B, T, workspace,
                       static_cast<cudaStream_t>(stream));
}

int dsx_fs2dec_train_masks(dsx_fs2dec_train* h, uint64_t seed, float p_drop, int B, int T, uint8_t* const* out,
                           void* stream) {
  DSX_TRY(check_geom(h, B, T));
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  DSX_CHECK(p_drop >= 0.f && p_drop < 1.f, DSX_E_INVALID, "dropout p = %g is outside [0, 1)", static_cast<double>(p_drop));
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t F = static_cast<size_t>(B) * T;
  for (int site = 0; site < 1 + 3 * h->cfg.layers; ++site) {
    DSX_CHECK(out[site], DSX_E_INVALID, "mask %d is NULL", site);
    const int n = (site > 0 && site % 3 == 2) ? 4 * h->cfg.hidden : h->cfg.hidden;
    k_drop_masks<<<static_cast<unsigned>(std::min<size_t>((F * n + 255) / 256, 4096)), 256, 0, s>>>(
        make_drop(seed, p_drop, site), F, n, out[site]);
    DSX_TRY(launch_check("k_drop_masks"));
  }
  return DSX_OK;
}

}  // extern "C"
