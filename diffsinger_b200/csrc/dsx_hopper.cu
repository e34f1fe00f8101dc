// Tensor-core path of the dsx sampler for Hopper (sm_90a): warpgroup MMA (wgmma.mma_async, fp16 operands from shared
// memory, fp32 accumulators in registers).  Two kernels:
//   k_hp_step<NWG>   residual layers [l0, l1) of one DiffNet evaluation (usr/diff/net.py:58-78) and, optionally, what
//                    follows them in a diffusion step: skip / output projections, the DDPM or PNDM update and the next
//                    evaluation's input projection (net.py:115-130, shallow_diffusion_tts.py:134-199).  Persistent and
//                    cooperative: every CTA walks over the frame tiles of a layer, a grid-wide barrier separates layers
//                    (layer l+1 of a tile reads the conv input of its neighbour tiles).
//   k_hp_condproj    conditioner projection of every layer, once per call (it does not depend on the diffusion step).
//
// Per residual layer and tile of 64 frames (one warpgroup; a CTA has NWG warpgroups = 64 * NWG frames):
//   GEMM1  D1[64 x 512] = [y(t-d) | y(t) | y(t+d)] (K = 768) . W1^T, as two N = 256 chunks [128 gate | 128 filter]
//   epi1   z = sigmoid(D1 gate + CP) * tanh(D1 filter + CP) -> fp16 (hi [, lo]) in shared memory
//   GEMM2  D2[64 x 512] = z (K = 256) . W2^T, as two N = 256 halves (residual | skip)
//   epi2   x <- (x + D2[:, :256] + b) / sqrt2 ; y_next = fp16 (split) of (x + d_{l+1}) ; skip += D2[:, 256:] + b
// CP = conditioner_projection_l(cond) + biases (fp32, [L][frames][512]) comes from k_hp_condproj.  x, skip and y live in
// global memory (frames-major [B][Tp][256], Tp = T rounded up to 128); the dilated taps read y at frame offsets -d, 0, +d
// and the loads zero-fill frames outside [0, T), which is the conv's zero padding applied after the FiLM add.
//
// Operands reach shared memory by cp.async in the 128-byte-swizzled K-major layout wgmma reads (dsx_ptx.cuh), double
// buffered: one stage = a 256-row x 64-k weight tile (32 KB, shared by the warpgroups) + one 64 x 64 activation block per
// warpgroup.  Each warpgroup's rows go through the same instruction sequence whatever NWG is, so 64- and 128-frame CTAs
// give bit-identical results.
//
// Precision (MMA passes P per k-block): P = 1 fp16 operands; P = 2 adds a W_lo pass (weights as hi+lo fp16 pairs);
// P = 3 accumulates A_hi*W_hi + A_hi*W_lo + A_lo*W_hi (~2^-22 relative).  The conditioner projection is always 3-pass.
#include <cooperative_groups.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "dsx_internal.h"
#include "dsx_ptx.cuh"
#include "dsx_rng.cuh"

namespace cg = cooperative_groups;

namespace dsx {

constexpr int kC = 256;                    // residual / conditioner channels supported by this path
constexpr int kRowsPerLayer = 80 * 256;    // wpack rows (of 64 fp16) per layer: 64 W1 tiles + 16 W2 tiles of 256 rows
constexpr int kSrRowsPerLayer = 32 * 256;  // rows per layer of one stochastically rounded weight set: 24 W1 + 8 W2 tiles
constexpr int kWBytes = 256 * 128;         // one weight tile: 256 rows x 64 fp16
constexpr int kABytes = 64 * 128;          // one activation block: 64 rows x 64 fp16
constexpr int kZBytes = 2 * 4 * kABytes;   // per warpgroup: z / h / x_in operand, [plane hi, lo][4 k-blocks]

template <int NWG>
struct StepCfg {
  static constexpr int THREADS = NWG * 128;
  static constexpr int STAGE = kWBytes + NWG * kABytes;
  static constexpr int SMEM = 1024 + 2 * STAGE + NWG * kZBytes;
  static_assert(SMEM <= 232448, "shared memory budget");
};
constexpr int kCondSmem = 1024 + 2 * StepCfg<2>::STAGE;

struct HpParams {
  const __half* w;           // residual-layer weights: wpack (hi / lo planes) or one stochastically rounded set
  int w_sr;                  // 1: w is a set of the fp16s pack (layout of k_pack_wsr)
  int P;                     // MMA passes of the residual layers (1..3)
  int HP;                    // MMA passes of the head projections (1 or 3)
  int ylo;                   // write the lo plane of y (read by P = 3 layers)
  int fast_gate;
  const __half* whead;       // [32 tiles][128 rows][64]
  float* X;                  // [B][Tp][256] residual stream
  float* SKIP;               // [B][Tp][256]
  __half* Y;                 // [2 buffers][2 planes][plane]: layer l reads buffer l & 1, writes buffer (l + 1) & 1
  __half* S16;               // [2 planes][plane]: skip_sum / sqrt(L), operand of the head
  const __half* CONDH;       // [2 planes][plane]
  size_t plane;              // B * Tp * 256
  float* CP;                 // [L][B * Tp][512]
  const float* b1p;          // [L][2 chunks][256]
  const float* b2;           // [L][512]
  const float* dtab;         // FiLM table row of this evaluation: [L][256], utterance b at + b * d_row_stride
  int d_row_stride;
  int T, Tp, B, units;       // units: tiles of 64 * NWG frames
  int l0, l1, L, cycle;
  float inv_sqrt_l;
  // what follows the layers (TC_* flags; 0: nothing)
  int head_flags;
  float* x;                  // mel state, addressed through xs
  dsx_strides xs;
  float* eps;
  const float* noise;
  unsigned long long seed, offset;
  int b_off;
  DdpmCoef c;
  PlmsFuse pl;
  const float* bs;           // skip_projection.bias
  const float* bf;           // output_projection.bias
  const float* bin;          // input_projection.bias
  const float* d0;           // FiLM vector of layer 0 of the evaluation being prepared (TC_INPROJ)
  int d0_row_stride;
  int M;
};

// ------------------------------------------------------------------------------------------
// operand loads and the GEMM loop
// ------------------------------------------------------------------------------------------
// 256 (NROWS) weight rows -> swizzled tile; row r comes from src0 (r < 128) or src1 (r >= 128, may be src0 + 128 rows)
template <int NT>
__device__ __forceinline__ void load_w(uint8_t* dst, const __half* src0, const __half* src1, int nrows, int tid) {
  const uint32_t d = smem_u32(dst);
  for (int i = tid; i < nrows * 8; i += NT) {
    const int r = i >> 3, c = i & 7;
    const __half* src = (r < 128 ? src0 + static_cast<size_t>(r) * 64 : src1 + static_cast<size_t>(r - 128) * 64) + c * 8;
    cp16(d + sw128(r, c), src, true);
  }
}
// 64 frames [t0, t0 + 64) of utterance b, channels [ch0, ch0 + 64) of a frames-major [B][Tp][256] fp16 plane; frames
// outside [0, T) read as zero.  Called by the 128 threads of one warpgroup.
__device__ __forceinline__ void load_a(uint8_t* dst, const __half* src, int b, int t0, int ch0, int T, int Tp, int wtid) {
  const uint32_t d = smem_u32(dst);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int i = wtid + k * 128;
    const int r = i >> 3, c = i & 7, t = t0 + r;
    const bool valid = t >= 0 && t < T;
    cp16(d + sw128(r, c), src + (static_cast<size_t>(b) * Tp + (valid ? t : 0)) * kC + ch0 + c * 8, valid);
  }
}

template <int N>
__device__ __forceinline__ void fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// c0 (weight rows 0..127) [and c1 (rows 128..255) when NH == 2] = sum over nst stages of A_s . W_s^T.  load(s, buf) issues
// the cp.async copies of stage s into buf; adesc(s, buf) is the descriptor of this warpgroup's A block of stage s.
// Every thread of the CTA runs it (the weight tile is shared); it ends with the accumulators complete and the stage
// buffers free.
template <int NH, class Load, class ADesc>
__device__ __forceinline__ void gemm(float (&c0)[64], float (&c1)[64], int nst, Load load, ADesc adesc, uint8_t* buf0,
                                     uint8_t* buf1) {
  load(0, buf0);
  cp_commit();
  fence_acc(c0);
  if (NH == 2) fence_acc(c1);
#pragma unroll 1
  for (int s = 0; s < nst; ++s) {
    uint8_t* cur = (s & 1) ? buf1 : buf0;
    if (s + 1 < nst) {
      load(s + 1, (s & 1) ? buf0 : buf1);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    const uint64_t a = adesc(s, cur);
    const uint64_t w = wg_desc(smem_u32(cur));
    wg_fence();
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      const int acc = (s > 0 || k4 > 0) ? 1 : 0;
      wgmma_n128(c0, a + 2 * k4, w + 2 * k4, acc);
      if (NH == 2) wgmma_n128(c1, a + 2 * k4, w + (16384 >> 4) + 2 * k4, acc);
    }
    wg_commit();
    wg_wait0();
    fence_acc(c0);
    if (NH == 2) fence_acc(c1);
    __syncthreads();
  }
}

// accumulator element e of thread (warp w of the warpgroup, lane): row and column inside the 64 x 128 block
__device__ __forceinline__ int acc_row(int wtid, int e) { return ((wtid >> 5) << 4) + ((wtid & 31) >> 2) + ((e & 2) ? 8 : 0); }
__device__ __forceinline__ int acc_col(int wtid, int e) { return ((e >> 2) << 3) + ((wtid & 3) << 1) + (e & 1); }
// byte offset of (row r, channel k) in a [4 k-blocks] K-major swizzled operand
__device__ __forceinline__ uint32_t opnd_off(int r, int k) {
  return static_cast<uint32_t>((k >> 6) * kABytes) + sw128(r, (k & 63) >> 3) + (k & 7) * 2;
}

__device__ __forceinline__ const __half* w1_tile(const HpParams& p, int l, int plane, int h, int kb) {
  if (p.w_sr) return p.w + (static_cast<size_t>(l) * kSrRowsPerLayer + (h * 12 + kb) * 256) * 64;
  return p.w + (static_cast<size_t>(l) * kRowsPerLayer + ((plane * 2 + h) * 16 + kb) * 256) * 64;
}
__device__ __forceinline__ const __half* w2_tile(const HpParams& p, int l, int plane, int q, int kb) {
  if (p.w_sr) return p.w + (static_cast<size_t>(l) * kSrRowsPerLayer + (24 + q * 4 + kb) * 256) * 64;
  return p.w + (static_cast<size_t>(l) * kRowsPerLayer + (64 + (plane * 2 + q) * 4 + kb) * 256) * 64;
}
__device__ __forceinline__ const __half* whead_tile(const HpParams& p, int idx) {
  return p.whead + static_cast<size_t>(idx) * 128 * 64;
}
// pass ps of a P-pass k-block: {W plane, A plane}
__device__ __forceinline__ int pass_wplane(int ps) { return ps == 1 ? 1 : 0; }
__device__ __forceinline__ int pass_aplane(int ps) { return ps == 2 ? 1 : 0; }

// ------------------------------------------------------------------------------------------
// one residual layer of one tile
// ------------------------------------------------------------------------------------------
template <int NWG>
__device__ __forceinline__ void layer_tile(const HpParams& p, int l, int u, uint8_t* buf0, uint8_t* buf1, uint8_t* zb) {
  constexpr int NT = NWG * 128;
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  const int frame0 = u * 64 * NWG;
  const int b = frame0 / p.Tp, t0 = frame0 % p.Tp + wg * 64;
  const size_t fbase = static_cast<size_t>(b) * p.Tp + t0;     // global frame of row 0 of this warpgroup
  const int d = 1 << (l % p.cycle);
  const int P = p.P;
  const __half* Yin = p.Y + static_cast<size_t>(l & 1) * 2 * p.plane;
  const size_t NF = p.plane / kC;
  float c0[64], c1[64];

  // ---- GEMM1 + gate, chunk by chunk ----
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    auto load = [&](int s, uint8_t* bf) {
      const int kb = s / P, ps = s % P;
      const __half* wt = w1_tile(p, l, pass_wplane(ps), h, kb);
      load_w<NT>(bf, wt, wt + 128 * 64, 256, tid);
      const int tap = kb >> 2, cb = kb & 3;
      load_a(bf + kWBytes + wg * kABytes, Yin + pass_aplane(ps) * p.plane, b, t0 + (tap - 1) * d, cb * 64, p.T, p.Tp, wtid);
    };
    auto adesc = [&](int, uint8_t* bf) { return wg_desc(smem_u32(bf + kWBytes + wg * kABytes)); };
    gemm<2>(c0, c1, 12 * P, load, adesc, buf0, buf1);
    const float* cp = p.CP + (static_cast<size_t>(l) * NF + fbase) * 512 + h * 256;
#pragma unroll
    for (int e = 0; e < 64; e += 2) {
      const int r = acc_row(wtid, e), n = acc_col(wtid, e);
      const float2 cgv = *reinterpret_cast<const float2*>(cp + static_cast<size_t>(r) * 512 + n);
      const float2 cfv = *reinterpret_cast<const float2*>(cp + static_cast<size_t>(r) * 512 + 128 + n);
      float z0, z1;
      if (p.fast_gate) {
        z0 = gate_fast(c0[e] + cgv.x, c1[e] + cfv.x);
        z1 = gate_fast(c0[e + 1] + cgv.y, c1[e + 1] + cfv.y);
      } else {
        z0 = gate_acc(c0[e] + cgv.x, c1[e] + cfv.x);
        z1 = gate_acc(c0[e + 1] + cgv.y, c1[e + 1] + cfv.y);
      }
      const __half2 hh = __floats2half2_rn(z0, z1);
      const uint32_t off = opnd_off(r, 128 * h + n);
      *reinterpret_cast<__half2*>(zb + off) = hh;
      if (P == 3) {
        const float2 hf = __half22float2(hh);
        *reinterpret_cast<__half2*>(zb + 4 * kABytes + off) = __floats2half2_rn(z0 - hf.x, z1 - hf.y);
      }
    }
  }

  // ---- GEMM2 + residual / skip epilogues ----
  const bool last = (l + 1 == p.L);
  const float* dnext = last ? nullptr : p.dtab + static_cast<size_t>(b) * p.d_row_stride + static_cast<size_t>(l + 1) * kC;
  __half* Yout = p.Y + static_cast<size_t>((l + 1) & 1) * 2 * p.plane;
#pragma unroll 1
  for (int q = 0; q < 2; ++q) {
    auto load = [&](int s, uint8_t* bf) {
      const int kb = s / P, ps = s % P;
      const __half* wt = w2_tile(p, l, pass_wplane(ps), q, kb);
      load_w<NT>(bf, wt, wt + 128 * 64, 256, tid);
    };
    auto adesc = [&](int s, uint8_t*) {
      const int kb = s / P, ps = s % P;
      return wg_desc(smem_u32(zb + (pass_aplane(ps) * 4 + kb) * kABytes));
    };
    gemm<2>(c0, c1, 4 * P, load, adesc, buf0, buf1);
    const float* bias = p.b2 + static_cast<size_t>(l) * 512 + q * 256;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
      for (int e = 0; e < 64; e += 2) {
        const int r = acc_row(wtid, e), col = hh * 128 + acc_col(wtid, e);
        if (t0 + r >= p.T) continue;
        const float a0 = hh ? c1[e] : c0[e], a1 = hh ? c1[e + 1] : c0[e + 1];
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + col));
        const size_t off = (fbase + r) * kC + col;
        if (q == 0) {
          float2 xv = *reinterpret_cast<const float2*>(p.X + off);
          xv.x = (xv.x + (a0 + bb.x)) * 0.70710678118654752440f;
          xv.y = (xv.y + (a1 + bb.y)) * 0.70710678118654752440f;
          *reinterpret_cast<float2*>(p.X + off) = xv;
          if (!last) {
            const float2 dv = __ldg(reinterpret_cast<const float2*>(dnext + col));
            const float ya = xv.x + dv.x, yb = xv.y + dv.y;
            const __half2 hy = __floats2half2_rn(ya, yb);
            *reinterpret_cast<__half2*>(Yout + off) = hy;
            if (p.ylo) {
              const float2 hf = __half22float2(hy);
              *reinterpret_cast<__half2*>(Yout + p.plane + off) = __floats2half2_rn(ya - hf.x, yb - hf.y);
            }
          }
        } else {
          float2 sk = make_float2(a0 + bb.x, a1 + bb.y);
          if (l > 0) {
            const float2 old = *reinterpret_cast<const float2*>(p.SKIP + off);
            sk.x = old.x + sk.x;
            sk.y = old.y + sk.y;
          }
          *reinterpret_cast<float2*>(p.SKIP + off) = sk;
          if (last) {
            const float sa = sk.x * p.inv_sqrt_l, sb = sk.y * p.inv_sqrt_l;
            const __half2 hs = __floats2half2_rn(sa, sb);
            const float2 hf = __half22float2(hs);
            *reinterpret_cast<__half2*>(p.S16 + off) = hs;
            *reinterpret_cast<__half2*>(p.S16 + p.plane + off) = __floats2half2_rn(sa - hf.x, sb - hf.y);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// head of one tile: eps = W_out . relu(W_s . s16 + b_s) + b_out, sampler update, next input projection
// ------------------------------------------------------------------------------------------
template <int NWG>
__device__ __forceinline__ void head_tile(const HpParams& p, int u, uint8_t* buf0, uint8_t* buf1, uint8_t* zb) {
  constexpr int NT = NWG * 128;
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  const int frame0 = u * 64 * NWG;
  const int b = frame0 / p.Tp, t0 = frame0 % p.Tp + wg * 64;
  const size_t fbase = static_cast<size_t>(b) * p.Tp + t0;
  const int flags = p.head_flags, HP = p.HP;
  const bool do_head = flags & TC_HEAD, do_in = flags & TC_INPROJ;
  float c0[64], c1[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) c0[i] = 0.f;

  if (do_head) {
    // H1: h = relu(s16 . W_s^T + b_s) -> fp16 hi / lo operand
    auto load1 = [&](int s, uint8_t* bf) {
      const int kb = s / HP, ps = s % HP, wp = pass_wplane(ps);
      load_w<NT>(bf, whead_tile(p, wp * 8 + kb), whead_tile(p, wp * 8 + 4 + kb), 256, tid);
      load_a(bf + kWBytes + wg * kABytes, p.S16 + pass_aplane(ps) * p.plane, b, t0, kb * 64, p.T, p.Tp, wtid);
    };
    auto adesc1 = [&](int, uint8_t* bf) { return wg_desc(smem_u32(bf + kWBytes + wg * kABytes)); };
    gemm<2>(c0, c1, 4 * HP, load1, adesc1, buf0, buf1);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
      for (int e = 0; e < 64; e += 2) {
        const int r = acc_row(wtid, e), col = hh * 128 + acc_col(wtid, e);
        const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bs + col));
        const float a0 = fmaxf((hh ? c1[e] : c0[e]) + bb.x, 0.f), a1 = fmaxf((hh ? c1[e + 1] : c0[e + 1]) + bb.y, 0.f);
        const __half2 hv = __floats2half2_rn(a0, a1);
        const uint32_t off = opnd_off(r, col);
        *reinterpret_cast<__half2*>(zb + off) = hv;
        const float2 hf = __half22float2(hv);
        *reinterpret_cast<__half2*>(zb + 4 * kABytes + off) = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
      }
    }
    // H2: eps (before bias) = h . W_out^T, N = 128 (rows >= M of the packed tile are zero)
    auto load2 = [&](int s, uint8_t* bf) {
      const int kb = s / HP, ps = s % HP;
      const __half* wt = whead_tile(p, 16 + pass_wplane(ps) * 4 + kb);
      load_w<NT>(bf, wt, wt, 128, tid);
    };
    auto adesc2 = [&](int s, uint8_t*) {
      const int kb = s / HP, ps = s % HP;
      return wg_desc(smem_u32(zb + (pass_aplane(ps) * 4 + kb) * kABytes));
    };
    gemm<1>(c0, c1, 4 * HP, load2, adesc2, buf0, buf1);
  }

  // ---- mel phase: eps, sampler update, x_in operand of the input projection ----
  const bool need_x = (flags & (TC_UPDATE | TC_INPROJ | TC_PLMS)) != 0;
  const bool need_z = (flags & TC_UPDATE) && p.c.sigma != 0.f;
#pragma unroll
  for (int e = 0; e < 64; e += 2) {
    const int r = acc_row(wtid, e), m = acc_col(wtid, e);
    const int t = t0 + r;
    const bool valid = t < p.T && m < p.M;
    float xv[2] = {0.f, 0.f};
    if (valid) {
      const size_t xrow = static_cast<size_t>(b) * p.xs.b + static_cast<size_t>(t) * p.xs.t;
      float zn[2] = {0.f, 0.f};
      if (need_x)
        for (int i = 0; i < 2; ++i) xv[i] = p.x[xrow + static_cast<size_t>(m + i) * p.xs.c];
      if (need_z) {
        if (p.noise) {
          for (int i = 0; i < 2; ++i) zn[i] = p.noise[(static_cast<size_t>(b) * p.M + m + i) * p.T + t];
        } else {
          const float4 z4 = philox_normal4(p.seed, p.offset, mel_noise_block(b + p.b_off, m, t, p.M, p.T));
          zn[0] = (m & 3) == 0 ? z4.x : z4.z;
          zn[1] = (m & 3) == 0 ? z4.y : z4.w;
        }
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int mm = m + i;
        const size_t ei = (static_cast<size_t>(b) * p.M + mm) * p.T + t;
        float ev = 0.f;
        if (do_head) ev = c0[e + i] + __ldg(p.bf + mm);
        if (flags & TC_WRITE_EPS) p.eps[ei] = ev;
        if (flags & TC_UPDATE) {
          float xr = __fsub_rn(__fmul_rn(p.c.A, xv[i]), __fmul_rn(p.c.Bc, ev));
          xr = fminf(fmaxf(xr, -1.f), 1.f);
          const float mean = __fadd_rn(__fmul_rn(p.c.c1, xr), __fmul_rn(p.c.c2, xv[i]));
          xv[i] = __fadd_rn(mean, __fmul_rn(p.c.sigma, zn[i]));
          p.x[xrow + static_cast<size_t>(mm) * p.xs.c] = xv[i];
        }
        if (flags & TC_PLMS) {
          // linear multistep combination + get_x_pred, the reference's left-to-right fp32 order (k_plms_update)
          float comb = __fmul_rn(p.pl.c.w0, ev);
          if (p.pl.h1) comb = __fadd_rn(comb, __fmul_rn(p.pl.c.w1, p.pl.h1[ei]));
          if (p.pl.h2) comb = __fadd_rn(comb, __fmul_rn(p.pl.c.w2, p.pl.h2[ei]));
          if (p.pl.h3) comb = __fadd_rn(comb, __fmul_rn(p.pl.c.w3, p.pl.h3[ei]));
          const float ep = __fdiv_rn(comb, p.pl.c.denom);
          const float inner = __fsub_rn(__fmul_rn(p.pl.c.kx, xv[i]), __fmul_rn(p.pl.c.ke, ep));
          xv[i] = __fadd_rn(xv[i], __fmul_rn(p.pl.c.a_diff, inner));
          if (p.pl.eps_store) p.pl.eps_store[ei] = ev;
          if (p.pl.x_out) p.pl.x_out[ei] = xv[i];
          else p.x[xrow + static_cast<size_t>(mm) * p.xs.c] = xv[i];
        }
      }
    }
    if (do_in) {
      // K = 128 operand: bins >= M and frames >= T are zero
      const __half2 hv = __floats2half2_rn(xv[0], xv[1]);
      const uint32_t off = opnd_off(r, m);
      *reinterpret_cast<__half2*>(zb + off) = hv;
      const float2 hf = __half22float2(hv);
      *reinterpret_cast<__half2*>(zb + 4 * kABytes + off) = __floats2half2_rn(xv[0] - hf.x, xv[1] - hf.y);
    }
  }
  if (!do_in) return;

  // ---- input projection: x0 = relu(x_in . W_in^T + b_in) -> X ; y0 = split(x0 + d_0) -> Y buffer 0 ----
  auto load3 = [&](int s, uint8_t* bf) {
    const int kb = s / HP, wp = pass_wplane(s % HP);
    load_w<NT>(bf, whead_tile(p, 24 + wp * 4 + kb), whead_tile(p, 24 + wp * 4 + 2 + kb), 256, tid);
  };
  auto adesc3 = [&](int s, uint8_t*) {
    const int kb = s / HP, ps = s % HP;
    return wg_desc(smem_u32(zb + (pass_aplane(ps) * 4 + kb) * kABytes));
  };
  gemm<2>(c0, c1, 2 * HP, load3, adesc3, buf0, buf1);
  const float* d0 = p.d0 + static_cast<size_t>(b) * p.d0_row_stride;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
    for (int e = 0; e < 64; e += 2) {
      const int r = acc_row(wtid, e), col = hh * 128 + acc_col(wtid, e);
      if (t0 + r >= p.T) continue;
      const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bin + col));
      const float2 dv = __ldg(reinterpret_cast<const float2*>(d0 + col));
      const float x0 = fmaxf((hh ? c1[e] : c0[e]) + bb.x, 0.f), x1 = fmaxf((hh ? c1[e + 1] : c0[e + 1]) + bb.y, 0.f);
      const size_t off = (fbase + r) * kC + col;
      *reinterpret_cast<float2*>(p.X + off) = make_float2(x0, x1);
      const float ya = x0 + dv.x, yb = x1 + dv.y;
      const __half2 hy = __floats2half2_rn(ya, yb);
      *reinterpret_cast<__half2*>(p.Y + off) = hy;
      if (p.ylo) {
        const float2 hf = __half22float2(hy);
        *reinterpret_cast<__half2*>(p.Y + p.plane + off) = __floats2half2_rn(ya - hf.x, yb - hf.y);
      }
    }
  }
}

template <int NWG>
__global__ void __launch_bounds__(NWG * 128, 1) k_hp_step(const __grid_constant__ HpParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* buf0 = base;
  uint8_t* buf1 = base + StepCfg<NWG>::STAGE;
  uint8_t* zb = base + 2 * StepCfg<NWG>::STAGE + (threadIdx.x >> 7) * kZBytes;
  for (int l = p.l0; l < p.l1; ++l) {
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) layer_tile<NWG>(p, l, u, buf0, buf1, zb);
    if (l + 1 < p.l1 || p.head_flags) cg::this_grid().sync();
  }
  if (p.head_flags)
    for (int u = blockIdx.x; u < p.units; u += gridDim.x) head_tile<NWG>(p, u, buf0, buf1, zb);
}

// CP[l][frame][h * 256 + n] = cond . W1cond^T (hi / lo operands, 3 passes) + dilated_conv.bias + conditioner_projection.bias,
// for job (tile of 128 frames, layer) = (blockIdx.x, blockIdx.y)
__global__ void __launch_bounds__(256, 1) k_hp_condproj(const __grid_constant__ HpParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* buf0 = base;
  uint8_t* buf1 = base + StepCfg<2>::STAGE;
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  const int u = blockIdx.x, l = blockIdx.y;
  const int frame0 = u * 128;
  const int b = frame0 / p.Tp, t0 = frame0 % p.Tp + wg * 64;
  const size_t fbase = static_cast<size_t>(b) * p.Tp + t0;
  const size_t NF = p.plane / kC;
  float c0[64], c1[64];
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    auto load = [&](int s, uint8_t* bf) {
      const int kb = s / 3, ps = s % 3;
      const __half* wt = p.w + (static_cast<size_t>(l) * kRowsPerLayer + ((pass_wplane(ps) * 2 + h) * 16 + 12 + kb) * 256) * 64;
      load_w<256>(bf, wt, wt + 128 * 64, 256, tid);
      load_a(bf + kWBytes + wg * kABytes, p.CONDH + pass_aplane(ps) * p.plane, b, t0, kb * 64, p.T, p.Tp, wtid);
    };
    auto adesc = [&](int, uint8_t* bf) { return wg_desc(smem_u32(bf + kWBytes + wg * kABytes)); };
    gemm<2>(c0, c1, 12, load, adesc, buf0, buf1);
    float* cp = p.CP + (static_cast<size_t>(l) * NF + fbase) * 512 + h * 256;
    const float* bias = p.b1p + (static_cast<size_t>(l) * 2 + h) * 256;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
      for (int e = 0; e < 64; e += 2) {
        const int r = acc_row(wtid, e), n = hh * 128 + acc_col(wtid, e);
        const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + n));
        *reinterpret_cast<float2*>(cp + static_cast<size_t>(r) * 512 + n) =
            make_float2((hh ? c1[e] : c0[e]) + bb.x, (hh ? c1[e + 1] : c0[e + 1]) + bb.y);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// weight packing (tiles of 64 fp16 per row, in the order the K loops consume them)
// ------------------------------------------------------------------------------------------
// whead tile order (128 rows x 64 k each): skip_projection [plane][row half][kb 0..3] (16 tiles),
// output_projection [plane][kb 0..3] with rows >= M zero (8 tiles), input_projection [plane][row half][kb 0..1]
// with k >= M zero (8 tiles).
__global__ void k_pack_whead(const float* __restrict__ skip_w, const float* __restrict__ fin_w,
                             const float* __restrict__ in_w, __half* __restrict__ whead, int M) {
  const int tileidx = blockIdx.x, n = threadIdx.x;   // 128 threads = rows
  int plane;
  __half* dst = whead + (static_cast<size_t>(tileidx) * 128 + n) * 64;
  for (int kk = 0; kk < 64; ++kk) {
    float v = 0.f;
    if (tileidx < 16) {
      plane = tileidx / 8;
      const int nh = (tileidx / 4) & 1, kb = tileidx & 3;
      v = skip_w[static_cast<size_t>(nh * 128 + n) * kC + kb * 64 + kk];
    } else if (tileidx < 24) {
      const int u = tileidx - 16;
      plane = u / 4;
      const int kb = u & 3;
      v = (n < M) ? fin_w[static_cast<size_t>(n) * kC + kb * 64 + kk] : 0.f;
    } else {
      const int u = tileidx - 24;
      plane = u / 4;
      const int nh = (u / 2) & 1, kb = u & 1;
      const int k = kb * 64 + kk;
      v = (k < M) ? in_w[static_cast<size_t>(nh * 128 + n) * M + k] : 0.f;
    }
    const __half hi = __float2half_rn(v);
    dst[kk] = plane == 0 ? hi : __float2half_rn(v - __half2float(hi));
  }
}

// Source row (in w1f / w2f, see dsx_simt.cu) of row n of a residual-layer weight tile.  W1 chunk h: n < 128 -> gate of
// channel 128 h + n (conv output row 128 h + n), n >= 128 -> its filter (row 256 + 128 h + n - 128).  W2 half q: output
// row 256 q + n.
__device__ __forceinline__ const float* w_src(const float* w1f, const float* w2f, int l, bool is_w1, int hq, int kb, int n) {
  if (is_w1) {
    const int j = (n < 128) ? (128 * hq + n) : (kC + 128 * hq + (n - 128));
    return w1f + (static_cast<size_t>(l) * 2 * kC + j) * (4 * kC) + kb * 64;
  }
  return w2f + (static_cast<size_t>(l) * 2 * kC + hq * 256 + n) * kC + kb * 64;
}

// hi / lo planes, per layer (tiles of 256 rows x 64 k):
//   W1: idx = (plane * 2 + chunk) * 16 + kb over k = [tap0 | tap1 | tap2 | cond]
//   W2: idx = 64 + (plane * 2 + half) * 4 + kb
__global__ void k_pack_wtc(const float* __restrict__ w1f, const float* __restrict__ w2f,
                           const float* __restrict__ b1f, __half* __restrict__ wpack, float* __restrict__ b1p) {
  const int l = blockIdx.y, tileidx = blockIdx.x, n = threadIdx.x;
  const float* src;
  int plane;
  if (tileidx < 64) {
    plane = tileidx / 32;
    const int h = (tileidx / 16) & 1, kb = tileidx & 15;
    src = w_src(w1f, w2f, l, true, h, kb, n);
    if (plane == 0 && kb == 0) {
      const int j = (n < 128) ? (128 * h + n) : (kC + 128 * h + (n - 128));
      b1p[(static_cast<size_t>(l) * 2 + h) * 256 + n] = b1f[static_cast<size_t>(l) * 2 * kC + j];
    }
  } else {
    const int u = tileidx - 64;
    plane = u / 8;
    src = w_src(w1f, w2f, l, false, (u / 4) & 1, u & 3, n);
  }
  __half* dst = wpack + (static_cast<size_t>(l) * kRowsPerLayer + static_cast<size_t>(tileidx) * 256 + n) * 64;
  for (int kk = 0; kk < 64; ++kk) {
    const float v = src[kk];
    const __half hi = __float2half_rn(v);
    dst[kk] = plane == 0 ? hi : __float2half_rn(v - __half2float(hi));
  }
}

// R stochastically rounded fp16 copies of the GEMM1 (conv taps) / GEMM2 weights (fp16s mode): element v lies between two
// fp16 neighbours lo <= v <= hi and becomes hi with probability (v - lo) / (hi - lo), so E[w] = v; set r is used by
// diffusion step j with j % R == r.  Layout [R][L][32 tiles][256 rows][64]: W1 tile = h * 12 + kb, W2 tile = 24 + q * 4 + kb.
// Philox4x32-10 keyed by (seed, set), counter = element index.
__global__ void k_pack_wsr(const float* __restrict__ w1f, const float* __restrict__ w2f, __half* __restrict__ wsr, int L,
                           unsigned long long seed) {
  const int l = blockIdx.y, tileidx = blockIdx.x, set = blockIdx.z, n = threadIdx.x;
  const float* src = (tileidx < 24) ? w_src(w1f, w2f, l, true, tileidx / 12, tileidx % 12, n)
                                    : w_src(w1f, w2f, l, false, (tileidx - 24) / 4, (tileidx - 24) & 3, n);
  const size_t row = ((static_cast<size_t>(set) * L + l) * 32 + tileidx) * 256 + n;
  __half* dst = wsr + row * 64;
  const uint2 key = make_uint2(static_cast<uint32_t>(seed) ^ (0x9E3779B9u * static_cast<uint32_t>(set + 1)),
                               static_cast<uint32_t>(seed >> 32) + static_cast<uint32_t>(set));
  for (int k4 = 0; k4 < 16; ++k4) {
    const size_t ctr = (static_cast<size_t>(l) * 32 + tileidx) * 256 * 16 + static_cast<size_t>(n) * 16 + k4;
    const uint4 rnd = philox4x32_10(make_uint4(static_cast<uint32_t>(ctr), static_cast<uint32_t>(ctr >> 32), 0x5352u, 0u), key);
    const uint32_t u4[4] = {rnd.x, rnd.y, rnd.z, rnd.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float v = src[k4 * 4 + e];
      const __half hn = __float2half_rn(v);
      const float fn = __half2float(hn);
      // the other neighbour: one fp16 ulp towards v
      __half ho = hn;
      if (fn != v) {
        unsigned short bits = __half_as_ushort(hn);
        const bool away = (fn < v) == (fn >= 0.f);     // move away from zero when v lies beyond |hn|
        if (fn == 0.f) bits = (v > 0.f) ? 0x0001 : 0x8001;
        else bits = static_cast<unsigned short>(away ? bits + 1 : bits - 1);
        ho = __ushort_as_half(bits);
      }
      const float fo = __half2float(ho);
      // P(take the other neighbour) = |v - fn| / |fo - fn|
      const float pr = (fo != fn) ? fabsf(v - fn) / fabsf(fo - fn) : 0.f;
      const float uu = static_cast<float>(u4[e] >> 8) * (1.0f / 16777216.0f);
      dst[k4 * 4 + e] = (uu < pr) ? ho : hn;
    }
  }
}

bool tc_supported(const dsx_handle* h) { return h->m.C == kC && h->m.H == kC && h->m.M == 80; }

int tc_pack_model(dsx_handle* h, cudaStream_t s) {
  DSX_CHECK(tc_supported(h), DSX_E_INVALID, "tensor-core path needs residual_channels == hidden_size == 256 (got %d, %d)",
            h->m.C, h->m.H);
  __half* wpack;
  float* b1p;
  const size_t rows = static_cast<size_t>(h->m.L) * kRowsPerLayer;
  DSX_TRY(dev_alloc(h, reinterpret_cast<void**>(&wpack), rows * 64 * sizeof(__half), true));
  DSX_TRY(dev_alloc(h, reinterpret_cast<void**>(&b1p), static_cast<size_t>(h->m.L) * 512 * sizeof(float), true));
  k_pack_wtc<<<dim3(kRowsPerLayer / 256, h->m.L), 256, 0, s>>>(h->m.w1f, h->m.w2f, h->m.b1f, wpack, b1p);
  h->launches++;
  DSX_CUDA(cudaGetLastError());
  h->m.wpack = wpack;
  h->m.b1p = b1p;
  __half* whead;
  DSX_TRY(dev_alloc(h, reinterpret_cast<void**>(&whead), static_cast<size_t>(32) * 128 * 64 * sizeof(__half), true));
  k_pack_whead<<<32, 128, 0, s>>>(h->m.skip_w, h->m.fin_w, h->m.in_w, whead, h->m.M);
  h->launches++;
  DSX_CUDA(cudaGetLastError());
  h->m.whead = whead;
  h->m.wsr = nullptr;
  h->m.wsr_sets = 0;
  if (h->precision == DSX_PREC_FP16S) {
    const int R = std::max(1, h->sr_sets);
    __half* wsr;
    const size_t srows = static_cast<size_t>(R) * h->m.L * kSrRowsPerLayer;
    DSX_TRY(dev_alloc(h, reinterpret_cast<void**>(&wsr), srows * 64 * sizeof(__half), true));
    k_pack_wsr<<<dim3(32, h->m.L, R), 256, 0, s>>>(h->m.w1f, h->m.w2f, wsr, h->m.L, h->sr_seed);
    h->launches++;
    DSX_CUDA(cudaGetLastError());
    h->m.wsr = wsr;
    h->m.wsr_sets = R;
  }
  return DSX_OK;
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// co-resident CTAs of k_hp_step<NWG> on this device (cached per handle)
template <int NWG>
static int step_capacity(dsx_handle* h) {
  int& cache = h->step_occ[NWG - 1];
  if (cache == 0) {
    cudaFuncSetAttribute(k_hp_step<NWG>, cudaFuncAttributeMaxDynamicSharedMemorySize, StepCfg<NWG>::SMEM);
    int n = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_hp_step<NWG>, StepCfg<NWG>::THREADS, StepCfg<NWG>::SMEM);
    if (e != cudaSuccess) cudaGetLastError();
    cache = (e == cudaSuccess && n >= 1) ? n * h->sm_count : -1;
  }
  return cache;
}

static HpParams base_params(dsx_handle* h, const Geom& g, int rows) {
  const ModelDev& m = h->m;
  HpParams prm;
  memset(&prm, 0, sizeof(prm));
  prm.whead = m.whead;
  prm.X = h->ws.X;
  prm.SKIP = h->ws.SKIP;
  prm.Y = h->ws.Y;
  prm.S16 = h->ws.S16;
  prm.CONDH = h->ws.CONDH;
  prm.plane = g.frames_padded() * kC;
  prm.CP = h->ws.CP;
  prm.b1p = m.b1p;
  prm.b2 = m.b2f;
  prm.T = g.T; prm.Tp = g.Tp; prm.B = g.B;
  prm.units = static_cast<int>(g.frames_padded() / rows);
  prm.L = m.L; prm.cycle = m.cycle;
  prm.inv_sqrt_l = 1.0f / sqrtf(static_cast<float>(m.L));
  prm.HP = (h->precision == DSX_PREC_FP16) ? 1 : 3;
  prm.ylo = (h->precision == DSX_PREC_FP16X3) ? 1 : 0;
  prm.M = m.M;
  prm.bs = m.skip_b;
  prm.bf = m.fin_b;
  prm.bin = m.in_b;
  return prm;
}

static void set_head(dsx_handle* h, HpParams& prm, int flags, float* x, dsx_strides xs, float* eps, const float* noise,
                     uint64_t seed, uint64_t offset, DdpmCoef c, int next_row0, int row_per_b, const PlmsFuse* plms) {
  prm.head_flags = flags;
  prm.x = x;
  prm.xs = xs;
  prm.eps = eps;
  prm.noise = noise;
  prm.seed = seed;
  prm.offset = offset;
  prm.b_off = h->batch_offset;
  prm.c = c;
  if (plms) prm.pl = *plms;
  prm.d0 = h->ws.DTAB + static_cast<size_t>(next_row0) * h->m.L * kC;
  prm.d0_row_stride = row_per_b * h->m.L * kC;
}

static int launch_step(dsx_handle* h, const HpParams& prm, int rows, cudaStream_t s) {
  const int cap = rows == 64 ? step_capacity<1>(h) : step_capacity<2>(h);
  DSX_CHECK(cap > 0, DSX_E_CUDA, "k_hp_step<%d> cannot be resident on this device", rows / 64);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(std::min(prm.units, cap)));
  cfg.blockDim = dim3(rows == 64 ? StepCfg<1>::THREADS : StepCfg<2>::THREADS);
  cfg.dynamicSmemBytes = rows == 64 ? StepCfg<1>::SMEM : StepCfg<2>::SMEM;
  cfg.stream = s;
  // cooperative: the layers of one launch are separated by grid-wide barriers, so every CTA must be resident
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  if (rows == 64) DSX_CUDA(cudaLaunchKernelEx(&cfg, k_hp_step<1>, prm));
  else DSX_CUDA(cudaLaunchKernelEx(&cfg, k_hp_step<2>, prm));
  h->launches++;
  return DSX_OK;
}

static int gate_mode(const dsx_handle* h, int P) { return h->gate_approx >= 0 ? h->gate_approx : (P == 3 ? 0 : 1); }

// Layers [l0, l1) of one evaluation with the hi / lo weight planes: one launch (stack mode) or one launch per layer.
int launch_tc_layers(dsx_handle* h, int l0, int l1, const Geom& g, int row0, int row_per_b, cudaStream_t s) {
  HpParams prm = base_params(h, g, 128);
  prm.w = h->m.wpack;
  prm.P = (h->precision == DSX_PREC_FP16S) ? 2 : h->precision;   // DSX_PREC_FP16 = 1, FP16X2 = 2, FP16X3 = 3 == MMA passes
  prm.fast_gate = gate_mode(h, prm.P);
  prm.dtab = h->ws.DTAB + static_cast<size_t>(row0) * h->m.L * kC;
  prm.d_row_stride = row_per_b * h->m.L * kC;
  if (h->stack_mode && l1 - l0 > 1) {
    prm.l0 = l0; prm.l1 = l1;
    return launch_step(h, prm, 128, s);
  }
  for (int l = l0; l < l1; ++l) {
    prm.l0 = l; prm.l1 = l + 1;
    DSX_TRY(launch_step(h, prm, 128, s));
  }
  return DSX_OK;
}

// CP for the conditioner currently packed in ws.CONDH (called once per API call, after launch_pack_cond).
int launch_tc_condproj(dsx_handle* h, const Geom& g, cudaStream_t s) {
  if (!h->attr_cond) {
    DSX_CUDA(cudaFuncSetAttribute(k_hp_condproj, cudaFuncAttributeMaxDynamicSharedMemorySize, kCondSmem));
    h->attr_cond = true;
  }
  HpParams prm = base_params(h, g, 128);
  prm.w = h->m.wpack;
  k_hp_condproj<<<dim3(static_cast<unsigned>(prm.units), static_cast<unsigned>(h->m.L)), 256, kCondSmem, s>>>(prm);
  h->launches++;
  DSX_CUDA(cudaGetLastError());
  return DSX_OK;
}

int launch_tc_head(dsx_handle* h, const Geom& g, int flags, float* x_state, dsx_strides xs, float* eps_out,
                   const float* noise, uint64_t seed, uint64_t offset, DdpmCoef c, int next_row0, int row_per_b,
                   cudaStream_t s, const PlmsFuse* plms) {
  HpParams prm = base_params(h, g, 128);
  set_head(h, prm, flags, x_state, xs, eps_out, noise, seed, offset, c, next_row0, row_per_b, plms);
  return launch_step(h, prm, 128, s);
}

// Frames per CTA for this call: 64 (one warpgroup per CTA, twice the CTAs) whenever the whole batch then has a CTA per
// tile at once, i.e. for small batches that would otherwise leave most SMs idle; 128 otherwise.
static int stack_rows(dsx_handle* h, const Geom& g) {
  if (h->stack_rows == 64 || h->stack_rows == 128) return h->stack_rows;      // DSX_OPT_STACK_ROWS
  const int cap64 = step_capacity<1>(h);
  return (cap64 > 0 && g.frames_padded() / 64 <= static_cast<size_t>(cap64)) ? 64 : 128;
}

// Does the one-launch-per-step form take this call?  (precisions with a single weight plane per pass set)
bool tc_stack_usable(dsx_handle* h, const Geom&) {
  if (h->stack_kernel == 0 || !h->stack_mode) return false;
  return h->precision == DSX_PREC_FP16 || h->precision == DSX_PREC_FP16X2 || h->precision == DSX_PREC_FP16S;
}

// Layers [0, nl) of one evaluation (table row row0, weight set `wset` in fp16s), optionally followed by the head, in one
// launch.
int launch_tc_stack(dsx_handle* h, int nl, const Geom& g, int row0, int row_per_b, int wset, cudaStream_t s, const HeadArgs* head) {
  const ModelDev& m = h->m;
  if (nl <= 0) return DSX_OK;
  const int rows = stack_rows(h, g);
  h->stack_rows_used = rows;
  HpParams prm = base_params(h, g, rows);
  const bool sr = (h->precision == DSX_PREC_FP16S);
  prm.w_sr = sr ? 1 : 0;
  prm.w = sr ? m.wsr + static_cast<size_t>(wset % std::max(1, m.wsr_sets)) * m.L * kSrRowsPerLayer * 64 : m.wpack;
  prm.P = (h->precision == DSX_PREC_FP16X2) ? 2 : 1;
  prm.fast_gate = gate_mode(h, prm.P);
  prm.dtab = h->ws.DTAB + static_cast<size_t>(row0) * m.L * kC;
  prm.d_row_stride = row_per_b * m.L * kC;
  prm.l0 = 0;
  prm.l1 = nl;
  if (head && head->flags) {
    DSX_CHECK(nl == m.L, DSX_E_INVALID, "the fused head needs the whole stack");
    set_head(h, prm, head->flags | TC_HEAD, head->x, head->xs, head->eps, head->noise, head->seed, head->offset, head->c,
             head->next_row0, head->row_per_b, head->plms);
  }
  DSX_TRY(launch_step(h, prm, rows, s));
  h->stack_launches++;
  return DSX_OK;
}

// ------------------------------------------------------------------------------------------
// self-test: the operand loads (swizzle, row shift, zero fill) and the wgmma descriptors against a host GEMM
// ------------------------------------------------------------------------------------------
struct SelfParams {
  const __half* a;   // [T][256] fp16, one utterance
  const __half* w;   // [256 rows][64]
  float* out;        // [64][256]
  int t0, T;
};

__global__ void __launch_bounds__(128, 1) k_selftest(const __grid_constant__ SelfParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int wtid = threadIdx.x;
  float c0[64], c1[64];
  auto load = [&](int s, uint8_t* bf) {
    load_w<128>(bf, p.w, p.w + 128 * 64, 256, wtid);
    load_a(bf + kWBytes, p.a, 0, p.t0, s * 64, p.T, p.T, wtid);
  };
  auto adesc = [&](int, uint8_t* bf) { return wg_desc(smem_u32(bf + kWBytes)); };
  gemm<2>(c0, c1, 1, load, adesc, base, base + kWBytes + kABytes);
  for (int e = 0; e < 64; ++e) {
    const int r = acc_row(wtid, e), n = acc_col(wtid, e);
    p.out[r * 256 + n] = c0[e];
    p.out[r * 256 + 128 + n] = c1[e];
  }
}

static int run_selftest(std::string& report) {
  const int T = 150;
  auto aval = [](int t, int c) { return static_cast<float>((t * 131 + c * 71) % 61 - 30) / 64.f; };
  auto wval = [](int n, int k) { return static_cast<float>((n * 37 + k * 11) % 53 - 26) / 128.f; };
  std::vector<__half> ha(static_cast<size_t>(T) * 256), hw(256 * 64);
  for (int t = 0; t < T; ++t)
    for (int c = 0; c < 256; ++c) ha[static_cast<size_t>(t) * 256 + c] = __float2half(aval(t, c));
  for (int n = 0; n < 256; ++n)
    for (int k = 0; k < 64; ++k) hw[static_cast<size_t>(n) * 64 + k] = __float2half(wval(n, k));
  __half *da = nullptr, *dw = nullptr;
  float* dout = nullptr;
  DSX_CUDA(cudaMalloc(&da, ha.size() * 2));
  DSX_CUDA(cudaMalloc(&dw, hw.size() * 2));
  DSX_CUDA(cudaMalloc(&dout, 64 * 256 * 4));
  DSX_CUDA(cudaMemcpy(da, ha.data(), ha.size() * 2, cudaMemcpyHostToDevice));
  DSX_CUDA(cudaMemcpy(dw, hw.data(), hw.size() * 2, cudaMemcpyHostToDevice));
  const int smem = 1024 + 2 * (kWBytes + kABytes);
  DSX_CUDA(cudaFuncSetAttribute(k_selftest, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int failures = 0;
  const int starts[] = {0, -8, 37, 120};     // interior, leading zero fill, unaligned, trailing zero fill
  for (int t0 : starts) {
    SelfParams prm{da, dw, dout, t0, T};
    DSX_CUDA(cudaMemset(dout, 0xff, 64 * 256 * 4));
    k_selftest<<<1, 128, smem>>>(prm);
    DSX_CUDA(cudaGetLastError());
    DSX_CUDA(cudaDeviceSynchronize());
    std::vector<float> out(64 * 256);
    DSX_CUDA(cudaMemcpy(out.data(), dout, out.size() * 4, cudaMemcpyDeviceToHost));
    int bad = 0;
    double maxerr = 0;
    for (int m = 0; m < 64; ++m)
      for (int n = 0; n < 256; ++n) {
        double ref = 0;
        const int t = t0 + m;
        if (t >= 0 && t < T)
          for (int k = 0; k < 64; ++k) ref += static_cast<double>(aval(t, k)) * wval(n, k);
        const double e = fabs(ref - out[static_cast<size_t>(m) * 256 + n]);
        if (!(e <= 1e-4)) bad++;
        if (e > maxerr || e != e) maxerr = e;
      }
    char line[160];
    snprintf(line, sizeof(line), "wgmma_m64n128k16 t0=%d: bad=%d/16384 maxerr=%.3g\n", t0, bad, maxerr);
    report += line;
    if (bad) failures++;
  }
  cudaFree(da);
  cudaFree(dw);
  cudaFree(dout);
  return failures ? DSX_E_KERNEL : DSX_OK;
}

}  // namespace dsx

extern "C" int dsx_selftest(int device, int which, char* report, int report_bytes) {
  using namespace dsx;
  DSX_CUDA(cudaSetDevice(device));
  std::string rep;
  int rc = DSX_OK;
  if (which < 0 || which == 0) rc = run_selftest(rep);
  if (report && report_bytes > 0) {
    strncpy(report, rep.c_str(), static_cast<size_t>(report_bytes) - 1);
    report[report_bytes - 1] = 0;
  }
  if (rc != DSX_OK) set_error("selftest failed: %s", rep.c_str());
  return rc;
}
