// DiffNet training step on sm_90a: DiffNet.forward (usr/diff/net.py:107-130) with its activations saved to a
// caller-owned tape, and the exact backward to every parameter and to cond.
//
// Operands are fp16 and every GEMM accumulates in fp32.  Forward GEMMs and the backward's data-gradient GEMMs run on the
// implicit-GEMM core of dsx_conv.cuh (k_train_gemm, one 64-frame x 256-column CTA, epilogue by mode):
//   F_IN    input_projection: x0 = relu(.) -> residual stream X (fp32), y_0 = x0 + d_0(t) (fp16, tape)
//   F_GATE  dilated conv on y_l (taps -d, 0, +d) + conditioner projection (a second operand pair into the same
//           accumulators); columns are packed gate / filter interleaved by 8 so each thread holds both halves of a
//           channel: sigma(g), tanh(f) and z = sigma(g) tanh(f) to the tape
//   F_OUT   output_projection on z: column tile 0 is the residual, x <- (x + r) / sqrt(2) and y_{l+1} = x + d_{l+1}(t);
//           tile 1 the skip, summed in fp32; the last layer writes skip_sum / sqrt(L) (fp16, tape)
//   F_SKIP  skip_projection + ReLU (tape), F_FIN output_projection -> eps [B, 1, M, T]
//   B_FIN   d eps -> d of the ReLU'd skip projection (fp16), B_SKIP -> d skip_l (the same for every layer)
//   B_OUT   output_projection's dgrad and the gate derivative -> dpre_l (fp16 [frames][2C], kept for d_cond)
//   B_DIL   the dilated conv's dgrad: a stride-1 transposed conv, tap j reading dpre at m + (1 - j) d; the epilogue forms
//           dx_l = dx_{l+1} / sqrt(2) + dy_l and the per-tile column sums of dy_l (the gradient of d_l(t))
//   B_COND  d_cond = sum_l W_cond,l^T dpre_l as one GEMM with K = L * 2C: tap l reads layer l's dpre
// Weight gradients reduce over the frame axis, so both operands are frames-major and enter wgmma MN-major
// (k_wgrad): the frames split over CTAs, each writes an fp32 partial, and k_wgrad_sum sums the partials in a fixed
// order (no atomics: gradients are bitwise reproducible).  Bias gradients are the column sums of the same A tiles.  The
// dilated conv and the conditioner projection share one wgrad launch whose B operand is [y(-d) | y | y(+d) | cond].  The
// step-embedding MLP and diffusion_projection (B rows) are on CUDA cores.
//
// The incoming gradient of a mean loss is tiny (1 / (B M T)), subnormal in fp16.  The backward finds amax |d eps| on the
// device and scales every fp16 gradient operand by the power of two S that brings it to [2^5, 2^6); the fp32 results are
// multiplied by 1 / S, which is exact, so the gradients for 2^k d_eps are exactly 2^k times those for d_eps.  d eps is
// the largest gradient operand of the backward (oracle/precision_study_train.py fp16dyn), so the scaled operands stay
// about 2^10 below the fp16 maximum, while the smallest stay clear of fp16's subnormals.
#include <math.h>

#include <algorithm>
#include <vector>

#include "dsx_conv.cuh"
#include "dsx_internal.h"
#include "dsx_ptx.cuh"
#include "dsx_wgrad.cuh"

namespace dsx {
namespace {

constexpr int kM = 80, kC = 256, kH = 256, kN1 = 2 * kC;
constexpr int kNT = 256;                 // columns per CTA of every training GEMM (two warpgroups of 128)
constexpr float kRsqrt2 = 0.70710678118654752f;

enum { F_IN, F_GATE, F_OUT, F_SKIP, F_FIN, B_FIN, B_SKIP, B_OUT, B_DIL, B_COND };

struct GemmArgs {
  ConvGemm g;
  const __half* x;             // A operand [B][T][g.cin]
  ConvGemm g2;                 // F_GATE: the conditioner projection, accumulated
  const __half* x2;
  int mode, B, T, L, layer;
  float rsqrtL;
  float* X;                    // fp32 [F][C]: residual stream (forward) / dx (B_DIL)
  float* SKIP;                 // fp32 [F][C]
  const float* D;              // [B][C] d_l(t) of the layer whose y this writes (F_IN, F_OUT), or null
  __half* o16;                 // the fp16 output of the mode
  __half* o16b;                // F_GATE: z; F_IN: the x0 copy; B_DIL: d of input_projection (layer 0)
  const __half* aux;           // F_GATE -; B_OUT: sigma | tanh; B_FIN: relu output; B_DIL: x0
  float* o32;                  // F_FIN: eps; B_COND: d_cond; B_DIL: per-tile column sums
  const float* inv_s;          // device 1 / S (B_COND)
};

// v > 0 stays > 0 in fp16 (smallest subnormal), so the stored value carries the exact ReLU mask of the fp32 value
__device__ __forceinline__ __half half_pos(float v) {
  return v > 0.f ? __float2half_rn(fmaxf(v, 5.9604645e-8f)) : __float2half_rn(0.f);
}

template <int NT>
__global__ void __launch_bounds__(256) k_train_gemm(const GemmArgs p) {
  constexpr int WG = 2, NH = NT / WG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ float red[8][NH];
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, b = blockIdx.y, m0 = blockIdx.x * kConvRows;
  const int tile = blockIdx.z, T = p.T;
  // B_COND: tap l reads layer l's dpre B * T frames further on; rows past T of the last utterance must stay in bounds
  const int valid = p.mode == B_COND ? (p.L * p.B - b) * T : T;

  float acc[NH / 2];
  conv_k_loop<NT, WG>(p.g, p.x, T, valid, b, m0, tile, smem, acc);
  if (p.mode == F_GATE) conv_k_loop<NT, WG>(p.g2, p.x2, T, T, b, m0, tile, smem, acc, true);

  const int r0 = acc_row(wtid, 0);
  const int c0 = tile * NT + wg * NH;         // first GEMM column of this warpgroup
  auto frame = [&](int e) -> int64_t {        // frame index of accumulator e, or -1 past the utterance
    const int m = m0 + r0 + ((e & 2) ? 8 : 0);
    return m < T ? static_cast<int64_t>(b) * T + m : -1;
  };
  const float* bias = p.g.b;

  switch (p.mode) {
    case F_IN:
    case F_SKIP:
#pragma unroll
      for (int e = 0; e < NH / 2; e += 2) {
        const int64_t f = frame(e);
        if (f < 0) continue;
        const int c = c0 + acc_col(wtid, e);
        const float v0 = fmaxf(acc[e] + bias[c], 0.f), v1 = fmaxf(acc[e + 1] + bias[c + 1], 0.f);
        if (p.mode == F_SKIP) {
          p.o16[f * kC + c] = half_pos(v0);
          p.o16[f * kC + c + 1] = half_pos(v1);
          continue;
        }
        *reinterpret_cast<float2*>(p.X + f * kC + c) = make_float2(v0, v1);
        p.o16b[f * kC + c] = half_pos(v0);
        p.o16b[f * kC + c + 1] = half_pos(v1);
        const float* d = p.D + b * kC;
        *reinterpret_cast<__half2*>(p.o16 + f * kC + c) = __floats2half2_rn(v0 + d[c], v1 + d[c + 1]);
      }
      break;
    case F_GATE:
      // packed column n = 16 q + r: channel 8 q + (r & 7), gate for r < 8, filter for r >= 8; element e (8-column group
      // i = e / 4 even) is a gate column and e + 4 the filter column of the same channel
#pragma unroll
      for (int e = 0; e < NH / 2; ++e) {
        if ((e >> 2) & 1) continue;
        const int64_t f = frame(e);
        if (f < 0) continue;
        const int n = c0 + acc_col(wtid, e), ch = 8 * (n >> 4) + (n & 7);
        const float sg = 1.f / (1.f + expf(-(acc[e] + bias[n])));
        const float tf = tanhf(acc[e + 4] + bias[n + 8]);
        p.o16[f * kN1 + ch] = __float2half_rn(sg);
        p.o16[f * kN1 + kC + ch] = __float2half_rn(tf);
        p.o16b[f * kC + ch] = __float2half_rn(sg * tf);
      }
      break;
    case F_OUT:
#pragma unroll
      for (int e = 0; e < NH / 2; e += 2) {
        const int64_t f = frame(e);
        if (f < 0) continue;
        const int n = c0 + acc_col(wtid, e);
        const float v0 = acc[e] + bias[n], v1 = acc[e + 1] + bias[n + 1];
        if (tile == 0) {
          float2* xp = reinterpret_cast<float2*>(p.X + f * kC + n);
          float2 x = *xp;
          x.x = (x.x + v0) * kRsqrt2;
          x.y = (x.y + v1) * kRsqrt2;
          *xp = x;
          if (p.D) {
            const float* d = p.D + b * kC;
            *reinterpret_cast<__half2*>(p.o16 + f * kC + n) = __floats2half2_rn(x.x + d[n], x.y + d[n + 1]);
          }
        } else {
          const int c = n - kC;
          float2* sp = reinterpret_cast<float2*>(p.SKIP + f * kC + c);
          float2 s = p.layer == 0 ? make_float2(0.f, 0.f) : *sp;
          s.x += v0;
          s.y += v1;
          *sp = s;
          if (p.layer == p.L - 1)
            *reinterpret_cast<__half2*>(p.o16b + f * kC + c) = __floats2half2_rn(s.x * p.rsqrtL, s.y * p.rsqrtL);
        }
      }
      break;
    case F_FIN:
#pragma unroll
      for (int e = 0; e < NH / 2; ++e) {
        const int64_t f = frame(e);
        const int n = c0 + acc_col(wtid, e);
        if (f < 0 || n >= kM) continue;
        const int m = m0 + r0 + ((e & 2) ? 8 : 0);
        p.o32[(static_cast<size_t>(b) * kM + n) * T + m] = acc[e] + bias[n];
      }
      break;
    case B_FIN:
#pragma unroll
      for (int e = 0; e < NH / 2; e += 2) {
        const int64_t f = frame(e);
        if (f < 0) continue;
        const int c = c0 + acc_col(wtid, e);
        const __half2 h = *reinterpret_cast<const __half2*>(p.aux + f * kC + c);
        *reinterpret_cast<__half2*>(p.o16 + f * kC + c) =
            __floats2half2_rn(__low2float(h) > 0.f ? acc[e] : 0.f, __high2float(h) > 0.f ? acc[e + 1] : 0.f);
      }
      break;
    case B_SKIP:
#pragma unroll
      for (int e = 0; e < NH / 2; e += 2) {
        const int64_t f = frame(e);
        if (f < 0) continue;
        const int c = c0 + acc_col(wtid, e);
        *reinterpret_cast<__half2*>(p.o16 + f * kN1 + kC + c) = __floats2half2_rn(acc[e] * p.rsqrtL, acc[e + 1] * p.rsqrtL);
      }
      break;
    case B_OUT:
      // z = sigma(g) tanh(f): dg = dz tanh(f) sigma (1 - sigma), df = dz sigma (1 - tanh^2)
#pragma unroll
      for (int e = 0; e < NH / 2; ++e) {
        const int64_t f = frame(e);
        if (f < 0) continue;
        const int c = c0 + acc_col(wtid, e);
        const float sg = __half2float(p.aux[f * kN1 + c]), tf = __half2float(p.aux[f * kN1 + kC + c]);
        p.o16[f * kN1 + c] = __float2half_rn(acc[e] * tf * sg * (1.f - sg));
        p.o16[f * kN1 + kC + c] = __float2half_rn(acc[e] * sg * (1.f - tf * tf));
      }
      break;
    case B_DIL: {
      float colsum[NH / 4];   // this thread's columns 8 i + 2 (t % 4) + j at index 2 i + j
#pragma unroll
      for (int i = 0; i < NH / 4; ++i) colsum[i] = 0.f;
#pragma unroll
      for (int e = 0; e < NH / 2; ++e) {
        const int64_t f = frame(e);
        if (f < 0) continue;
        const int c = c0 + acc_col(wtid, e);
        colsum[((e >> 2) << 1) | (e & 1)] += acc[e];
        const float dx = (p.layer == p.L - 1 ? 0.f : p.X[f * kC + c] * kRsqrt2) + acc[e];
        p.X[f * kC + c] = dx;
        p.o16[f * kN1 + c] = __float2half_rn(dx * kRsqrt2);
        if (p.layer == 0) p.o16b[f * kC + c] = __float2half_rn(__half2float(p.aux[f * kC + c]) > 0.f ? dx : 0.f);
      }
      // column sums over the tile's 64 rows: the 8 row groups of a warp, then its 4 warps, in a fixed order
      const int warp = tid >> 5, lane = tid & 31;
#pragma unroll
      for (int i = 0; i < NH / 4; ++i) {
        float v = colsum[i];
        v += __shfl_xor_sync(0xffffffffu, v, 4);
        v += __shfl_xor_sync(0xffffffffu, v, 8);
        v += __shfl_xor_sync(0xffffffffu, v, 16);
        if (lane < 4) red[warp][((i >> 1) << 3) + 2 * lane + (i & 1)] = v;
      }
      __syncthreads();
      {
        const int w = tid >> 7, cl = tid & 127;
        const float s = ((red[4 * w][cl] + red[4 * w + 1][cl]) + red[4 * w + 2][cl]) + red[4 * w + 3][cl];
        p.o32[(static_cast<size_t>(b) * gridDim.x + blockIdx.x) * kC + tile * NT + tid] = s;
      }
      break;
    }
    case B_COND: {
      const float is = *p.inv_s;
#pragma unroll
      for (int e = 0; e < NH / 2; ++e) {
        const int m = m0 + r0 + ((e & 2) ? 8 : 0);
        if (m >= T) continue;
        const int h = c0 + acc_col(wtid, e);
        p.o32[(static_cast<size_t>(b) * kH + h) * T + m] = acc[e] * is;
      }
      break;
    }
  }
}

// ---- packing --------------------------------------------------------------------------------------------------------
// the dilated conv (k = 3) or the conditioner projection (k = 1) with gate / filter columns interleaved by 8 (see
// F_GATE); bias (b1 + b2, either may be null) -> g.b
__global__ void k_pack_gate(const ConvGemm g, const float* v, int k, const float* b1, const float* b2) {
  const size_t total = static_cast<size_t>(g.ntiles) * g.kc * g.nt * 64;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(i & 63);
    size_t t = i >> 6;
    const int rr = static_cast<int>(t % g.nt);
    t /= g.nt;
    const int s = static_cast<int>(t % g.kc), tile = static_cast<int>(t / g.kc);
    const int n = tile * g.nt + rr, kk = s * 64 + q, j = kk / g.cin, c = kk - j * g.cin;
    const int o = ((n & 15) < 8 ? 0 : kC) + 8 * (n >> 4) + (n & 7);
    const float val = j < g.taps ? v[(static_cast<size_t>(o) * g.cin + c) * k + j] : 0.f;
    g.w[i] = __float2half_rn(val);
    if (i < static_cast<size_t>(kN1)) {
      const int oo = ((static_cast<int>(i) & 15) < 8 ? 0 : kC) + 8 * (static_cast<int>(i) >> 4) + (static_cast<int>(i) & 7);
      g.b[i] = (b1 ? b1[oo] : 0.f) + (b2 ? b2[oo] : 0.f);
    }
  }
}

// x logically [B, C, T] (any strides) -> fp16 [B][T][C]; one warp per frame
__global__ void k_pack_frames(const float* x, dsx_strides xs, int B, int T, int C, __half* out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * T) return;
  const int b = warp / T, t = warp - b * T;
  const float* src = x + b * xs.b + t * xs.t;
  for (int c = lane; c < C; c += 32) out[static_cast<size_t>(warp) * C + c] = __float2half_rn(src[c * xs.c]);
}

// d_l(t) = diffusion_projection_l(emb): out [B][C]; one warp per output
__global__ void k_dproj(const float* w, const float* bias, const float* emb, int B, float* out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * kC) return;
  const int b = warp / kC, c = warp % kC;
  float acc = 0.f;
  for (int k = lane; k < kC; k += 32) acc = fmaf(w[c * kC + k], emb[b * kC + k], acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) out[warp] = acc + bias[c];
}

// ---- backward prologue: S from amax |d eps|, and d eps * S -> fp16 [B][T][M] ------------------------------------------
__global__ void k_grad_in(const float* g, const float* scal, int B, int T, __half* out) {
  const size_t n = static_cast<size_t>(B) * kM * T;
  const float S = scal[0];
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int t = static_cast<int>(i % T), m = static_cast<int>((i / T) % kM), b = static_cast<int>(i / (static_cast<size_t>(T) * kM));
    out[(static_cast<size_t>(b) * T + t) * kM + m] = __float2half_rn(g[i] * S);
  }
}

// ---- step embedding backward (CUDA cores) -----------------------------------------------------------------------------
// layer l: dD = sum over the tiles of the B_DIL column sums; blocks [0, C): diffusion_projection's weight row c and
// bias; blocks [C, C + B): dE_l[b][k] = sum_c W[c][k] dD[b][c]
__global__ void k_dif_grad(const float* ddp, int mtiles, int B, const float* emb, const float* w, const float* scal,
                           float* dw, float* db, float* de_l) {
  __shared__ float dd[kC];
  const int k = threadIdx.x;
  const float is = scal[1];
  if (blockIdx.x < kC) {
    const int c = blockIdx.x;
    float sw = 0.f, sb = 0.f;
    for (int b = 0; b < B; ++b) {
      float d = 0.f;
      for (int t = 0; t < mtiles; ++t) d += ddp[(static_cast<size_t>(b) * mtiles + t) * kC + c];
      sw = fmaf(d, emb[b * kC + k], sw);
      sb += d;
    }
    dw[c * kC + k] = sw * is;
    if (k == 0) db[c] = sb * is;
  } else {
    const int b = blockIdx.x - kC;
    float d = 0.f;
    for (int t = 0; t < mtiles; ++t) d += ddp[(static_cast<size_t>(b) * mtiles + t) * kC + k];
    dd[k] = d;
    __syncthreads();
    float s = 0.f;
    for (int c = 0; c < kC; ++c) s = fmaf(w[c * kC + k], dd[c], s);
    de_l[b * kC + k] = s;
  }
}

// de[b][k] = sum_l dE_l[b][k], in layer order
__global__ void k_de_sum(const float* de_l, int L, int B, float* de) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * kC) return;
  float s = 0.f;
  for (int l = 0; l < L; ++l) s += de_l[static_cast<size_t>(l) * B * kC + i];
  de[i] = s;
}

// ---- tape layout --------------------------------------------------------------------------------------------------
struct Tape {
  __half* spec;   // [F][M]
  __half* cond;   // [F][H]
  __half* x0;     // [F][C] relu(input_projection), positivity kept (the ReLU mask)
  __half* s16;    // [F][C] skip_sum / sqrt(L)
  __half* h1;     // [F][C] relu(skip_projection), positivity kept
  float* emb;     // [B][C] mlp output
  float* save;    // [B][9 C] sinusoid, mlp.0 output, Mish of it
  std::vector<__half*> y, sg, z;   // per layer: [F][C] conv input, [F][2C] sigma(g) | tanh(f), [F][C] gate output
};

}  // namespace
}  // namespace dsx

struct dsx_train {
  int device = 0;
  int L = 0, cycle = 1;
  dsx::ConvGemm in, skip, fin, skip_t, fin_t, cond_t;
  std::vector<dsx::ConvGemm> dil, cnd, out, out_t, dil_t;
  float* zeros = nullptr;      // bias slot of the transposed packs
  dsx::DevAllocs mem;
};

namespace dsx {
namespace {

// every region of the tape for (L, B, T), in order; bytes of the whole tape
size_t tape_carve(int L, int B, int T, uint8_t* base, Tape* t) {
  const size_t f = static_cast<size_t>(B) * T;
  size_t n = 0;
  auto take = [&](size_t bytes) {
    uint8_t* p = base ? base + n : nullptr;
    n += align256(bytes);
    return p;
  };
  Tape dummy;
  Tape& tp = t ? *t : dummy;
  tp.spec = reinterpret_cast<__half*>(take(f * kM * 2));
  tp.cond = reinterpret_cast<__half*>(take(f * kH * 2));
  tp.x0 = reinterpret_cast<__half*>(take(f * kC * 2));
  tp.s16 = reinterpret_cast<__half*>(take(f * kC * 2));
  tp.h1 = reinterpret_cast<__half*>(take(f * kC * 2));
  tp.emb = reinterpret_cast<float*>(take(static_cast<size_t>(B) * kC * 4));
  tp.save = reinterpret_cast<float*>(take(static_cast<size_t>(B) * 9 * kC * 4));
  tp.y.resize(L);
  tp.sg.resize(L);
  tp.z.resize(L);
  for (int l = 0; l < L; ++l) {
    tp.y[l] = reinterpret_cast<__half*>(take(f * kC * 2));
    tp.sg[l] = reinterpret_cast<__half*>(take(f * kN1 * 2));
    tp.z[l] = reinterpret_cast<__half*>(take(f * kC * 2));
  }
  return n;
}

void gemm_shape(ConvGemm& g, int cin, int n, int taps) {
  g.cin = cin;
  g.n = n;
  g.taps = taps;
  g.nt = kNT;
  g.ntiles = (n + kNT - 1) / kNT;
  g.kc = (taps * cin + 63) / 64;
}

size_t gemm_elems(const ConvGemm& g) { return static_cast<size_t>(g.ntiles) * g.kc * g.nt * 64; }

int gemm_alloc(DevAllocs& mem, ConvGemm& g, int cin, int n, int taps) {
  gemm_shape(g, cin, n, taps);
  DSX_TRY(mem.alloc(&g.w, gemm_elems(g) * sizeof(__half)));
  DSX_TRY(mem.alloc(&g.b, static_cast<size_t>(g.ntiles) * g.nt * sizeof(float)));
  return DSX_OK;
}

unsigned pack_blocks(const ConvGemm& g) { return static_cast<unsigned>(std::min<size_t>((gemm_elems(g) + 255) / 256, 2048)); }

int pack(const ConvGemm& g, const PackArgs& a, cudaStream_t s) {
  k_pack_conv<<<pack_blocks(g), 256, 0, s>>>(g, a);
  return launch_check("k_pack_conv");
}

int run_gemm(const GemmArgs& a, int B, int T, cudaStream_t s) {
  dim3 grid((T + kConvRows - 1) / kConvRows, B, a.g.ntiles);
  k_train_gemm<kNT><<<grid, 256, conv_smem<kNT>(), s>>>(a);
  return launch_check("k_train_gemm");
}

// the backward's workspace regions: scalars, d eps (fp16), dh1, [d res | d skip] (fp16), dx (fp32), d of
// input_projection, dpre of every layer, tile column sums, dE per layer, dh of the MLP, wgrad partials (for the
// (m tiles, n tiles) of the backward's wgrads), dE summed
constexpr int kBwdRegions = 12;
void bwd_sizes(int L, int B, int T, int device, size_t (&sz)[kBwdRegions]) {
  const size_t F = static_cast<size_t>(B) * T;
  const size_t mtiles = (T + kConvRows - 1) / kConvRows;
  const size_t v[kBwdRegions] = {256,
                                 F * kM * 2,
                                 F * kC * 2,
                                 F * kN1 * 2,
                                 F * kC * 4,
                                 F * kC * 2,
                                 static_cast<size_t>(L) * F * kN1 * 2,
                                 static_cast<size_t>(L) * B * mtiles * kC * 4,
                                 static_cast<size_t>(L) * B * kC * 4,
                                 static_cast<size_t>(B) * 4 * kC * 4,
                                 wgrad_part_floats(static_cast<int>(F), {{8, 4}, {8, 1}, {4, 1}, {2, 1}}, device) * 4,
                                 static_cast<size_t>(B) * kC * 4};
  for (int i = 0; i < kBwdRegions; ++i) sz[i] = v[i];
}

// the forward's workspace: the fp32 residual stream and skip sum, and d_l(t) of every layer
size_t fwd_ws_bytes(int L, int B, int T) {
  const size_t F = static_cast<size_t>(B) * T;
  return 2 * align256(F * kC * 4) + align256(static_cast<size_t>(L) * B * kC * 4);
}

size_t ws_bytes(int L, int B, int T, int device) {
  size_t sz[kBwdRegions], n = 0;
  bwd_sizes(L, B, T, device, sz);
  for (size_t z : sz) n += align256(z);
  return std::max(n, fwd_ws_bytes(L, B, T));
}

int check_params(const dsx_diffnet_params* w, int L) {
  DSX_CHECK(w, DSX_E_INVALID, "null parameters");
  DSX_CHECK(w->in_w && w->in_b && w->mlp0_w && w->mlp0_b && w->mlp2_w && w->mlp2_b && w->skip_w && w->skip_b &&
                w->fin_w && w->fin_b && w->dil_w && w->dil_b && w->dif_w && w->dif_b && w->cond_w && w->cond_b &&
                w->out_w && w->out_b,
            DSX_E_INVALID, "a parameter pointer is NULL");
  for (int l = 0; l < L; ++l)
    DSX_CHECK(w->dil_w[l] && w->dil_b[l] && w->dif_w[l] && w->dif_b[l] && w->cond_w[l] && w->cond_b[l] && w->out_w[l] &&
                  w->out_b[l],
              DSX_E_INVALID, "a parameter pointer of residual layer %d is NULL", l);
  return DSX_OK;
}

int check_geom(int B, int T) {
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(B <= 65535, DSX_E_INVALID, "B = %d is above the 65535 utterances the launch grid holds", B);
  DSX_CHECK(static_cast<long long>(B) * T <= (1ll << 24), DSX_E_INVALID, "B * T = %lld frames is above 2^24",
            static_cast<long long>(B) * T);
  return DSX_OK;
}

// the d_cond GEMM addresses every layer's dpre with one int frame index
int check_frames(int L, int B, int T) {
  DSX_CHECK(static_cast<long long>(L) * B * T < (1ll << 26), DSX_E_INVALID,
            "residual_layers * B * T = %lld is above 2^26", static_cast<long long>(L) * B * T);
  return DSX_OK;
}

}  // namespace
}  // namespace dsx

using namespace dsx;

extern "C" {

int dsx_train_create(int device, const dsx_train_config* c, dsx_train** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_CHECK(c, DSX_E_INVALID, "config is NULL");
  DSX_CHECK(c->M == kM && c->C == kC && c->H == kH, DSX_E_INVALID,
            "unsupported DiffNet shape M=%d C=%d H=%d: the training step runs M = 80, C = H = 256", c->M, c->C, c->H);
  DSX_CHECK(c->L >= 1 && c->L <= 1024, DSX_E_INVALID, "unsupported residual_layers %d: 1..1024", c->L);
  DSX_CHECK(c->dilation_cycle >= 1 && c->dilation_cycle <= 24, DSX_E_INVALID,
            "unsupported dilation_cycle_length %d: 1..24", c->dilation_cycle);
  DSX_TRY(select_sm90_device(device, "DiffNet training step"));
  DSX_CUDA(cudaFuncSetAttribute(k_train_gemm<kNT>, cudaFuncAttributeMaxDynamicSharedMemorySize, conv_smem<kNT>()));
  DSX_CUDA(cudaFuncSetAttribute(k_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmem));
  dsx_train* h = new dsx_train();
  h->device = device;
  h->L = c->L;
  h->cycle = c->dilation_cycle;
  const int L = c->L;
  auto fail = [&](int rc) {
    dsx_train_destroy(h);
    return rc;
  };
  int rc = DSX_OK;
  h->dil.resize(L);
  h->cnd.resize(L);
  h->out.resize(L);
  h->out_t.resize(L);
  h->dil_t.resize(L);
  if ((rc = gemm_alloc(h->mem, h->in, kM, kC, 1)) || (rc = gemm_alloc(h->mem, h->skip, kC, kC, 1)) ||
      (rc = gemm_alloc(h->mem, h->fin, kC, kM, 1)) || (rc = gemm_alloc(h->mem, h->skip_t, kC, kC, 1)) ||
      (rc = gemm_alloc(h->mem, h->fin_t, kM, kC, 1)) || (rc = gemm_alloc(h->mem, h->cond_t, kN1, kH, L)))
    return fail(rc);
  for (int l = 0; l < L; ++l) {
    const int d = 1 << (l % c->dilation_cycle);
    if ((rc = gemm_alloc(h->mem, h->dil[l], kC, kN1, 3)) || (rc = gemm_alloc(h->mem, h->cnd[l], kH, kN1, 1)) ||
        (rc = gemm_alloc(h->mem, h->out[l], kC, kN1, 1)) || (rc = gemm_alloc(h->mem, h->out_t[l], kN1, kC, 1)) ||
        (rc = gemm_alloc(h->mem, h->dil_t[l], kN1, kC, 3)))
      return fail(rc);
    h->dil[l].tap0 = -d;
    h->dil[l].tstep = d;
    h->dil_t[l].tap0 = d;      // dx[m] = sum_j W_j^T dpre[m + (1 - j) d]
    h->dil_t[l].tstep = -d;
  }
  if ((rc = h->mem.alloc(&h->zeros, kNT * sizeof(float)))) return fail(rc);
  *out = h;
  return DSX_OK;
}

void dsx_train_destroy(dsx_train* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  h->mem.free_all();
  delete h;
}

int dsx_train_tape_bytes(dsx_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  DSX_TRY(check_geom(B, T));
  DSX_TRY(check_frames(h->L, B, T));
  *out = tape_carve(h->L, B, T, nullptr, nullptr);
  return DSX_OK;
}

int dsx_train_workspace_bytes(dsx_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  DSX_TRY(check_geom(B, T));
  DSX_TRY(check_frames(h->L, B, T));
  *out = ws_bytes(h->L, B, T, h->device);
  return DSX_OK;
}

int dsx_train_forward(dsx_train* h, const dsx_diffnet_params* w, const float* spec, dsx_strides ss, const int64_t* t,
                      const float* cond, dsx_strides cs, int B, int T, void* tape, size_t tape_bytes, void* workspace,
                      size_t workspace_bytes, float* eps, void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_TRY(check_geom(B, T));
  const int L = h->L;
  DSX_TRY(check_frames(L, B, T));
  DSX_TRY(check_params(w, L));
  DSX_CHECK(spec && t && cond && tape && eps, DSX_E_INVALID, "spec, t, cond, tape and eps must not be NULL");
  const size_t need = tape_carve(L, B, T, nullptr, nullptr);
  DSX_CHECK(tape_bytes >= need, DSX_E_INVALID, "tape of %zu bytes is below the %zu this (B, T) needs", tape_bytes, need);
  DSX_CHECK(workspace, DSX_E_INVALID, "workspace must not be NULL");
  const size_t wneed = ws_bytes(L, B, T, h->device);
  DSX_CHECK(workspace_bytes >= wneed, DSX_E_INVALID, "workspace of %zu bytes is below the %zu this (B, T) needs",
            workspace_bytes, wneed);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t F = static_cast<size_t>(B) * T;
  Tape tp;
  tape_carve(L, B, T, static_cast<uint8_t*>(tape), &tp);

  // round-to-nearest fp16 packs of this step's weights, and the transposed packs of the backward
  DSX_TRY(pack(h->in, PackArgs{w->in_w, nullptr, w->in_b, kM, kC, kC, 1, 1, 0}, s));
  DSX_TRY(pack(h->skip, PackArgs{w->skip_w, nullptr, w->skip_b, kC, kC, kC, 1, 1, 0}, s));
  DSX_TRY(pack(h->fin, PackArgs{w->fin_w, nullptr, w->fin_b, kC, kM, kM, 1, 1, 0}, s));
  ConvGemm st = h->skip_t, ft = h->fin_t;
  st.b = ft.b = h->zeros;
  DSX_TRY(pack(st, PackArgs{w->skip_w, nullptr, nullptr, kC, kC, kC, 1, 1, 1}, s));
  DSX_TRY(pack(ft, PackArgs{w->fin_w, nullptr, nullptr, kM, kC, kC, 1, 1, 1}, s));
  for (int l = 0; l < L; ++l) {
    k_pack_gate<<<pack_blocks(h->dil[l]), 256, 0, s>>>(h->dil[l], w->dil_w[l], 3, w->dil_b[l], w->cond_b[l]);
    DSX_TRY(launch_check("k_pack_gate"));
    k_pack_gate<<<pack_blocks(h->cnd[l]), 256, 0, s>>>(h->cnd[l], w->cond_w[l], 1, nullptr, nullptr);
    DSX_TRY(launch_check("k_pack_gate"));
    DSX_TRY(pack(h->out[l], PackArgs{w->out_w[l], nullptr, w->out_b[l], kC, kN1, kN1, 1, 1, 0}, s));
    ConvGemm ot = h->out_t[l], dt = h->dil_t[l], ct = h->cond_t;
    ot.b = dt.b = ct.b = h->zeros;
    DSX_TRY(pack(ot, PackArgs{w->out_w[l], nullptr, nullptr, kN1, kC, kC, 1, 1, 1}, s));
    DSX_TRY(pack(dt, PackArgs{w->dil_w[l], nullptr, nullptr, kN1, kC, kC, 3, 1, 1}, s));
    // layer l's K chunks of the one d_cond GEMM: a one-tap view at chunk 8 l
    ct.taps = 1;
    ct.kc = kN1 / 64;
    ct.w = h->cond_t.w + static_cast<size_t>(l) * ct.kc * kNT * 64;
    DSX_TRY(pack(ct, PackArgs{w->cond_w[l], nullptr, nullptr, kN1, kH, kH, 1, 1, 1}, s));
  }

  // inputs to fp16 frames-major, step embedding (with the MLP's activations saved) and d_l(t) of every layer
  const unsigned fb = static_cast<unsigned>((F * 32 + 255) / 256);
  k_pack_frames<<<fb, 256, 0, s>>>(spec, ss, B, T, kM, tp.spec);
  DSX_TRY(launch_check("k_pack_frames"));
  k_pack_frames<<<fb, 256, 0, s>>>(cond, cs, B, T, kH, tp.cond);
  DSX_TRY(launch_check("k_pack_frames"));
  ModelDev m{};
  m.C = kC;
  m.mlp0_w = w->mlp0_w;
  m.mlp0_b = w->mlp0_b;
  m.mlp2_w = w->mlp2_w;
  m.mlp2_b = w->mlp2_b;
  DSX_TRY(launch_embed_saved(m, t, B, tp.emb, tp.save, s));

  Bump fws{static_cast<uint8_t*>(workspace)};
  float* X = fws.take<float>(F * kC * 4);
  float* SKIP = fws.take<float>(F * kC * 4);
  float* D = fws.take<float>(static_cast<size_t>(L) * B * kC * 4);
  const unsigned db = static_cast<unsigned>((B * kC * 32 + 255) / 256);
  for (int l = 0; l < L; ++l) {
    k_dproj<<<db, 256, 0, s>>>(w->dif_w[l], w->dif_b[l], tp.emb, B, D + static_cast<size_t>(l) * B * kC);
    DSX_TRY(launch_check("k_dproj"));
  }

  GemmArgs a{};
  a.B = B;
  a.T = T;
  a.L = L;
  a.rsqrtL = 1.f / sqrtf(static_cast<float>(L));
  a.X = X;
  a.SKIP = SKIP;
  a.mode = F_IN;
  a.g = h->in;
  a.x = tp.spec;
  a.D = D;
  a.o16 = tp.y[0];
  a.o16b = tp.x0;
  DSX_TRY(run_gemm(a, B, T, s));
  for (int l = 0; l < L; ++l) {
    a.layer = l;
    a.mode = F_GATE;
    a.g = h->dil[l];
    a.x = tp.y[l];
    a.g2 = h->cnd[l];
    a.x2 = tp.cond;
    a.o16 = tp.sg[l];
    a.o16b = tp.z[l];
    DSX_TRY(run_gemm(a, B, T, s));
    a.mode = F_OUT;
    a.g = h->out[l];
    a.x = tp.z[l];
    a.D = l + 1 < L ? D + static_cast<size_t>(l + 1) * B * kC : nullptr;
    a.o16 = l + 1 < L ? tp.y[l + 1] : nullptr;
    a.o16b = tp.s16;
    DSX_TRY(run_gemm(a, B, T, s));
  }
  a.mode = F_SKIP;
  a.g = h->skip;
  a.x = tp.s16;
  a.o16 = tp.h1;
  DSX_TRY(run_gemm(a, B, T, s));
  a.mode = F_FIN;
  a.g = h->fin;
  a.x = tp.h1;
  a.o32 = eps;
  return run_gemm(a, B, T, s);
}

int dsx_train_backward(dsx_train* h, const dsx_diffnet_params* w, const void* tape, const float* d_eps,
                       const dsx_diffnet_params* grads, float* d_cond, int B, int T, void* workspace,
                       size_t workspace_bytes, void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_TRY(check_geom(B, T));
  const int L = h->L;
  DSX_TRY(check_frames(L, B, T));
  DSX_TRY(check_params(w, L));
  DSX_TRY(check_params(grads, L));
  DSX_CHECK(tape && d_eps && workspace, DSX_E_INVALID, "tape, d_eps and workspace must not be NULL");
  const size_t wneed = ws_bytes(L, B, T, h->device);
  DSX_CHECK(workspace_bytes >= wneed, DSX_E_INVALID, "workspace of %zu bytes is below the %zu this (B, T) needs",
            workspace_bytes, wneed);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t F = static_cast<size_t>(B) * T;
  const int mtiles = (T + kConvRows - 1) / kConvRows;
  Tape tp;
  tape_carve(L, B, T, static_cast<uint8_t*>(const_cast<void*>(tape)), &tp);

  size_t sizes[kBwdRegions];
  bwd_sizes(L, B, T, h->device, sizes);
  Bump bump{static_cast<uint8_t*>(workspace)};
  unsigned* amax = bump.take<unsigned>(sizes[0]);
  float* scal = reinterpret_cast<float*>(amax + 4);
  __half* G0 = bump.take<__half>(sizes[1]);
  __half* DH = bump.take<__half>(sizes[2]);
  __half* GO = bump.take<__half>(sizes[3]);
  float* DX = bump.take<float>(sizes[4]);
  __half* DIN = bump.take<__half>(sizes[5]);
  __half* DPRE = bump.take<__half>(sizes[6]);
  float* DDP = bump.take<float>(sizes[7]);
  float* DE = bump.take<float>(sizes[8]);
  float* DHM = bump.take<float>(sizes[9]);
  float* PART = bump.take<float>(sizes[10]);
  float* DESUM = bump.take<float>(sizes[11]);

  DSX_CUDA(cudaMemsetAsync(GO, 0, F * kN1 * 2, s));   // d res of the last layer is 0
  const size_t ne = F * kM;
  DSX_TRY(run_scale(d_eps, ne, amax, scal, nullptr, B, T, s));
  k_grad_in<<<static_cast<unsigned>(std::min<size_t>((ne + 255) / 256, 4096)), 256, 0, s>>>(d_eps, scal, B, T, G0);
  DSX_TRY(launch_check("k_grad_in"));
  const float* inv_s = scal + 1;

  // wgrad of one GEMM into grads
  auto wgrad = [&](const __half* A, int lda, int am, int ntiles, WgradArgs t, const WgradDst& o) -> int {
    t.a = A;
    t.lda = lda;
    t.am = am;
    t.F = static_cast<int>(F);
    t.T = T;
    return run_wgrad(t, ntiles, o, PART, scal, h->device, s);
  };
  auto plain = [](int ldd, float* dst, float* db) {   // dst[m * ldd + c]
    WgradDst o{};
    o.dst[0] = dst;
    o.ms[0] = ldd;
    o.cs[0] = 1;
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

  GemmArgs a{};
  a.B = B;
  a.T = T;
  a.L = L;
  a.rsqrtL = 1.f / sqrtf(static_cast<float>(L));
  a.inv_s = inv_s;
  // head: output_projection, ReLU, skip_projection
  a.mode = B_FIN;
  a.g = h->fin_t;
  a.x = G0;
  a.aux = tp.h1;
  a.o16 = DH;
  DSX_TRY(run_gemm(a, B, T, s));
  DSX_TRY(wgrad(G0, kM, kM, 1, single(tp.h1, kC, kC),
                plain(kC, const_cast<float*>(grads->fin_w), const_cast<float*>(grads->fin_b))));
  a.mode = B_SKIP;
  a.g = h->skip_t;
  a.x = DH;
  a.o16 = GO;
  DSX_TRY(run_gemm(a, B, T, s));
  DSX_TRY(wgrad(DH, kC, kC, 1, single(tp.s16, kC, kC),
                plain(kC, const_cast<float*>(grads->skip_w), const_cast<float*>(grads->skip_b))));
  for (int l = L - 1; l >= 0; --l) {
    const int d = 1 << (l % h->cycle);
    __half* dpre = DPRE + static_cast<size_t>(l) * F * kN1;
    a.layer = l;
    a.mode = B_OUT;
    a.g = h->out_t[l];
    a.x = GO;
    a.aux = tp.sg[l];
    a.o16 = dpre;
    DSX_TRY(run_gemm(a, B, T, s));
    DSX_TRY(wgrad(GO, kN1, kN1, 1, single(tp.z[l], kC, kC),
                  plain(kC, const_cast<float*>(grads->out_w[l]), const_cast<float*>(grads->out_b[l]))));
    a.mode = B_DIL;
    a.g = h->dil_t[l];
    a.x = dpre;
    a.X = DX;
    a.aux = tp.x0;
    a.o16 = GO;
    a.o16b = DIN;
    a.o32 = DDP + static_cast<size_t>(l) * B * mtiles * kC;
    DSX_TRY(run_gemm(a, B, T, s));
    // columns [tap 0 | tap 1 | tap 2 | cond] -> dil_w [m][c][tap], cond_w [m][h]
    WgradArgs t4{};
    WgradDst o{};
    for (int j = 0; j < 4; ++j) {
      t4.b[j] = j < 3 ? tp.y[l] : tp.cond;
      t4.ldb[j] = kC;
      t4.bn[j] = kC;
      t4.shift[j] = j < 3 ? (j - 1) * d : 0;
      o.dst[j] = j < 3 ? const_cast<float*>(grads->dil_w[l]) + j : const_cast<float*>(grads->cond_w[l]);
      o.ms[j] = j < 3 ? 3 * kC : kH;
      o.cs[j] = j < 3 ? 3 : 1;
    }
    o.db = const_cast<float*>(grads->dil_b[l]);
    o.db2 = const_cast<float*>(grads->cond_b[l]);
    DSX_TRY(wgrad(dpre, kN1, kN1, 4, t4, o));
    k_dif_grad<<<kC + B, kC, 0, s>>>(DDP + static_cast<size_t>(l) * B * mtiles * kC, mtiles, B, tp.emb, w->dif_w[l], scal,
                                     const_cast<float*>(grads->dif_w[l]), const_cast<float*>(grads->dif_b[l]),
                                     DE + static_cast<size_t>(l) * B * kC);
    DSX_TRY(launch_check("k_dif_grad"));
  }
  // input_projection (its ReLU mask is in DIN), the MLP, and d_cond
  DSX_TRY(wgrad(DIN, kC, kC, 1, single(tp.spec, kM, kM),
                plain(kM, const_cast<float*>(grads->in_w), const_cast<float*>(grads->in_b))));
  k_de_sum<<<(B * kC + 255) / 256, 256, 0, s>>>(DE, L, B, DESUM);
  DSX_TRY(launch_check("k_de_sum"));
  DSX_TRY(run_mlp_grad(DESUM, B, kC, tp.save, w->mlp2_w, scal, const_cast<float*>(grads->mlp2_w),
                       const_cast<float*>(grads->mlp2_b), DHM, const_cast<float*>(grads->mlp0_w),
                       const_cast<float*>(grads->mlp0_b), s));
  if (d_cond) {
    a.mode = B_COND;
    a.g = h->cond_t;
    a.g.tap0 = 0;
    a.g.tstep = static_cast<int>(F);
    a.x = DPRE;
    a.o32 = d_cond;
    DSX_TRY(run_gemm(a, B, T, s));
  }
  return DSX_OK;
}

}  // extern "C"
