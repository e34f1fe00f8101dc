// Pitch extractor on sm_90a: mel [B, T, 80] -> pitch_pred [B, T, 2] and the denormalised f0 [B, T]
// (modules/fastspeech/pe.py:119-149: Prenet, ConvStacks with GroupNorm, PitchPredictor, utils/pitch_utils.py:denorm_f0).
//
// Every conv and linear is one implicit GEMM on wgmma (k_pe_conv, on the core of dsx_conv.cuh) over frames-major fp16
// [B][T][C]: tap j reads frame m + tap0 + j, zero outside [0, T).  That one rule is the prenet's zero padding (tap0 = -2),
// the PitchPredictor's ConstantPad1d 'SAME' (tap0 = -(k-1)/2) and 'LEFT' (tap0 = -(k-1)), and a linear (one tap).  A CTA
// covers 64 frames x ALL output channels (N <= 256), so a row's normalisation and the head's P -> 2 linear run in the
// epilogue from registers: one warpgroup up to N = 128; at N = 256 two warpgroups share the A tile, each with its 128
// columns (m64n128) and a row reduction through shared memory.  Epilogues by mode:
//   PE_PRENET  bias, ReLU, BatchNorm (eval: per-channel scale and shift packed at load), padding mask -> fp16
//   PE_LINEAR  bias, optional padding mask -> fp32 and / or fp16
//   PE_GN      bias -> fp32 pre-norm values, plus per-tile, per-16-channel-group (count, mean, M2) partials
//   PE_LN      bias, ReLU, LayerNorm over the row (two-pass, reduced over the accumulator quad) -> fp16
//   PE_HEAD    PE_LN, then Linear(P, 2) from registers -> pitch_pred, and f0 with the uv and padding rules
//   PE_DUR     PE_LN, then the DurationPredictor's Linear(P, 1) from registers, * !mask -> xs, and out2dur -> int64 dur
// GroupNorm statistics span a whole utterance, so k_pe_gn merges the tile partials in a fixed order (Chan's formula, no
// atomics: deterministic) and applies x += relu(gn(y)).  The position embedding is dsx_posemb.cuh's: a scan per utterance
// (k_pos_scan), then k_pos_add adds alpha * table[pos] with the table evaluated in fp32 on the fly.
#include <math.h>
#include <stdio.h>

#include <algorithm>

#include "dsx_conv.cuh"
#include "dsx_internal.h"
#include "dsx_posemb.cuh"
#include "dsx_ptx.cuh"

namespace dsx {
namespace {

constexpr int kPeMel = 80;
constexpr int kPePrenetLayers = 3, kPePredLayers = 5, kPeEncKernel = 5, kPePrenetKernel = 5;
constexpr int kPeMaxConvLayers = 16;
constexpr float kBnEps = 1e-5f, kGnEps = 1e-5f, kLnEps = 1e-12f;

enum { PE_PRENET = 0, PE_LINEAR = 1, PE_GN = 2, PE_LN = 3, PE_HEAD = 4, PE_DUR = 5 };
enum { PE_MASK = 1, PE_OUT32 = 2, PE_OUT16 = 4 };

// one conv or linear: its GEMM (one column tile) and the per-channel affine of its epilogue
struct PePacked : ConvGemm {
  float* s = nullptr;          // per-channel scale (BatchNorm, GroupNorm / LayerNorm weight) [n], or null
  float* t = nullptr;          // per-channel shift [n], or null
};

struct PeConvArgs {
  ConvGemm g;
  const __half* x;             // [B][T][g.cin]
  int T, mode, flags;
  const float* scale;          // PE_PRENET: BN scale; PE_LN / PE_HEAD: LayerNorm weight
  const float* shift;          // PE_PRENET: BN shift; PE_LN / PE_HEAD: LayerNorm bias
  const uint8_t* pad;          // [B][T] 1 = padding frame
  float* o32;                  // [B][T][n]
  __half* o16;                 // [B][T][n]
  float* stats;                // PE_GN: [B][mtiles][n / 16][3]
  int mtiles;
  const float* hw;             // PE_HEAD: linear.weight [2][n] and bias [2]
  const float* hb;
  float* pitch;                // [B][T][2] or null
  float* f0;                   // [B][T] or null
  int pitch_norm, use_uv;
  float f0_mean, f0_std;
  int64_t* dur;                // PE_DUR: [B][T] or null (xs goes to o32 [B][T])
  float offset;
  // the training form (k_pe_conv<NT, true>, PE_LN and PE_DUR): the LayerNorm input (bias + ReLU) -> r32 [B][T][n], the
  // LayerNorm output * dropout(drop) before * !mask, and PE_DUR's head input (that, * !mask) -> h32 [B][T][n]
  float* r32;
  float* h32;
  Fs2Drop drop;
};

template <int NT>
struct PeShape {
  static constexpr int WG = NT > 128 ? 2 : 1;      // warpgroups per CTA; each owns NH columns of the same 64 rows
  static constexpr int NH = NT / WG;
};

template <int NT, bool TRAIN = false>
__global__ void __launch_bounds__(128 * PeShape<NT>::WG) k_pe_conv(const PeConvArgs p) {
  constexpr int NH = PeShape<NT>::NH, WG = PeShape<NT>::WG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ float red[4 * WG][16];
  __shared__ float gmean[16];
  __shared__ float xrow[WG][kConvRows];   // per-warpgroup row partials of the LayerNorm / head reductions
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, b = blockIdx.y, m0 = blockIdx.x * kConvRows;
  const int T = p.T;

  float acc[NH / 2];
  conv_k_loop<NT, WG>(p.g, p.x, T, T, b, m0, 0, smem, acc);

  // ---- epilogue: thread wtid holds rows r0 = acc_row(wtid, 0) (e & 2 == 0) and r0 + 8 (e & 2 != 0) ----
  const int n = p.g.n, c0 = wg * NH;
  const int r0 = acc_row(wtid, 0);
  const int mrow[2] = {m0 + r0, m0 + r0 + 8};
  const size_t rbase = static_cast<size_t>(b) * T;
  // sum of the two rows' values over all n columns: the quad, then (two warpgroups) both halves in a fixed order
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
  // bias (+ ReLU) in place; columns >= n stay 0 (zero weights and bias)
#pragma unroll
  for (int e = 0; e < NH / 2; ++e) {
    const int col = c0 + acc_col(wtid, e);
    float v = col < n ? acc[e] + __ldg(p.g.b + col) : 0.f;
    if (p.mode == PE_PRENET || p.mode == PE_LN || p.mode == PE_HEAD || p.mode == PE_DUR) v = fmaxf(v, 0.f);
    acc[e] = v;
  }
  if constexpr (TRAIN) {
#pragma unroll
    for (int e = 0; e < NH / 2; e += 2) {
      const int col = c0 + acc_col(wtid, e), m = mrow[(e >> 1) & 1];
      if (col < n && m < T) *reinterpret_cast<float2*>(p.r32 + (rbase + m) * n + col) = make_float2(acc[e], acc[e + 1]);
    }
  }

  if (p.mode == PE_GN) {
    // per 16-channel group: count, mean and M2 over the tile's valid rows, two passes, fixed reduction order.  Local
    // group gl of this warpgroup (global group c0 / 16 + gl) is elements e in [8 gl, 8 gl + 8).
    const int rows = min(kConvRows, T - m0);
    const bool ok0 = r0 < rows, ok1 = r0 + 8 < rows;
    const int warp = tid >> 5, lane = tid & 31;
    const int groups = n / 16;
#pragma unroll
    for (int pass = 0; pass < 2; ++pass) {
#pragma unroll
      for (int gl = 0; gl < NH / 16; ++gl) {
        const int g = c0 / 16 + gl;
        float sum = 0.f;
        const float mu = pass ? gmean[g] : 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const bool ok = (i & 2) ? ok1 : ok0;
          const float d = acc[8 * gl + i] - mu;
          sum += ok ? (pass ? d * d : d) : 0.f;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) red[warp][g] = sum;
      }
      __syncthreads();
      if (tid < groups) {
        const int w0 = (tid / (NH / 16)) * 4;
        const float tot = ((red[w0][tid] + red[w0 + 1][tid]) + red[w0 + 2][tid]) + red[w0 + 3][tid];
        const float cnt = static_cast<float>(rows * 16);
        if (pass == 0) {
          gmean[tid] = tot / cnt;
        } else {
          float* st = p.stats + ((static_cast<size_t>(b) * p.mtiles + blockIdx.x) * groups + tid) * 3;
          st[0] = cnt;
          st[1] = gmean[tid];
          st[2] = tot;
        }
      }
      __syncthreads();
    }
  }

  if (p.mode == PE_LN || p.mode == PE_HEAD || p.mode == PE_DUR) {
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
    const float rstd0 = 1.f / sqrtf(q[0] * inv_n + kLnEps), rstd1 = 1.f / sqrtf(q[1] * inv_n + kLnEps);
#pragma unroll
    for (int e = 0; e < NH / 2; ++e) {
      const int col = c0 + acc_col(wtid, e);
      const bool hi = e & 2;
      acc[e] = col < n ? (acc[e] - (hi ? mean1 : mean0)) * (hi ? rstd1 : rstd0) * __ldg(p.scale + col) + __ldg(p.shift + col)
                       : 0.f;
    }
    if constexpr (TRAIN) {
#pragma unroll
      for (int e = 0; e < NH / 2; e += 2) {
        const int col = c0 + acc_col(wtid, e), m = mrow[(e >> 1) & 1];
        const float2 ds = dropout_scale2(p.drop, rbase + m, col);
        acc[e] *= ds.x;
        acc[e + 1] *= ds.y;
        if (p.mode == PE_DUR && col < n && m < T) {
          if (p.pad[rbase + m]) acc[e] = acc[e + 1] = 0.f;
          *reinterpret_cast<float2*>(p.h32 + (rbase + m) * n + col) = make_float2(acc[e], acc[e + 1]);
        }
      }
    }
  }

  if (p.mode == PE_HEAD) {
    float o[2][2] = {{0.f, 0.f}, {0.f, 0.f}};   // [row][output]
#pragma unroll
    for (int e = 0; e < NH / 2; ++e) {
      const int col = c0 + acc_col(wtid, e);
      if (col >= n) continue;
      const int r = (e >> 1) & 1;
      o[r][0] = fmaf(acc[e], __ldg(p.hw + col), o[r][0]);
      o[r][1] = fmaf(acc[e], __ldg(p.hw + n + col), o[r][1]);
    }
    row_sum(o[0][0], o[1][0]);
    row_sum(o[0][1], o[1][1]);
    if (wg != 0 || (wtid & 3) != 0) return;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float p0 = o[r][0] + __ldg(p.hb), p1 = o[r][1] + __ldg(p.hb + 1);
      const int m = mrow[r];
      if (m >= T) continue;
      const size_t idx = rbase + m;
      if (p.pitch) *reinterpret_cast<float2*>(p.pitch + idx * 2) = make_float2(p0, p1);
      if (p.f0) {   // denorm_f0 (utils/pitch_utils.py:63-76)
        float f = p.pitch_norm == 1 ? p0 * p.f0_std + p.f0_mean : exp2f(p0);
        if (p.use_uv && p1 > 0.f) f = 0.f;
        if (p.pad[idx]) f = 0.f;
        p.f0[idx] = f;
      }
    }
    return;
  }

  if (p.mode == PE_DUR) {
    // DurationPredictor (tts_modules.py:113-129): xs = Linear(LN(x) * !mask) * !mask, dur = clamp(round(exp(xs) - offset),
    // 0) with round half to even.  A padding row is 0 in both.
    float o[2] = {0.f, 0.f};
#pragma unroll
    for (int e = 0; e < NH / 2; ++e) {
      const int col = c0 + acc_col(wtid, e);
      if (col < n) o[(e >> 1) & 1] = fmaf(acc[e], __ldg(p.hw + col), o[(e >> 1) & 1]);
    }
    row_sum(o[0], o[1]);
    if (wg != 0 || (wtid & 3) != 0) return;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int m = mrow[r];
      if (m >= T) continue;
      const size_t idx = rbase + m;
      const float x = p.pad[idx] ? 0.f : o[r] + __ldg(p.hb);
      p.o32[idx] = x;
      if (p.dur) p.dur[idx] = __float2ll_rz(fmaxf(rintf(expf(x) - p.offset), 0.f));
    }
    return;
  }

  // element-wise tail: PE_PRENET (BN affine + mask), PE_LINEAR, PE_GN (pre-norm values), PE_LN -> stores
#pragma unroll
  for (int e = 0; e < NH / 2; e += 2) {
    const int col = c0 + acc_col(wtid, e), m = mrow[(e >> 1) & 1];
    if (col >= n || m >= T) continue;
    const size_t idx = (rbase + m) * n + col;
    float v0 = acc[e], v1 = acc[e + 1];
    if (p.mode == PE_PRENET) {
      v0 = fmaf(v0, __ldg(p.scale + col), __ldg(p.shift + col));
      v1 = fmaf(v1, __ldg(p.scale + col + 1), __ldg(p.shift + col + 1));
    }
    if ((p.flags & PE_MASK) && p.pad[rbase + m]) v0 = v1 = 0.f;
    if (p.flags & PE_OUT32) *reinterpret_cast<float2*>(p.o32 + idx) = make_float2(v0, v1);
    if (p.flags & PE_OUT16) *reinterpret_cast<__half2*>(p.o16 + idx) = __floats2half2_rn(v0, v1);
  }
}

// ---- operand pack --------------------------------------------------------------------------------
// mel logically [B, T, 80] (any strides: b, c = bin, t) -> fp16 [B][T][80] and pad[b][t] = all 80 bins exactly 0
// (pe.py:29 mel.abs().sum(-1) == 0, decided on the fp32 values).  One warp per frame.
__global__ void k_pe_pack_mel(const float* mel, dsx_strides ms, int B, int T, __half* out, uint8_t* pad) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * T) return;
  const int b = warp / T, t = warp - b * T;
  const float* src = mel + b * ms.b + t * ms.t;
  bool nz = false;
  for (int c = lane; c < kPeMel; c += 32) {
    const float v = src[c * ms.c];
    nz |= v != 0.f;
    out[static_cast<size_t>(warp) * kPeMel + c] = __float2half_rn(v);
  }
  const unsigned any = __ballot_sync(0xffffffffu, nz);
  if (lane == 0) pad[warp] = any ? 0 : 1;
}

// ---- GroupNorm ---------------------------------------------------------------------------------
// Merge the per-tile (count, mean, M2) of utterance b in tile order (Chan et al.), then x += relu(gn(y)) over kGnRows
// frames per block: writes the fp32 residual and the fp16 operand of the next conv (pe.py:107-109, ConvBlock.forward).
constexpr int kGnRows = 32;
__global__ void __launch_bounds__(256) k_pe_gn(const float* y, const float* stats, int mtiles, const float* gw,
                                               const float* gb, int T, int n, float* x, __half* x16) {
  __shared__ float mean_s[16], rstd_s[16];
  const int b = blockIdx.y, groups = n / 16, tid = threadIdx.x;
  if (tid < groups) {
    const float* st = stats + static_cast<size_t>(b) * mtiles * groups * 3 + tid * 3;
    float na = st[0], ma = st[1], m2 = st[2];
    for (int i = 1; i < mtiles; ++i) {
      const float* q = st + static_cast<size_t>(i) * groups * 3;
      const float nb = q[0], nn = na + nb, d = q[1] - ma;
      ma += d * (nb / nn);
      m2 += q[2] + d * d * (na * nb / nn);
      na = nn;
    }
    mean_s[tid] = ma;
    rstd_s[tid] = 1.f / sqrtf(m2 / na + kGnEps);
  }
  __syncthreads();
  const int t0 = blockIdx.x * kGnRows, t1 = min(T, t0 + kGnRows);
  const size_t base = (static_cast<size_t>(b) * T + t0) * n, cnt = static_cast<size_t>(t1 - t0) * n;
  for (size_t i = tid; i < cnt; i += blockDim.x) {
    const int c = static_cast<int>(i % n), g = c >> 4;
    const float v = (y[base + i] - mean_s[g]) * rstd_s[g] * gw[c] + gb[c];
    const float r = x[base + i] + fmaxf(v, 0.f);
    x[base + i] = r;
    x16[base + i] = __float2half_rn(r);
  }
}

// BatchNorm1d in eval mode as y = x * scale + shift: scale = w / sqrt(var + eps), shift = b - mean * scale
__global__ void k_pe_bn(const float* w, const float* b, const float* mean, const float* var, int n, float* scale,
                        float* shift) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float s = w[i] / sqrtf(var[i] + kBnEps);
  scale[i] = s;
  shift[i] = b[i] - mean[i] * s;
}

}  // namespace
}  // namespace dsx

using namespace dsx;

struct dsx_pe {
  int device = 0;
  dsx_pe_config cfg{};
  int P = 0;
  bool loaded = false;
  PePacked prenet[kPePrenetLayers], prenet_out, enc_in, enc_out, pred[kPePredLayers];
  std::vector<PePacked> enc;
  float* head = nullptr;       // linear.weight [2][P], bias [2]
  float* alpha = nullptr;      // pos_embed_alpha [1]
  DevAllocs mem;               // the packs above
  GrowBuffer ws;               // workspace of a forward call
};

namespace {

void pe_free_model(dsx_pe* h) {
  h->mem.free_all();
  h->enc.clear();
  h->loaded = false;
}

int pe_copy(dsx_pe* h, float** dst, const float* src, int n, const char* what, cudaStream_t s) {
  DSX_CHECK(src, DSX_E_INVALID, "missing %s", what);
  DSX_TRY(h->mem.alloc(dst, static_cast<size_t>(n) * sizeof(float)));
  DSX_CUDA(cudaMemcpyAsync(*dst, src, static_cast<size_t>(n) * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return DSX_OK;
}

// pack one conv (k taps starting at tap0) or linear (k = 1, tap0 = 0) of cin -> n channels, all n in one column tile
int pe_pack(dsx_pe* h, PePacked& pc, const float* w, const float* b, int cin, int n, int k, int tap0, const char* what,
            cudaStream_t s) {
  DSX_CHECK(w && b, DSX_E_INVALID, "missing %s weight or bias", what);
  pc.cin = cin;
  pc.n = n;
  pc.taps = k;
  pc.tap0 = tap0;
  return conv_pack(h->mem, pc, 256, PackArgs{w, nullptr, b, cin, n, n, k, 1, 0}, s);
}

int pe_run(const PePacked& pc, PeConvArgs a, int B, cudaStream_t s) {
  a.g = pc;
  a.mtiles = (a.T + kConvRows - 1) / kConvRows;
  return conv_dispatch<256>(pc.nt, [&](auto c) {
    constexpr int NT = decltype(c)::value;
    k_pe_conv<NT><<<dim3(a.mtiles, B), 128 * PeShape<NT>::WG, conv_smem<NT>(), s>>>(a);
    return launch_check("k_pe_conv");
  });
}

int pe_validate(const dsx_pe_config* c) {
  DSX_CHECK(c, DSX_E_INVALID, "config is NULL");
  DSX_CHECK(c->n_mel_bins == kPeMel, DSX_E_INVALID, "n_mel_bins must be 80 (got %d)", c->n_mel_bins);
  DSX_CHECK(c->hidden >= 16 && c->hidden <= 256 && c->hidden % 16 == 0, DSX_E_INVALID,
            "hidden must be a multiple of 16 in [16, 256] (got %d)", c->hidden);
  DSX_CHECK(c->predictor_hidden >= 16 && c->predictor_hidden <= 256 && c->predictor_hidden % 16 == 0, DSX_E_INVALID,
            "predictor_hidden must be a multiple of 16 in [16, 256] (got %d)", c->predictor_hidden);
  DSX_CHECK(c->predictor_kernel >= 1 && c->predictor_kernel <= 31 && c->predictor_kernel % 2 == 1, DSX_E_INVALID,
            "predictor_kernel must be odd and in [1, 31] (got %d)", c->predictor_kernel);
  DSX_CHECK(c->conv_layers >= 0 && c->conv_layers <= kPeMaxConvLayers, DSX_E_INVALID,
            "conv_layers must be in [0, %d] (got %d)", kPeMaxConvLayers, c->conv_layers);
  DSX_CHECK(c->causal == 0 || c->causal == 1, DSX_E_INVALID, "causal must be 0 (SAME) or 1 (LEFT) (got %d)", c->causal);
  DSX_CHECK(c->pitch_norm == 0 || c->pitch_norm == 1, DSX_E_INVALID, "pitch_norm must be 0 (log) or 1 (standard) (got %d)",
            c->pitch_norm);
  DSX_CHECK(c->use_uv == 0 || c->use_uv == 1, DSX_E_INVALID, "use_uv must be 0 or 1 (got %d)", c->use_uv);
  DSX_CHECK(isfinite(c->f0_mean) && isfinite(c->f0_std), DSX_E_INVALID, "f0_mean and f0_std must be finite");
  return DSX_OK;
}

}  // namespace

extern "C" {

int dsx_pe_create(int device, const dsx_pe_config* cfg, dsx_pe** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_TRY(pe_validate(cfg));
  DSX_TRY(select_sm90_device(device, "pitch extractor"));
  DSX_TRY(conv_opt_in<256>([](auto c) { return k_pe_conv<decltype(c)::value>; }));
  dsx_pe* h = new dsx_pe();
  h->device = device;
  h->cfg = *cfg;
  h->P = cfg->predictor_hidden;
  *out = h;
  return DSX_OK;
}

void dsx_pe_destroy(dsx_pe* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  pe_free_model(h);
  h->ws.release();
  delete h;
}

int dsx_pe_load(dsx_pe* h, const dsx_pe_params* p, void* stream) {
  DSX_CHECK(h && p, DSX_E_INVALID, "null handle or params");
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const dsx_pe_config& c = h->cfg;
  const int H = c.hidden, P = h->P, L = c.conv_layers, k = c.predictor_kernel;
  DSX_CHECK(p->prenet_w && p->prenet_b && p->bn_w && p->bn_b && p->bn_mean && p->bn_var, DSX_E_INVALID,
            "missing per-layer prenet arrays");
  DSX_CHECK(p->pred_w && p->pred_b && p->ln_w && p->ln_b, DSX_E_INVALID, "missing per-layer pitch_predictor arrays");
  DSX_CHECK(L == 0 || (p->enc_w && p->enc_b && p->gn_w && p->gn_b), DSX_E_INVALID, "missing per-layer mel_encoder arrays");
  DSX_CUDA(cudaStreamSynchronize(s));   // the old packs may still be read by queued work
  pe_free_model(h);
  char what[64];
  for (int i = 0; i < kPePrenetLayers; ++i) {
    snprintf(what, sizeof what, "mel_prenet.layers.%d.0", i);
    PePacked& pc = h->prenet[i];
    DSX_TRY(pe_pack(h, pc, p->prenet_w[i], p->prenet_b[i], i ? H : kPeMel, H, kPePrenetKernel, -kPePrenetKernel / 2,
                    what, s));
    DSX_CHECK(p->bn_w[i] && p->bn_b[i] && p->bn_mean[i] && p->bn_var[i], DSX_E_INVALID, "missing mel_prenet.layers.%d.2", i);
    DSX_TRY(h->mem.alloc(&pc.s, H * sizeof(float)));
    DSX_TRY(h->mem.alloc(&pc.t, H * sizeof(float)));
    k_pe_bn<<<(H + 255) / 256, 256, 0, s>>>(p->bn_w[i], p->bn_b[i], p->bn_mean[i], p->bn_var[i], H, pc.s, pc.t);
    DSX_TRY(launch_check("k_pe_bn"));
  }
  DSX_TRY(pe_pack(h, h->prenet_out, p->prenet_out_w, p->prenet_out_b, H, H, 1, 0, "mel_prenet.out_proj", s));
  if (L > 0) {
    DSX_TRY(pe_pack(h, h->enc_in, p->enc_in_w, p->enc_in_b, H, H, 1, 0, "mel_encoder.in_proj", s));
    h->enc.resize(L);
    for (int i = 0; i < L; ++i) {
      snprintf(what, sizeof what, "mel_encoder.conv.%d", i);
      DSX_TRY(pe_pack(h, h->enc[i], p->enc_w[i], p->enc_b[i], H, H, kPeEncKernel, -kPeEncKernel / 2, what, s));
      DSX_TRY(pe_copy(h, &h->enc[i].s, p->gn_w[i], H, "mel_encoder GroupNorm weight", s));
      DSX_TRY(pe_copy(h, &h->enc[i].t, p->gn_b[i], H, "mel_encoder GroupNorm bias", s));
    }
    DSX_TRY(pe_pack(h, h->enc_out, p->enc_out_w, p->enc_out_b, H, H, 1, 0, "mel_encoder.out_proj", s));
  }
  const int tap0 = c.causal ? -(k - 1) : -(k - 1) / 2;   // ConstantPad1d LEFT (k - 1, 0) or SAME
  for (int i = 0; i < kPePredLayers; ++i) {
    snprintf(what, sizeof what, "pitch_predictor.conv.%d.1", i);
    PePacked& pc = h->pred[i];
    DSX_TRY(pe_pack(h, pc, p->pred_w[i], p->pred_b[i], i ? P : H, P, k, tap0, what, s));
    DSX_TRY(pe_copy(h, &pc.s, p->ln_w[i], P, "pitch_predictor LayerNorm weight", s));
    DSX_TRY(pe_copy(h, &pc.t, p->ln_b[i], P, "pitch_predictor LayerNorm bias", s));
  }
  DSX_CHECK(p->linear_w && p->linear_b && p->pos_embed_alpha, DSX_E_INVALID,
            "missing pitch_predictor.linear or pos_embed_alpha");
  DSX_TRY(h->mem.alloc(&h->head, (2 * P + 2) * sizeof(float)));
  DSX_CUDA(cudaMemcpyAsync(h->head, p->linear_w, 2 * P * sizeof(float), cudaMemcpyDeviceToDevice, s));
  DSX_CUDA(cudaMemcpyAsync(h->head + 2 * P, p->linear_b, 2 * sizeof(float), cudaMemcpyDeviceToDevice, s));
  DSX_TRY(pe_copy(h, &h->alpha, p->pos_embed_alpha, 1, "pos_embed_alpha", s));
  h->loaded = true;
  return DSX_OK;
}

int dsx_pe_forward(dsx_pe* h, const float* mel, dsx_strides ms, int B, int T, float* pitch_pred, float* f0,
                   void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(h->loaded, DSX_E_STATE, "dsx_pe_load has not been called");
  DSX_CHECK(mel, DSX_E_INVALID, "mel must not be NULL");
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(B <= 65535, DSX_E_INVALID, "B = %d utterances per call is above the 65535 the launch grid holds", B);
  const dsx_pe_config& c = h->cfg;
  const int H = c.hidden, P = h->P, L = c.conv_layers, C = std::max(H, P);
  DSX_CHECK(static_cast<long long>(B) * T * C < (1ll << 31), DSX_E_INVALID, "B * T = %lld frames is too large",
            static_cast<long long>(B) * T);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (!pitch_pred && !f0) return DSX_OK;

  // workspace: fp16 MEL / A0 / A1, fp32 X / Y, padding flags, positions, GroupNorm partials
  const size_t frames = static_cast<size_t>(B) * T;
  const int mtiles = (T + kConvRows - 1) / kConvRows;
  const size_t st_b = static_cast<size_t>(B) * mtiles * (H / 16) * 3 * 4;
  DSX_TRY(h->ws.reserve(align256(frames * kPeMel * 2) + 2 * align256(frames * C * 2) + 2 * align256(frames * H * 4) +
                        align256(frames) + align256(frames * 4) + align256(st_b), s));
  Bump ws{static_cast<uint8_t*>(h->ws.ptr)};
  __half* MEL = ws.take<__half>(frames * kPeMel * 2);
  __half* A[2] = {ws.take<__half>(frames * C * 2), ws.take<__half>(frames * C * 2)};
  float* X = ws.take<float>(frames * H * 4);
  float* Y = ws.take<float>(frames * H * 4);
  uint8_t* PAD = ws.take<uint8_t>(frames);
  int* POS = ws.take<int>(frames * 4);
  float* ST = ws.take<float>(st_b);

  k_pe_pack_mel<<<static_cast<unsigned>((frames * 32 + 255) / 256), 256, 0, s>>>(mel, ms, B, T, MEL, PAD);
  DSX_TRY(launch_check("k_pe_pack_mel"));

  PeConvArgs base{};
  base.T = T;
  base.pad = PAD;
  PeConvArgs a = base;
  // Prenet (pe.py:23-41): 3 x [conv k5, ReLU, BatchNorm, * nonpadding], then out_proj * nonpadding
  const __half* in = MEL;
  int cur = 0;
  for (int i = 0; i < kPePrenetLayers; ++i) {
    a = base;
    a.x = in;
    a.mode = PE_PRENET;
    a.flags = PE_MASK | PE_OUT16;
    a.scale = h->prenet[i].s;
    a.shift = h->prenet[i].t;
    a.o16 = A[cur];
    DSX_TRY(pe_run(h->prenet[i], a, B, s));
    in = A[cur];
    cur ^= 1;
  }
  a = base;
  a.x = in;
  a.mode = PE_LINEAR;
  a.flags = PE_MASK | (L > 0 ? PE_OUT16 : PE_OUT32);
  a.o16 = A[cur];
  a.o32 = X;
  DSX_TRY(pe_run(h->prenet_out, a, B, s));
  if (L > 0) {
    // ConvStacks (pe.py:98-116): in_proj, conv_layers x [x += relu(GroupNorm(conv(x)))], out_proj; no masking
    in = A[cur];
    cur ^= 1;
    a = base;
    a.x = in;
    a.mode = PE_LINEAR;
    a.flags = PE_OUT32 | PE_OUT16;
    a.o32 = X;
    a.o16 = A[cur];
    DSX_TRY(pe_run(h->enc_in, a, B, s));
    for (int i = 0; i < L; ++i) {
      a = base;
      a.x = A[cur];
      a.mode = PE_GN;
      a.flags = PE_OUT32;
      a.o32 = Y;
      a.stats = ST;
      DSX_TRY(pe_run(h->enc[i], a, B, s));
      k_pe_gn<<<dim3((T + kGnRows - 1) / kGnRows, B), 256, 0, s>>>(Y, ST, mtiles, h->enc[i].s, h->enc[i].t, T, H, X,
                                                                   A[cur ^ 1]);
      DSX_TRY(launch_check("k_pe_gn"));
      cur ^= 1;
    }
    a = base;
    a.x = A[cur];
    a.mode = PE_LINEAR;
    a.flags = PE_OUT32;
    a.o32 = Y;
    DSX_TRY(pe_run(h->enc_out, a, B, s));
  }
  // PitchPredictor (tts_modules.py:222-235): + alpha * position embedding, 4 x [conv, ReLU, LayerNorm], the head
  const float* xs = L > 0 ? Y : X;
  k_pos_scan<<<B, kScanThreads, 0, s>>>(xs, T, H, POS);
  DSX_TRY(launch_check("k_pos_scan"));
  const size_t ne = frames * H;
  k_pos_add<<<static_cast<unsigned>((ne + 255) / 256), 256, 0, s>>>(xs, POS, h->alpha, static_cast<int>(frames), H,
                                                                    pos_neg_emb(H), A[0]);
  DSX_TRY(launch_check("k_pos_add"));
  cur = 0;
  for (int i = 0; i < kPePredLayers; ++i) {
    a = base;
    a.x = A[cur];
    a.scale = h->pred[i].s;
    a.shift = h->pred[i].t;
    if (i + 1 < kPePredLayers) {
      a.mode = PE_LN;
      a.flags = PE_OUT16;
      a.o16 = A[cur ^ 1];
    } else {
      a.mode = PE_HEAD;
      a.hw = h->head;
      a.hb = h->head + 2 * P;
      a.pitch = pitch_pred;
      a.f0 = f0;
      a.pitch_norm = c.pitch_norm;
      a.use_uv = c.use_uv;
      a.f0_mean = c.f0_mean;
      a.f0_std = c.f0_std;
    }
    DSX_TRY(pe_run(h->pred[i], a, B, s));
    cur ^= 1;
  }
  return DSX_OK;
}

}  // extern "C"

// ---- duration predictor ---------------------------------------------------------------------------------------------
namespace dsx {
namespace {

constexpr int kDpMaxLayers = 16;

// x logically [B, T, C] (any strides: b, c = channel, t) -> fp16 [B][T][C].  One warp per frame.
__global__ void k_dp_pack(const float* x, dsx_strides xs, int B, int T, int C, __half* out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * T) return;
  const int b = warp / T, t = warp - b * T;
  const float* src = x + b * xs.b + t * xs.t;
  for (int c = lane; c < C; c += 32) out[static_cast<size_t>(warp) * C + c] = __float2half_rn(src[c * xs.c]);
}

}  // namespace
}  // namespace dsx

struct dsx_durpred {
  int device = 0;
  dsx_durpred_config cfg{};
  bool loaded = false;
  PePacked conv[dsx::kDpMaxLayers];
  float* head = nullptr;       // linear.weight [P], bias [1]
  DevAllocs mem;
  GrowBuffer ws;
};

namespace dsx {

// DurationPredictor._forward (tts_modules.py:113-129): n_layers x [conv, ReLU, LayerNorm, (dropout), * !mask], then the
// head, from layer 0's fp16 operand A[0].  Eval (tr == NULL) alternates A[0] and A[1]; training reads layer i's operand
// from tr->a[i], writes layer i + 1's there, and saves the LayerNorm inputs and the head's input (DurTrain).  Without a
// mask (the pitch predictor), the last layer's output goes to hin (fp32) and no head runs.
int dp_stack_run(const dsx_durpred* h, __half* const* A, const uint8_t* mask, int B, int T, float* xs, int64_t* dur,
                 const DurTrain* tr, float* hin, cudaStream_t s) {
  const dsx_durpred_config& c = h->cfg;
  const int P = c.chans;
  int cur = 0;
  for (int i = 0; i < c.layers; ++i) {
    PeConvArgs a{};
    a.T = T;
    a.pad = mask;
    a.x = tr ? tr->a[i] : A[cur];
    a.scale = h->conv[i].s;
    a.shift = h->conv[i].t;
    if (i + 1 < c.layers) {
      a.mode = PE_LN;
      a.flags = (mask ? PE_MASK : 0) | PE_OUT16;
      a.o16 = tr ? tr->a[i + 1] : A[cur ^ 1];
    } else if (!mask) {
      a.mode = PE_LN;
      a.flags = PE_OUT32;
      a.o32 = hin;
    } else {
      a.mode = PE_DUR;
      a.hw = h->head;
      a.hb = h->head + P;
      a.o32 = xs;
      a.dur = dur;
      a.offset = c.offset;
    }
    if (!tr) {
      DSX_TRY(pe_run(h->conv[i], a, B, s));
    } else {
      a.r32 = tr->r[i];
      a.h32 = tr->hin;
      a.drop = tr->drop(i);
      a.g = h->conv[i];
      a.mtiles = (T + kConvRows - 1) / kConvRows;
      DSX_TRY(conv_dispatch<256>(h->conv[i].nt, [&](auto k) {
        constexpr int NT = decltype(k)::value;
        k_pe_conv<NT, true><<<dim3(a.mtiles, B), 128 * PeShape<NT>::WG, conv_smem<NT>(), s>>>(a);
        return launch_check("k_pe_conv");
      }));
    }
    cur ^= 1;
  }
  return DSX_OK;
}

}  // namespace dsx

namespace dsx {

int durpred_train_alloc(dsx_durpred* h) {
  DSX_TRY(conv_opt_in<256>([](auto k) { return k_pe_conv<decltype(k)::value, true>; }));
  const dsx_durpred_config& c = h->cfg;
  for (int i = 0; i < c.layers; ++i) {
    PePacked& pc = h->conv[i];
    pc = PePacked{};
    pc.cin = i ? c.chans : c.idim;
    pc.n = c.chans;
    pc.taps = c.kernel;
    pc.tap0 = c.padding ? -(c.kernel - 1) : -(c.kernel - 1) / 2;
    DSX_TRY(conv_alloc(h->mem, pc, 256));
  }
  DSX_TRY(h->mem.alloc(&h->head, (c.chans + 1) * sizeof(float)));
  h->loaded = true;
  return DSX_OK;
}

int durpred_train_pack(dsx_durpred* h, const dsx_durpred_params* p, cudaStream_t s, bool head) {
  const dsx_durpred_config& c = h->cfg;
  const int P = c.chans;
  for (int i = 0; i < c.layers; ++i) {
    PePacked& pc = h->conv[i];
    DSX_TRY(conv_repack(pc, PackArgs{p->conv_w[i], nullptr, p->conv_b[i], pc.cin, P, P, c.kernel, 1, 0}, s));
    pc.s = const_cast<float*>(p->ln_w[i]);
    pc.t = const_cast<float*>(p->ln_b[i]);
  }
  if (!head) return DSX_OK;
  DSX_CUDA(cudaMemcpyAsync(h->head, p->linear_w, P * sizeof(float), cudaMemcpyDeviceToDevice, s));
  DSX_CUDA(cudaMemcpyAsync(h->head + P, p->linear_b, sizeof(float), cudaMemcpyDeviceToDevice, s));
  return DSX_OK;
}

int durpred_train_run(const dsx_durpred* h, const float* x, dsx_strides xs_, const uint8_t* mask, int B, int T,
                      const DurTrain& tr, float* xs, cudaStream_t s) {
  const size_t frames = static_cast<size_t>(B) * T;
  k_dp_pack<<<static_cast<unsigned>((frames * 32 + 255) / 256), 256, 0, s>>>(x, xs_, B, T, h->cfg.idim, tr.a[0]);
  DSX_TRY(launch_check("k_dp_pack"));
  return dp_stack_run(h, nullptr, mask, B, T, xs, nullptr, &tr, nullptr, s);
}

}  // namespace dsx

extern "C" {

int dsx_durpred_create(int device, const dsx_durpred_config* c, dsx_durpred** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_CHECK(c, DSX_E_INVALID, "config is NULL");
  DSX_CHECK(c->idim >= 16 && c->idim <= 256 && c->idim % 16 == 0, DSX_E_INVALID,
            "unsupported idim %d: a multiple of 16 in [16, 256]", c->idim);
  DSX_CHECK(c->chans >= 16 && c->chans <= 256 && c->chans % 16 == 0, DSX_E_INVALID,
            "unsupported n_chans %d: a multiple of 16 in [16, 256]", c->chans);
  DSX_CHECK(c->layers >= 1 && c->layers <= kDpMaxLayers, DSX_E_INVALID, "unsupported n_layers %d: 1..%d", c->layers,
            kDpMaxLayers);
  DSX_CHECK(c->padding == 0 || c->padding == 1, DSX_E_INVALID, "unsupported padding %d: 0 (SAME) or 1 (LEFT)",
            c->padding);
  DSX_CHECK(c->kernel >= 1 && c->kernel <= 31 && (c->padding == 1 || c->kernel % 2 == 1), DSX_E_INVALID,
            "unsupported kernel_size %d: in [1, 31], odd for SAME", c->kernel);
  DSX_CHECK(isfinite(c->offset), DSX_E_INVALID, "unsupported offset: must be finite");
  DSX_TRY(select_sm90_device(device, "duration predictor"));
  DSX_TRY(conv_opt_in<256>([](auto k) { return k_pe_conv<decltype(k)::value>; }));
  dsx_durpred* h = new dsx_durpred();
  h->device = device;
  h->cfg = *c;
  *out = h;
  return DSX_OK;
}

void dsx_durpred_destroy(dsx_durpred* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  h->mem.free_all();
  h->ws.release();
  delete h;
}

int dsx_durpred_load(dsx_durpred* h, const dsx_durpred_params* p, void* stream) {
  DSX_CHECK(h && p, DSX_E_INVALID, "null handle or params");
  DSX_CHECK(p->conv_w && p->conv_b && p->ln_w && p->ln_b && p->linear_w && p->linear_b, DSX_E_INVALID,
            "missing conv, LayerNorm or linear arrays");
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const dsx_durpred_config& c = h->cfg;
  const int P = c.chans, k = c.kernel;
  DSX_CUDA(cudaStreamSynchronize(s));   // the old packs may still be read by queued work
  h->mem.free_all();
  h->loaded = false;
  const int tap0 = c.padding ? -(k - 1) : -(k - 1) / 2;   // ConstantPad1d LEFT (k - 1, 0) or SAME
  char what[64];
  for (int i = 0; i < c.layers; ++i) {
    PePacked& pc = h->conv[i];
    pc = PePacked{};
    snprintf(what, sizeof what, "conv.%d.1", i);
    DSX_CHECK(p->conv_w[i] && p->conv_b[i], DSX_E_INVALID, "missing %s", what);
    pc.cin = i ? P : c.idim;
    pc.n = P;
    pc.taps = k;
    pc.tap0 = tap0;
    DSX_TRY(conv_pack(h->mem, pc, 256, PackArgs{p->conv_w[i], nullptr, p->conv_b[i], pc.cin, P, P, k, 1, 0}, s));
    DSX_CHECK(p->ln_w[i] && p->ln_b[i], DSX_E_INVALID, "missing conv.%d.3", i);
    DSX_TRY(h->mem.alloc(&pc.s, P * sizeof(float)));
    DSX_TRY(h->mem.alloc(&pc.t, P * sizeof(float)));
    DSX_CUDA(cudaMemcpyAsync(pc.s, p->ln_w[i], P * sizeof(float), cudaMemcpyDeviceToDevice, s));
    DSX_CUDA(cudaMemcpyAsync(pc.t, p->ln_b[i], P * sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  DSX_TRY(h->mem.alloc(&h->head, (P + 1) * sizeof(float)));
  DSX_CUDA(cudaMemcpyAsync(h->head, p->linear_w, P * sizeof(float), cudaMemcpyDeviceToDevice, s));
  DSX_CUDA(cudaMemcpyAsync(h->head + P, p->linear_b, sizeof(float), cudaMemcpyDeviceToDevice, s));
  h->loaded = true;
  return DSX_OK;
}

int dsx_durpred_forward(dsx_durpred* h, const float* x, dsx_strides xs_, const uint8_t* mask, int B, int T, float* xs,
                        int64_t* dur, void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(h->loaded, DSX_E_STATE, "dsx_durpred_load has not been called");
  DSX_CHECK(x && mask && xs, DSX_E_INVALID, "x, mask and xs must not be NULL");
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(B <= 65535, DSX_E_INVALID, "B = %d utterances per call is above the 65535 the launch grid holds", B);
  const dsx_durpred_config& c = h->cfg;
  const int P = c.chans, C = std::max(c.idim, P);
  DSX_CHECK(static_cast<long long>(B) * T * C < (1ll << 31), DSX_E_INVALID, "B * T = %lld tokens is too large",
            static_cast<long long>(B) * T);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t frames = static_cast<size_t>(B) * T;
  DSX_TRY(h->ws.reserve(2 * align256(frames * C * 2), s));
  Bump ws{static_cast<uint8_t*>(h->ws.ptr)};
  __half* A[2] = {ws.take<__half>(frames * C * 2), ws.take<__half>(frames * C * 2)};
  k_dp_pack<<<static_cast<unsigned>((frames * 32 + 255) / 256), 256, 0, s>>>(x, xs_, B, T, c.idim, A[0]);
  DSX_TRY(launch_check("k_dp_pack"));
  return dp_stack_run(h, A, mask, B, T, xs, dur, nullptr, nullptr, s);
}

}  // extern "C"
