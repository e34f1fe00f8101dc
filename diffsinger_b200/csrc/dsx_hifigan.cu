// HiFi-GAN (NSF) generator on sm_90a: the vocoder that turns the sampler's mel spectrogram into a waveform
// (modules/hifigan/hifigan.py:104-171 with the harmonic source of modules/parallel_wavegan/models/source.py).
//
// Every convolution with a tensor-core shape is one implicit GEMM on wgmma (k_conv, on the core of dsx_conv.cuh), over
// activations padded to a multiple of 16 channels, the layout of the sampler's step kernel:
//   Conv1d(k, dilation d, padding (k - 1) d / 2)        tap0 = -(k - 1) d / 2, tstep = d, N = C_out
//   ConvTranspose1d(k, stride u, padding (k - u) / 2)   polyphase: out[m u + r - pad] = sum_{j < k/u} x[m - j] W[:, :, r + j u]
//                                                       tap0 = 0, tstep = -1, N = u C_out (column n = r C_out + o); the
//                                                       epilogue scatters the phases
// The epilogue adds the bias and, by flags, the NSF branch's noise conv (ups), a fp32 residual, the fp32 multi-receptive-
// field sum and its 1 / num_kernels, and writes fp32 and / or leaky_relu(., 0.1) in fp16 (the next conv's operand).
// On stages of at most 64 channels a whole ResBlock runs as one chained launch instead (k_chain, below).  The harmonic
// source and conv_post (N = 1) run on CUDA cores.
#include <math.h>
#include <stdio.h>

#include <algorithm>

#include "dsx_conv.cuh"
#include "dsx_internal.h"
#include "dsx_ptx.cuh"
#include "dsx_rng.cuh"
#include "dsx_wnorm.cuh"

namespace dsx {
namespace {

constexpr int kMelBins = 80;
constexpr int kHarmonics = 9;        // SineGen dim = harmonic_num + 1 (hifigan.py:112)
constexpr float kLrelu = 0.1f;       // LRELU_SLOPE (hifigan.py:11)
constexpr float kSineAmp = 0.1f, kNoiseStd = 0.003f;   // SineGen defaults (source.py)

inline int round16(int c) { return (c + 15) & ~15; }

// one packed convolution: the GEMM (cin padded to 16, at most 128 columns per tile) and its output channels
struct PackedConv : ConvGemm {
  int cout = 0, cout_p = 0;    // cout_p: padded to 16
  int u = 1, pad = 0;          // ConvTranspose1d: stride and padding (u == 1, pad == 0 for Conv1d)
};

enum { EPI_OUT32 = 1, EPI_OUT16 = 2, EPI_RES = 4, EPI_SUM = 8, EPI_DIV = 16, EPI_NOISE = 32 };

struct ConvArgs {
  ConvGemm g;
  const __half* x;             // A source [B][lx][g.cin]
  int lx;
  int cout_p, u, pad, ups;     // ups: polyphase ConvTranspose1d
  const int* lens;             // [B] frames, or null (all T)
  int T, in_mul;               // valid input rows of utterance b = len_b * in_mul
  int flags;
  float* o32;                  // [B][lo][cout_p] fp32 out (EPI_OUT32), the MRF sum read first when EPI_SUM
  __half* o16;                 // [B][lo][cout_p] fp16 leaky_relu(out) (EPI_OUT16)
  const float* res;            // [B][lo][cout_p] residual added (EPI_RES)
  int lo;
  float div;                   // EPI_DIV: out /= div (the MRF mean)
  const float* har;            // EPI_NOISE: harmonic source [B][lh]
  const float* nw;             // [cout_p][nks]
  const float* nb;             // [cout_p]
  int lh, hop, ns, nks, npad;
};

__device__ __forceinline__ int utt_len(const int* lens, int b, int T) {
  return lens ? min(max(lens[b], 0), T) : T;
}

template <int NT>
__global__ void __launch_bounds__(128) k_conv(const ConvArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, b = blockIdx.z, nt = blockIdx.y, m0 = blockIdx.x * kConvRows;
  const int len_frames = utt_len(p.lens, b, p.T);
  const int len_in = len_frames * p.in_mul;
  const int len_out = len_in * p.u;
  const int rows = p.ups ? len_in + (p.pad + p.u - 1) / p.u : len_in;   // ups: the last output rows come from m >= len_in
  if (m0 >= rows) return;

  float acc[NT / 2];
  conv_k_loop<NT, 1>(p.g, p.x, p.lx, len_in, b, m0, nt, smem, acc);

  // epilogue: element pairs (n, n + 1) share the phase r (cout_p is even) and are adjacent in memory
  const int len_h = len_frames * p.hop;
#pragma unroll
  for (int e = 0; e < NT / 2; e += 2) {
    const int m = m0 + acc_row(tid, e), n = nt * NT + acc_col(tid, e);
    if (n >= p.g.n || m >= rows) continue;
    int row = m, o = n;
    if (p.ups) {
      const int r = n / p.cout_p;
      o = n - r * p.cout_p;
      row = m * p.u + r - p.pad;
    }
    if (row < 0 || row >= len_out) continue;
    float v0 = acc[e] + p.g.b[n], v1 = acc[e + 1] + p.g.b[n + 1];
    if (p.flags & EPI_NOISE) {         // noise_convs[i](har): stride ns, nks taps, padding npad, zero outside [0, len_h)
      const float* hb = p.har + static_cast<size_t>(b) * p.lh;
      const float* w0 = p.nw + static_cast<size_t>(o) * p.nks;
      const float* w1 = w0 + p.nks;
      float s0 = 0.f, s1 = 0.f;
      const int t0 = row * p.ns - p.npad;
      for (int j = 0; j < p.nks; ++j) {
        const int t = t0 + j;
        const float hv = (t >= 0 && t < len_h) ? __ldg(hb + t) : 0.f;
        s0 = fmaf(__ldg(w0 + j), hv, s0);
        s1 = fmaf(__ldg(w1 + j), hv, s1);
      }
      v0 += s0 + p.nb[o];
      v1 += s1 + p.nb[o + 1];
    }
    const size_t idx = (static_cast<size_t>(b) * p.lo + row) * p.cout_p + o;
    if (p.flags & EPI_RES) {
      const float2 rv = *reinterpret_cast<const float2*>(p.res + idx);
      v0 += rv.x;
      v1 += rv.y;
    }
    if (p.flags & EPI_SUM) {
      const float2 sv = *reinterpret_cast<const float2*>(p.o32 + idx);
      v0 = sv.x + v0;
      v1 = sv.y + v1;
    }
    if (p.flags & EPI_DIV) {
      v0 = v0 / p.div;
      v1 = v1 / p.div;
    }
    if (p.flags & EPI_OUT32) *reinterpret_cast<float2*>(p.o32 + idx) = make_float2(v0, v1);
    if (p.flags & EPI_OUT16)
      *reinterpret_cast<__half2*>(p.o16 + idx) =
          __floats2half2_rn(v0 > 0.f ? v0 : kLrelu * v0, v1 > 0.f ? v1 : kLrelu * v1);
  }
}

// ---- weight packing ------------------------------------------------------------------------------
// dst[r][j] = src[r][j] * (scale ? scale[0] : 1) for r < rows, 0 for rows <= r < rows_p (noise_convs, conv_post)
__global__ void k_pack_rows(float* dst, const float* src, const float* scale, int rows, int rows_p, int cols) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows_p * cols) return;
  dst[i] = (i / cols < rows) ? src[i] * (scale ? scale[0] : 1.f) : 0.f;
}

// ---- forward helpers -----------------------------------------------------------------------------
// mel [B, 80, T] (any strides) -> fp16 [B][T][80]
__global__ void k_pack_mel(const float* mel, dsx_strides ms, int B, int T, __half* out) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<size_t>(B) * T * kMelBins) return;
  const int c = static_cast<int>(i % kMelBins);
  const size_t bt = i / kMelBins;
  const int t = static_cast<int>(bt % T), b = static_cast<int>(bt / T);
  out[i] = __float2half_rn(mel[b * ms.b + c * ms.c + t * ms.t]);
}

// rad = (f0 * (h + 1) / sr) % 1, in the reference's fp32 order (source.py: f0_buf, then / samp_rate, then % 1)
__device__ __forceinline__ float nsf_rad(float f0, int h, float sr) {
  const float f = h == 0 ? f0 : f0 * static_cast<float>(h + 1);
  const float x = f / sr;
  return x - floorf(x);
}

// Phase of harmonic h at the start of every frame, kept in [0, 1) (what cumsum_shift does in SineGen._f02sine): f0 is
// upsampled by nearest, so a frame advances the phase by frac(hop * rad).  One block per (b, h) scans the frames in
// fp64, kPhaseChunk frames per thread and 256 * kPhaseChunk per pass.  The summation tree depends only on the frame
// index, so an utterance gets the same phases whatever T the batch is padded to.
constexpr int kPhaseChunk = 8;
__global__ void __launch_bounds__(256) k_nsf_phase(const float* f0, const float* phase0, uint64_t seed, int T, int hop,
                                                   float sr, double* ph) {
  const int b = blockIdx.x / kHarmonics, h = blockIdx.x - b * kHarmonics, tid = threadIdx.x;
  double carry = 0.0;
  if (h > 0) {
    if (phase0) {
      carry = phase0[b * kHarmonics + h];
    } else {   // torch.rand(B, 9) with column 0 zeroed: Philox uniforms, counter (2 b + (h > 4), 0), offset 1
      const uint4 r = philox4x32_10(make_uint4(2u * b + (h > 4), 0u, 1u, 0u),
                                    make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)));
      const uint32_t v[4] = {r.x, r.y, r.z, r.w};
      carry = static_cast<float>(v[(h - 1) & 3]) * 2.3283064365386963e-10f;
    }
  }
  __shared__ double sh[256];
  const float* fb = f0 + static_cast<size_t>(b) * T;
  auto step = [&](int t) {
    const double d = static_cast<double>(hop) * nsf_rad(fb[t], h, sr);
    return d - floor(d);
  };
  for (int base = 0; base < T; base += 256 * kPhaseChunk) {
    const int t0 = base + tid * kPhaseChunk, t1 = min(T, t0 + kPhaseChunk);
    double local = 0.0;
    for (int t = t0; t < t1; ++t) local += step(t);
    sh[tid] = local;
    __syncthreads();
    for (int off = 1; off < 256; off <<= 1) {   // inclusive scan over the block
      const double v = tid >= off ? sh[tid - off] : 0.0;
      __syncthreads();
      sh[tid] += v;
      __syncthreads();
    }
    double s = carry + (sh[tid] - local);
    s -= floor(s);
    for (int t = t0; t < t1; ++t) {
      ph[(static_cast<size_t>(b) * T + t) * kHarmonics + h] = s;
      s += step(t);
      s -= floor(s);
    }
    carry += sh[255];
    carry -= floor(carry);
    __syncthreads();
  }
}

// SourceModuleHnNSF: har = tanh(l_linear(sine_waves * uv + noise)), sine_waves = 0.1 sin(2 pi phase); one thread per sample
__global__ void k_nsf_source(const float* f0, const double* ph, const float* noise, uint64_t seed, const float* lw,
                             const float* lb, int B, int T, int hop, float sr, float* har) {
  const size_t lh = static_cast<size_t>(T) * hop;
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<size_t>(B) * lh) return;
  const size_t b = i / lh, n = i - b * lh;
  const int t = static_cast<int>(n / hop), k = static_cast<int>(n - static_cast<size_t>(t) * hop);
  const float f = f0[b * T + t];
  const float uv = f > 0.f ? 1.f : 0.f;
  const float amp = uv * kNoiseStd + (1.f - uv) * kSineAmp / 3.f;
  float z[12];
  if (noise) {
#pragma unroll
    for (int h = 0; h < kHarmonics; ++h) z[h] = noise[i * kHarmonics + h];
  } else {   // torch.randn_like(sine_waves): Philox normals, block (b * lh + n) * 3 + q, offset 0
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const float4 g = philox_normal4(seed, 0, i * 3 + q);
      z[4 * q] = g.x;
      z[4 * q + 1] = g.y;
      z[4 * q + 2] = g.z;
      z[4 * q + 3] = g.w;
    }
  }
  const double* p0 = ph + (b * T + t) * kHarmonics;
  float acc = lb[0];
#pragma unroll
  for (int h = 0; h < kHarmonics; ++h) {
    double phase = p0[h] + static_cast<double>(k + 1) * nsf_rad(f, h, sr);
    phase -= floor(phase);
    const float sine = sinf(6.283185307179586f * static_cast<float>(phase)) * kSineAmp;
    acc = fmaf(lw[h], sine * uv + amp * z[h], acc);
  }
  har[i] = tanhf(acc);
}

// conv_post on CUDA cores: wav = tanh(conv1d(leaky_relu(x, 0.01), k = 7, pad 3)); samples from len_b * hop on are 0
__global__ void k_post(const float* x, int lo, int cp, int c, const float* w, const float* bias, const int* lens, int T,
                       int hop, int B, float* wav) {
  const size_t lh = static_cast<size_t>(T) * hop;
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<size_t>(B) * lh) return;
  const int b = static_cast<int>(i / lh), n = static_cast<int>(i - static_cast<size_t>(b) * lh);
  const int len = utt_len(lens, b, T) * hop;
  float acc = 0.f;
  if (n < len) {
    acc = bias[0];
    for (int j = 0; j < 7; ++j) {
      const int t = n + j - 3;
      if (t < 0 || t >= len) continue;
      const float* xr = x + (static_cast<size_t>(b) * lo + t) * cp;
      for (int ch = 0; ch < c; ++ch) {
        const float v = xr[ch];
        acc = fmaf(w[ch * 7 + j], v > 0.f ? v : 0.01f * v, acc);
      }
    }
    acc = tanhf(acc);
  }
  wav[i] = acc;
}

// ---- one ResBlock as a chain of convs over one tile -----------------------------------------------
// Stages of at most 64 (padded) channels are bandwidth-bound one conv per launch, so k_chain runs a whole ResBlock per
// CTA: 4 warpgroups cover kChainRows tile rows, global rows [g0 - H, g0 - H + kChainRows), H = the block's halo (the sum
// of (k - 1) / 2 * d over its convs).  Each warpgroup keeps the fp32 residual x of its 64 rows in registers; the fp16
// operand leaky_relu(.) of all rows sits in shared memory (rows outside the utterance held at 0, which is the convs' zero
// padding), and tap j of a conv is the wgmma A descriptor started (j - (k - 1) / 2) * d rows away.  Rows near the tile
// edge go wrong conv by conv, H rows in all, so only the kChainRows - 2H centre rows are written: the block's share of
// the MRF sum, and after the last block the stage output.  A conv's weights (all taps) are loaded into shared memory
// while the previous conv's epilogue runs.
constexpr int kChainRows = 256, kChainPad = 32, kChainMaxConvs = 6;
constexpr int kChainOpBytes = (kChainRows + 2 * kChainPad) * 128;
constexpr int kChainSmemMax = 227 * 1024;   // opt-in shared memory per block on sm_90

struct ChainArgs {
  const float* x;              // ups output [B][lo][cp]
  float* s;                    // MRF sum [B][lo][cp]
  __half* o16;                 // leaky_relu(stage output) [B][lo][cp] (EPI_OUT16)
  const int* lens;
  int T, mul, lo, halo, nconv, flags;
  float div;
  const __half* w[kChainMaxConvs];   // PackedConv::w (one column tile)
  const float* b[kChainMaxConvs];
  int taps[kChainMaxConvs], tap0[kChainMaxConvs], tstep[kChainMaxConvs];
  int resid;                   // bit q: conv q adds into the residual (else its output is only the next operand)
};

template <int NT>
constexpr int chain_smem(int taps) { return 1024 + kChainOpBytes + taps * NT * 128; }

template <int NT>
__global__ void __launch_bounds__(512) k_chain(const ChainArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* op = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* wbuf = op + kChainOpBytes;
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, b = blockIdx.y;
  const int len = utt_len(p.lens, b, p.T) * p.mul;
  const int out_rows = kChainRows - 2 * p.halo;
  const int g0 = blockIdx.x * out_rows;
  if (g0 >= len) return;
  const int gbase = g0 - p.halo;

  auto load_w = [&](int q) {
    const uint32_t d = smem_u32(wbuf);
    const int nchunk = p.taps[q] * NT * (NT / 8);
    for (int i = tid; i < nchunk; i += 512) {
      const int c = i % (NT / 8), rn = i / (NT / 8), n = rn % NT, j = rn / NT;
      const int kk = j * NT + c * 8;   // (tap, channel) of the K-flattened pack
      cp16(d + j * NT * 128 + sw128(n, c), p.w[q] + (static_cast<size_t>(kk >> 6) * NT + n) * 64 + (kk & 63), true);
    }
  };
  load_w(0);
  cp_commit();
  for (int i = tid; i < 2 * kChainPad * 8; i += 512) {   // the pad rows above and below the tile read as 0
    const int r = i >> 3, row = r < kChainPad ? r : kChainRows + r;
    *reinterpret_cast<uint4*>(op + row * 128 + (i & 7) * 16) = make_uint4(0, 0, 0, 0);
  }
  float x[NT / 2], acc[NT / 2];
  auto put_op = [&](int e, float v0, float v1) {
    const int rt = wg * 64 + acc_row(wtid, e), n = acc_col(wtid, e), g = gbase + rt;
    const bool valid = g >= 0 && g < len;
    const __half2 hv = valid ? __floats2half2_rn(v0 > 0.f ? v0 : kLrelu * v0, v1 > 0.f ? v1 : kLrelu * v1)
                             : __floats2half2_rn(0.f, 0.f);
    *reinterpret_cast<__half2*>(op + sw128(kChainPad + rt, n >> 3) + (n & 7) * 2) = hv;
  };
#pragma unroll
  for (int e = 0; e < NT / 2; e += 2) {
    const int rt = wg * 64 + acc_row(wtid, e), n = acc_col(wtid, e), g = gbase + rt;
    float2 v = make_float2(0.f, 0.f);
    if (g >= 0 && g < len) v = *reinterpret_cast<const float2*>(p.x + (static_cast<size_t>(b) * p.lo + g) * NT + n);
    x[e] = v.x;
    x[e + 1] = v.y;
    put_op(e, v.x, v.y);
  }
  cp_wait<0>();
  fence_proxy_async_smem();
  __syncthreads();

#pragma unroll 1
  for (int q = 0; q < p.nconv; ++q) {
#pragma unroll
    for (int e = 0; e < NT / 2; ++e) acc[e] = 0.f;
    wg_fence();
#pragma unroll 1
    for (int j = 0; j < p.taps[q]; ++j) {
      const int row = kChainPad + wg * 64 + p.tap0[q] + j * p.tstep[q];
      const uint64_t da = wg_desc(smem_u32(op + row * 128)), db = wg_desc(smem_u32(wbuf + j * NT * 128));
#pragma unroll
      for (int k = 0; k < NT / 16; ++k) wgmma_f16<NT>(acc, da + 2 * k, db + 2 * k, 1);
    }
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < NT / 2; ++e) asm volatile("" : "+f"(acc[e])::"memory");
    __syncthreads();                   // every warpgroup is done with this conv's operand and weights
    if (q + 1 < p.nconv) {
      load_w(q + 1);
      cp_commit();
    }
    const float* bias = p.b[q];
    const bool resid = (p.resid >> q) & 1;
#pragma unroll
    for (int e = 0; e < NT / 2; e += 2) {
      const int n = acc_col(wtid, e);
      float v0 = acc[e] + bias[n], v1 = acc[e + 1] + bias[n + 1];
      if (resid) {
        x[e] = v0 + x[e];
        x[e + 1] = v1 + x[e + 1];
        v0 = x[e];
        v1 = x[e + 1];
      }
      if (q + 1 < p.nconv) put_op(e, v0, v1);
    }
    cp_wait<0>();
    fence_proxy_async_smem();
    __syncthreads();
  }

  // the block's output x joins the MRF sum (EPI_SUM), divided by num_kernels after the last block (EPI_DIV)
#pragma unroll
  for (int e = 0; e < NT / 2; e += 2) {
    const int rt = wg * 64 + acc_row(wtid, e), n = acc_col(wtid, e), g = gbase + rt;
    if (rt < p.halo || rt >= p.halo + out_rows || g >= len) continue;
    const size_t idx = (static_cast<size_t>(b) * p.lo + g) * NT + n;
    float v0 = x[e], v1 = x[e + 1];
    if (p.flags & EPI_SUM) {
      const float2 sv = *reinterpret_cast<const float2*>(p.s + idx);
      v0 = sv.x + v0;
      v1 = sv.y + v1;
    }
    if (p.flags & EPI_DIV) {
      v0 = v0 / p.div;
      v1 = v1 / p.div;
    }
    if (p.flags & EPI_OUT32) *reinterpret_cast<float2*>(p.s + idx) = make_float2(v0, v1);
    if (p.flags & EPI_OUT16)
      *reinterpret_cast<__half2*>(p.o16 + idx) =
          __floats2half2_rn(v0 > 0.f ? v0 : kLrelu * v0, v1 > 0.f ? v1 : kLrelu * v1);
  }
}

}  // namespace
}  // namespace dsx

using namespace dsx;

struct dsx_hifigan {
  int device = 0;
  dsx_hifigan_config cfg{};
  int hop = 1, nconv_block = 0;
  bool loaded = false;
  PackedConv pre;
  std::vector<PackedConv> ups, rb;
  std::vector<float*> noise_w, noise_b;   // [cout_p][nks], [cout_p]
  std::vector<int> noise_ks, noise_s;
  float* src_w = nullptr;                 // [9] + bias [1]
  float* post_w = nullptr;                // [cp][7] + bias at [cp * 7]
  DevAllocs mem;                          // the packs above
  GrowBuffer scale;                       // weight-norm scratch
  GrowBuffer ws;                          // workspace of a forward call
};

namespace {

void free_model(dsx_hifigan* h) {
  h->mem.free_all();
  h->ups.clear();
  h->rb.clear();
  h->noise_w.clear();
  h->noise_b.clear();
  h->loaded = false;
}

int stage_cin(const dsx_hifigan_config& c, int i) { return c.upsample_initial_channel >> i; }

int pack_conv(dsx_hifigan* h, PackedConv& pc, const float* v, const float* g, const float* bias, int cin, int cout,
              int k, int dil, int u, bool transposed, cudaStream_t s) {
  DSX_CHECK(v && bias, DSX_E_INVALID, "missing conv weight or bias");
  pc.cin = round16(cin);
  pc.cout = cout;
  pc.cout_p = round16(cout);
  if (transposed) {
    pc.u = u;
    pc.pad = (k - u) / 2;
    pc.taps = k / u;
    pc.tap0 = 0;
    pc.tstep = -1;
    pc.n = u * pc.cout_p;
  } else {
    pc.u = 1;
    pc.pad = 0;
    pc.taps = k;
    pc.tap0 = -(k - 1) / 2 * dil;
    pc.tstep = dil;
    pc.n = pc.cout_p;
  }
  float* scale = static_cast<float*>(h->scale.ptr);
  k_wnorm<<<transposed ? cin : cout, 256, 0, s>>>(v, g, (transposed ? cout : cin) * k, scale);
  DSX_TRY(launch_check("k_wnorm"));
  return conv_pack(h->mem, pc, 128, PackArgs{v, scale, bias, cin, cout, pc.cout_p, k, u, transposed ? 1 : 0}, s);
}

// one conv over the batch; rows_max = GEMM rows of the longest utterance
int run_conv(const PackedConv& pc, ConvArgs a, int B, int rows_max, cudaStream_t s) {
  a.g = pc;
  a.cout_p = pc.cout_p;
  a.u = pc.u;
  a.pad = pc.pad;
  const dim3 grid((rows_max + kConvRows - 1) / kConvRows, pc.ntiles, B);
  return conv_dispatch<128>(pc.nt, [&](auto c) {
    constexpr int NT = decltype(c)::value;
    k_conv<NT><<<grid, 128, conv_smem<NT>(), s>>>(a);
    return launch_check("k_conv");
  });
}

// chain order of a block's convs: ResBlock1 convs1.0, convs2.0, convs1.1, ... (packed as convs1.*, convs2.*)
const PackedConv& chain_conv(const dsx_hifigan* h, int blk, int q) {
  const PackedConv* cv = &h->rb[static_cast<size_t>(blk) * h->nconv_block];
  return h->cfg.resblock == 1 ? cv[(q & 1) * 3 + (q >> 1)] : cv[q];
}

int chain_halo(const dsx_hifigan* h, int blk) {
  int halo = 0;
  for (int q = 0; q < h->nconv_block; ++q) halo += -chain_conv(h, blk, q).tap0;
  return halo;
}

// The chained ResBlock kernel takes a stage whose padded width is 16, 32 or 64 channels when every block's tile keeps
// at least 64 centre rows, every tap stays inside the tile's zero pad and a conv's weights fit in shared memory.
// Wider stages run one k_conv launch per conv: their weights (taps x C x C) do not fit next to the tile.
bool chain_usable(const dsx_hifigan* h, int stage) {
  const int nk = h->cfg.num_kernels, cp = h->ups[stage].cout_p;
  if (cp != 16 && cp != 32 && cp != 64) return false;
  for (int j = 0; j < nk; ++j) {
    const int blk = stage * nk + j;
    if (kChainRows - 2 * chain_halo(h, blk) < 64) return false;
    for (int q = 0; q < h->nconv_block; ++q) {
      const PackedConv& pc = chain_conv(h, blk, q);
      if (-pc.tap0 > kChainPad || 1024 + kChainOpBytes + pc.taps * cp * 128 > kChainSmemMax) return false;
    }
  }
  return true;
}

template <int NT>
int launch_chain_nt(const ChainArgs& a, int taps_max, int tiles, int B, cudaStream_t s) {
  k_chain<NT><<<dim3(tiles, B), 512, chain_smem<NT>(taps_max), s>>>(a);
  return launch_check("k_chain");
}

int run_chain(const dsx_hifigan* h, int blk, const float* X, float* S, __half* P, const int* lens, int T, int mul,
              int lo, int flags, float div, int B, cudaStream_t s) {
  ChainArgs a{};
  a.x = X;
  a.s = S;
  a.o16 = P;
  a.lens = lens;
  a.T = T;
  a.mul = mul;
  a.lo = lo;
  a.halo = chain_halo(h, blk);
  a.nconv = h->nconv_block;
  a.flags = flags;
  a.div = div;
  int taps_max = 0;
  for (int q = 0; q < a.nconv; ++q) {
    const PackedConv& pc = chain_conv(h, blk, q);
    a.w[q] = pc.w;
    a.b[q] = pc.b;
    a.taps[q] = pc.taps;
    a.tap0[q] = pc.tap0;
    a.tstep[q] = pc.tstep;
    if (h->cfg.resblock == 2 || (q & 1)) a.resid |= 1 << q;
    taps_max = std::max(taps_max, pc.taps);
  }
  const int out_rows = kChainRows - 2 * a.halo, tiles = (T * mul + out_rows - 1) / out_rows;
  switch (h->ups[blk / h->cfg.num_kernels].cout_p) {
    case 16: return launch_chain_nt<16>(a, taps_max, tiles, B, s);
    case 32: return launch_chain_nt<32>(a, taps_max, tiles, B, s);
    default: return launch_chain_nt<64>(a, taps_max, tiles, B, s);
  }
}

int validate(const dsx_hifigan_config* c) {
  DSX_CHECK(c, DSX_E_INVALID, "config is NULL");
  DSX_CHECK(c->num_upsamples >= 1 && c->num_upsamples <= 4, DSX_E_INVALID, "num_upsamples must be 1..4 (got %d)",
            c->num_upsamples);
  long long hop = 1;
  for (int i = 0; i < c->num_upsamples; ++i) {
    const int u = c->upsample_rates[i], k = c->upsample_kernel_sizes[i];
    DSX_CHECK(u >= 1 && u <= 64 && k >= u && k <= 256 && k % u == 0 && (k - u) % 2 == 0, DSX_E_INVALID,
              "ups.%d: need 1 <= u <= 64, u <= k <= 256, k %% u == 0 and k - u even (got u = %d, k = %d)", i, u, k);
    hop *= u;
  }
  DSX_CHECK(hop <= 4096, DSX_E_INVALID, "product of the upsample rates must be <= 4096 (got %lld)", hop);
  const int c0 = c->upsample_initial_channel;
  DSX_CHECK(c0 >= 2 && c0 <= 2048 && c0 % (1 << c->num_upsamples) == 0, DSX_E_INVALID,
            "upsample_initial_channel must be in [2, 2048] and divisible by 2^num_upsamples (got %d)", c0);
  DSX_CHECK(c->resblock == 1 || c->resblock == 2, DSX_E_INVALID, "resblock must be 1 or 2 (got %d)", c->resblock);
  DSX_CHECK(c->num_kernels >= 1 && c->num_kernels <= 3, DSX_E_INVALID, "num_kernels must be 1..3 (got %d)", c->num_kernels);
  const int nd = c->resblock == 1 ? 3 : 2;
  for (int j = 0; j < c->num_kernels; ++j) {
    const int k = c->resblock_kernel_sizes[j];
    DSX_CHECK(k >= 1 && k <= 31 && k % 2 == 1, DSX_E_INVALID, "resblock kernel size %d must be odd and <= 31", k);
    for (int q = 0; q < nd; ++q)
      DSX_CHECK(c->resblock_dilation_sizes[j][q] >= 1 && c->resblock_dilation_sizes[j][q] <= 64, DSX_E_INVALID,
                "resblock dilation [%d][%d] must be in [1, 64] (got %d)", j, q, c->resblock_dilation_sizes[j][q]);
  }
  DSX_CHECK(c->audio_sample_rate > 0, DSX_E_INVALID, "audio_sample_rate must be positive (got %d)", c->audio_sample_rate);
  DSX_CHECK(c->use_pitch_embed == 0 || c->use_pitch_embed == 1, DSX_E_INVALID, "use_pitch_embed must be 0 or 1");
  if (c->use_pitch_embed) {
    long long s = hop;
    for (int i = 0; i + 1 < c->num_upsamples; ++i) {
      s /= c->upsample_rates[i];
      DSX_CHECK(s % 2 == 0, DSX_E_INVALID, "noise_convs.%d: stride %lld must be even to match the stage length", i, s);
    }
  }
  return DSX_OK;
}

}  // namespace

extern "C" {

int dsx_hifigan_create(int device, const dsx_hifigan_config* cfg, dsx_hifigan** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_TRY(validate(cfg));
  DSX_TRY(select_sm90_device(device, "vocoder"));
  DSX_TRY(conv_opt_in<128>([](auto c) { return k_conv<decltype(c)::value>; }));
  DSX_CUDA(cudaFuncSetAttribute(k_chain<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kChainSmemMax));
  DSX_CUDA(cudaFuncSetAttribute(k_chain<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, kChainSmemMax));
  DSX_CUDA(cudaFuncSetAttribute(k_chain<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, kChainSmemMax));
  dsx_hifigan* h = new dsx_hifigan();
  h->device = device;
  h->cfg = *cfg;
  for (int i = 0; i < cfg->num_upsamples; ++i) h->hop *= cfg->upsample_rates[i];
  h->nconv_block = cfg->resblock == 1 ? 6 : 2;
  *out = h;
  return DSX_OK;
}

void dsx_hifigan_destroy(dsx_hifigan* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  free_model(h);
  h->scale.release();
  h->ws.release();
  delete h;
}

int dsx_hifigan_load(dsx_hifigan* h, const dsx_hifigan_params* p, void* stream) {
  DSX_CHECK(h && p, DSX_E_INVALID, "null handle or params");
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const dsx_hifigan_config& c = h->cfg;
  const int nu = c.num_upsamples, nk = c.num_kernels;
  DSX_CHECK(p->ups_w && p->ups_b && p->rb_w && p->rb_b, DSX_E_INVALID, "missing per-module weight arrays");
  DSX_CHECK(!c.use_pitch_embed || (p->noise_w && p->noise_b && p->source_w && p->source_b), DSX_E_INVALID,
            "use_pitch_embed needs noise_convs and m_source parameters");
  DSX_CHECK(p->conv_post_w && p->conv_post_b, DSX_E_INVALID, "missing conv_post parameters");
  DSX_CUDA(cudaStreamSynchronize(s));   // the old packs may still be read by queued work
  free_model(h);
  DSX_TRY(h->scale.reserve(static_cast<size_t>(std::max(c.upsample_initial_channel, kMelBins)) * sizeof(float), s));
  const int c0 = c.upsample_initial_channel;
  DSX_TRY(pack_conv(h, h->pre, p->conv_pre_w, p->conv_pre_g, p->conv_pre_b, kMelBins, c0, 7, 1, 1, false, s));
  h->ups.resize(nu);
  h->rb.resize(static_cast<size_t>(nu) * nk * h->nconv_block);
  for (int i = 0; i < nu; ++i) {
    const int cin = stage_cin(c, i), cout = cin / 2;
    DSX_TRY(pack_conv(h, h->ups[i], p->ups_w[i], p->ups_g ? p->ups_g[i] : nullptr, p->ups_b[i], cin, cout,
                      c.upsample_kernel_sizes[i], 1, c.upsample_rates[i], true, s));
    for (int j = 0; j < nk; ++j) {
      const int blk = i * nk + j, k = c.resblock_kernel_sizes[j];
      for (int q = 0; q < h->nconv_block; ++q) {
        // ResBlock1: convs1.q (q < 3, dilation d[q]) then convs2.(q - 3) (dilation 1); ResBlock2: convs.q (dilation d[q])
        const int dil = (c.resblock == 1 && q >= 3) ? 1 : c.resblock_dilation_sizes[j][q];
        const int e = blk * h->nconv_block + q;
        DSX_TRY(pack_conv(h, h->rb[e], p->rb_w[e], p->rb_g ? p->rb_g[e] : nullptr, p->rb_b[e], cout, cout, k, dil, 1,
                          false, s));
      }
    }
  }
  const int clast = stage_cin(c, nu), cp_last = round16(clast);
  if (c.use_pitch_embed) {
    long long stride = h->hop;
    h->noise_w.resize(nu);
    h->noise_b.resize(nu);
    h->noise_ks.resize(nu);
    h->noise_s.resize(nu);
    for (int i = 0; i < nu; ++i) {
      stride /= c.upsample_rates[i];
      const int cout = stage_cin(c, i) / 2, cp = round16(cout);
      const int ks = (i + 1 < nu) ? static_cast<int>(2 * stride) : 1;
      DSX_CHECK(p->noise_w[i] && p->noise_b[i], DSX_E_INVALID, "missing noise_convs.%d", i);
      h->noise_s[i] = static_cast<int>(stride);
      h->noise_ks[i] = ks;
      DSX_TRY(h->mem.alloc(&h->noise_w[i], static_cast<size_t>(cp) * ks * sizeof(float)));
      DSX_TRY(h->mem.alloc(&h->noise_b[i], cp * sizeof(float)));
      k_pack_rows<<<(cp * ks + 255) / 256, 256, 0, s>>>(h->noise_w[i], p->noise_w[i], nullptr, cout, cp, ks);
      k_pack_rows<<<1, 256, 0, s>>>(h->noise_b[i], p->noise_b[i], nullptr, cout, cp, 1);
      DSX_TRY(launch_check("k_pack_rows"));
    }
    DSX_TRY(h->mem.alloc(&h->src_w, (kHarmonics + 1) * sizeof(float)));
    DSX_CUDA(cudaMemcpyAsync(h->src_w, p->source_w, kHarmonics * sizeof(float), cudaMemcpyDeviceToDevice, s));
    DSX_CUDA(cudaMemcpyAsync(h->src_w + kHarmonics, p->source_b, sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  DSX_TRY(h->mem.alloc(&h->post_w, (static_cast<size_t>(cp_last) * 7 + 1) * sizeof(float)));
  float* scale = static_cast<float*>(h->scale.ptr);
  k_wnorm<<<1, 256, 0, s>>>(p->conv_post_w, p->conv_post_g, clast * 7, scale);
  k_pack_rows<<<(cp_last * 7 + 255) / 256, 256, 0, s>>>(h->post_w, p->conv_post_w, scale, clast, cp_last, 7);
  DSX_CUDA(cudaMemcpyAsync(h->post_w + cp_last * 7, p->conv_post_b, sizeof(float), cudaMemcpyDeviceToDevice, s));
  DSX_TRY(launch_check("conv_post pack"));
  h->loaded = true;
  return DSX_OK;
}

int dsx_hifigan_forward(dsx_hifigan* h, const float* mel, dsx_strides ms, const float* f0, const int* lengths,
                        const float* phase0, const float* src_noise, uint64_t seed, int B, int T, float* wav,
                        void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(h->loaded, DSX_E_STATE, "dsx_hifigan_load has not been called");
  DSX_CHECK(mel && wav, DSX_E_INVALID, "mel and wav must not be NULL");
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(B <= 65535, DSX_E_INVALID, "B = %d utterances per call is above the 65535 the launch grid holds", B);
  const dsx_hifigan_config& c = h->cfg;
  DSX_CHECK(!f0 || c.use_pitch_embed, DSX_E_INVALID, "f0 given but the generator has no NSF source (use_pitch_embed = 0)");
  const long long lh_ll = static_cast<long long>(T) * h->hop;
  DSX_CHECK(lh_ll * B < (1ll << 31), DSX_E_INVALID, "B * T * hop = %lld samples is too large", lh_ll * B);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int nu = c.num_upsamples, nk = c.num_kernels, lh = static_cast<int>(lh_ll);

  // workspace: fp16 MEL / P / Q / T / U0 / U1, fp32 X / R / S, the harmonic source and the frame phases
  size_t act = static_cast<size_t>(T) * round16(c.upsample_initial_channel);   // per utterance, elements
  int f = 1;
  for (int i = 0; i < nu; ++i) {
    f *= c.upsample_rates[i];
    act = std::max(act, static_cast<size_t>(T) * f * round16(stage_cin(c, i + 1)));
  }
  act *= B;
  const size_t mel_e = static_cast<size_t>(B) * T * kMelBins;
  const size_t har_b = static_cast<size_t>(B) * lh * 4, ph_b = static_cast<size_t>(B) * T * kHarmonics * 8;
  DSX_TRY(h->ws.reserve(align256(mel_e * 2) + 5 * align256(act * 2) + 3 * align256(act * 4) +
                        (f0 ? align256(har_b) + align256(ph_b) : 0), s));
  Bump ws{static_cast<uint8_t*>(h->ws.ptr)};
  __half* MEL = ws.take<__half>(mel_e * 2);
  __half* P = ws.take<__half>(act * 2);    // leaky_relu(stage input) -> ups
  __half* Q = ws.take<__half>(act * 2);    // leaky_relu(ups output) -> first conv of every block
  __half* Tm = ws.take<__half>(act * 2);   // ResBlock1: leaky_relu(convs1 output)
  __half* U[2] = {ws.take<__half>(act * 2), ws.take<__half>(act * 2)};
  float* X = ws.take<float>(act * 4);      // ups output (+ noise conv)
  float* R = ws.take<float>(act * 4);      // the running residual inside a block
  float* S = ws.take<float>(act * 4);      // multi-receptive-field sum
  float* HAR = f0 ? ws.take<float>(har_b) : nullptr;
  double* PH = f0 ? ws.take<double>(ph_b) : nullptr;

  k_pack_mel<<<static_cast<unsigned>((mel_e + 255) / 256), 256, 0, s>>>(mel, ms, B, T, MEL);
  DSX_TRY(launch_check("k_pack_mel"));
  const float sr = static_cast<float>(c.audio_sample_rate);
  if (f0) {
    k_nsf_phase<<<B * kHarmonics, 256, 0, s>>>(f0, phase0, seed, T, h->hop, sr, PH);
    DSX_TRY(launch_check("k_nsf_phase"));
    const size_t ns = static_cast<size_t>(B) * lh;
    k_nsf_source<<<static_cast<unsigned>((ns + 255) / 256), 256, 0, s>>>(f0, PH, src_noise, seed, h->src_w,
                                                                         h->src_w + kHarmonics, B, T, h->hop, sr, HAR);
    DSX_TRY(launch_check("k_nsf_source"));
  }

  ConvArgs base{};
  base.lens = lengths;
  base.T = T;
  base.hop = h->hop;
  base.lh = lh;
  base.har = HAR;
  base.div = 1.f;

  ConvArgs a = base;   // conv_pre -> P
  a.x = MEL;
  a.lx = T;
  a.in_mul = 1;
  a.flags = EPI_OUT16;
  a.o16 = P;
  a.lo = T;
  DSX_TRY(run_conv(h->pre, a, B, T, s));
  f = 1;
  long long nstride = h->hop;
  for (int i = 0; i < nu; ++i) {
    const PackedConv& up = h->ups[i];
    const int lin = T * f, lout = lin * up.u;
    nstride /= up.u;
    a = base;          // ups[i] (+ noise_convs[i](har)) -> X, leaky_relu -> Q
    a.x = P;
    a.lx = lin;
    a.in_mul = f;
    a.ups = 1;
    const bool chain = chain_usable(h, i);
    a.flags = EPI_OUT32 | (chain ? 0 : EPI_OUT16) | (f0 ? EPI_NOISE : 0);
    a.o32 = X;
    a.o16 = Q;
    a.lo = lout;
    if (f0) {
      a.nw = h->noise_w[i];
      a.nb = h->noise_b[i];
      a.ns = h->noise_s[i];
      a.nks = h->noise_ks[i];
      a.npad = h->noise_s[i] / 2;
    }
    DSX_TRY(run_conv(up, a, B, lin + (up.pad + up.u - 1) / up.u, s));
    f *= up.u;
    const bool last_stage = i + 1 == nu;
    for (int j = 0; j < nk; ++j) {
      const PackedConv* cv = &h->rb[static_cast<size_t>(i * nk + j) * h->nconv_block];
      const bool last_block = j + 1 == nk;
      const int mrf = (j > 0 ? EPI_SUM : 0) | (last_block ? EPI_DIV : 0) |
                      ((!last_block || last_stage) ? EPI_OUT32 : 0) | ((last_block && !last_stage) ? EPI_OUT16 : 0);
      if (chain) {
        DSX_TRY(run_chain(h, i * nk + j, X, S, P, lengths, T, f, lout, mrf, static_cast<float>(nk), B, s));
        continue;
      }
      const int npair = c.resblock == 1 ? 3 : 2;
      for (int q = 0; q < npair; ++q) {
        const __half* in = q == 0 ? Q : U[(q - 1) & 1];
        ConvArgs b2 = base;
        b2.lx = lout;
        b2.lo = lout;
        b2.in_mul = f;
        if (c.resblock == 1) {   // xt = convs1[q](lrelu(x)) -> leaky_relu -> Tm
          ConvArgs b1 = b2;
          b1.x = in;
          b1.flags = EPI_OUT16;
          b1.o16 = Tm;
          DSX_TRY(run_conv(cv[q], b1, B, lout, s));
          b2.x = Tm;
        } else {
          b2.x = in;
        }
        const PackedConv& c2 = c.resblock == 1 ? cv[3 + q] : cv[q];
        b2.res = q == 0 ? X : R;   // x = conv(xt) + x
        if (q + 1 < npair) {
          b2.flags = EPI_RES | EPI_OUT32 | EPI_OUT16;
          b2.o32 = R;
          b2.o16 = U[q & 1];
        } else {                   // the block's output joins the MRF sum; after the last block, the stage output
          b2.flags = EPI_RES | mrf;
          b2.o32 = S;
          b2.o16 = P;
          b2.div = static_cast<float>(nk);
        }
        DSX_TRY(run_conv(c2, b2, B, lout, s));
      }
    }
  }
  const size_t nwav = static_cast<size_t>(B) * lh;
  const int clast = stage_cin(c, nu);
  k_post<<<static_cast<unsigned>((nwav + 255) / 256), 256, 0, s>>>(S, lh, round16(clast), clast, h->post_w,
                                                                   h->post_w + round16(clast) * 7, lengths, T, h->hop, B,
                                                                   wav);
  return launch_check("k_post");
}

}  // extern "C"
