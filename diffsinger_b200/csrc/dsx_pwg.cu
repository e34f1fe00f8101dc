// Parallel WaveGAN generator on sm_90a: noise + mel (+ coarse pitch) to waveform, the vocoder vocoders/pwg.py runs
// (modules/parallel_wavegan/models/parallel_wavegan.py:21-191 with the ConvInUpsampleNetwork of
// modules/parallel_wavegan/layers/upsample.py and the ResidualBlock of layers/residual_block.py).
//
// Layout: audio-rate tensors are samples-major, one row per output sample, utterance b's rows at [b * L, (b + 1) * L)
// with L = T * hop.  Per call:
//   conditioning  (k_pwg_cproj) -> k_pwg_convin -> k_pwg_upsample per scale, fp32 on CUDA cores, zero padding at each
//                 stage's utterance edges; the last stage writes c_up, the fp16 GEMM operand [rows][80]
//   first_conv    k_pwg_first: x = w z + b in fp32, and its fp16 operand copy
//   each layer    k_pwg_layer, one launch: GEMM1 (N = 128, K = 3 taps x 64 + 80 c_up channels) on wgmma, the bias and the
//                 tanh . sigmoid gate in the epilogue into shared memory, GEMM2 (N = 128: conv1x1_out | conv1x1_skip over
//                 the 64 gate channels), and the epilogue x <- (out + b + x) sqrt(1/2), skip += s + b in fp32 with the
//                 fp16 operand copy of x written to the other of two buffers (the next layer reads shifted rows)
//   head          k_pwg_head: ReLU(skip sqrt(1 / layers)), 64 x 64 + b, ReLU, 64 -> 1 + b, fp32
// Each CTA of k_pwg_layer holds the layer's packed weights in shared memory and its two warpgroups walk 64-row tiles
// independently; a tile never spans two utterances, so an utterance's rows see the same tile edges in any batch.
#include <math.h>

#include <algorithm>

#include "dsx_internal.h"
#include "dsx_ptx.cuh"
#include "dsx_wnorm.cuh"

namespace dsx {
namespace {

constexpr int kRes = 64, kGate = 128, kSkip = 64, kAux = 80, kKernel = 3;   // the only widths the kernels implement
constexpr int kPitchBins = 300;          // nn.Embedding(300, aux_channels) (parallel_wavegan.py:132)
constexpr int kTileRows = 64;            // rows per warpgroup tile
constexpr int kW1Chunks = 5;             // GEMM1's K in 64-wide chunks: 3 taps x 64, then c_up channels 0..63 and 64..79
constexpr int kChunkBytes = kGate * 128;                     // one 64-wide K chunk of 128 weight rows
constexpr int kWBytes = (kW1Chunks + 1) * kChunkBytes;       // W1, then W2 [128][64]
constexpr int kABytes = kW1Chunks * kTileRows * 128;         // a warpgroup's A tiles: 3 taps, c_up 0..63, c_up 64..79
constexpr int kZBytes = kTileRows * 128;                     // the gate output, GEMM2's A
constexpr int kLayerSmem = 1024 + kWBytes + 2 * (kABytes + kZBytes);
constexpr int kLayerWeights = (kW1Chunks + 1) * kGate * 64;  // fp16 elements of one layer's pack
constexpr long long kMaxSamples = 1ll << 25;                 // cap on B * T * hop

// ---- weight packing ------------------------------------------------------------------------------
// dst[i] = v[i] * scale[i / inner]: a conv's weight with its weight norm (scale from k_wnorm)
__global__ void k_pwg_scale(float* dst, const float* v, const float* scale, int n, int inner) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = v[i] * scale[i / inner];
}

// One residual layer's GEMM operands, fp16, unswizzled: W1 [5][128][64] (chunk, gate channel n, K inside the chunk;
// K = j * 64 + c for tap j and residual channel c, then 192 + a for aux channel a, zero past 272), W2 [128][64] (rows
// 0..63 conv1x1_out, 64..127 conv1x1_skip); biases b1 [128] (conv) and b2 [128] (out | skip).  s: the weight-norm
// scales, [128] conv, [128] aux, [64] out, [64] skip.
struct LayerPackArgs {
  const float *conv_w, *aux_w, *out_w, *skip_w, *conv_b, *out_b, *skip_b, *s;
  __half* w;
  float* b;
};

__global__ void k_pwg_pack_layer(const LayerPackArgs p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kLayerWeights) return;
  const int q = i & 63, n = (i >> 6) & 127, ch = i >> 13;
  float v = 0.f;
  if (ch < kW1Chunks) {
    const int kk = ch * 64 + q;
    if (kk < kKernel * kRes) {
      const int j = kk >> 6, c = kk & 63;
      v = p.conv_w[(n * kRes + c) * kKernel + j] * p.s[n];
    } else if (kk < kKernel * kRes + kAux) {
      v = p.aux_w[n * kAux + kk - kKernel * kRes] * p.s[kGate + n];
    }
  } else {
    v = (n < kRes ? p.out_w[n * 64 + q] : p.skip_w[(n - kRes) * 64 + q]) * p.s[2 * kGate + n];
  }
  p.w[i] = __float2half_rn(v);
  if (i < kGate) {
    p.b[i] = p.conv_b[i];
    p.b[kGate + i] = i < kRes ? p.out_b[i] : p.skip_b[i - kRes];
  }
}

// ---- conditioning (frame rate, then each upsampling stage) ----------------------------------------
// c_proj(cat[c^T, pitch_embed(pitch)]) (parallel_wavegan.py:157-159): c [B, 80, Tp] (strides cs), pitch int64 [B][Tp];
// a pitch outside [0, 300) reads a zero row.  -> out [B][Tp][80] fp32
__global__ void k_pwg_cproj(const float* c, dsx_strides cs, const int64_t* pitch, const float* emb, const float* w,
                            const float* bias, int B, int Tp, float* out) {
  const size_t n = static_cast<size_t>(B) * Tp * kAux;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int o = static_cast<int>(i % kAux);
    const size_t bt = i / kAux;
    const int t = static_cast<int>(bt % Tp), b = static_cast<int>(bt / Tp);
    const float* wr = w + o * 2 * kAux;
    float acc = bias[o];
    for (int a = 0; a < kAux; ++a) acc = fmaf(wr[a], c[b * cs.b + a * cs.c + t * cs.t], acc);
    const int64_t pv = pitch[bt];
    if (pv >= 0 && pv < kPitchBins) {
      const float* er = emb + pv * kAux;
      for (int a = 0; a < kAux; ++a) acc = fmaf(wr[kAux + a], er[a], acc);
    }
    out[i] = acc;
  }
}

// conv_in (upsample.py:155,176): Conv1d(80, 80, K = 2w + 1, no padding, no bias) over c [B, 80, T + 2w] (strides cs)
// -> out [B][T][80] fp32; w holds [80][80][K] with its weight norm applied
__global__ void k_pwg_convin(const float* c, dsx_strides cs, const float* w, int K, int B, int T, float* out) {
  const size_t n = static_cast<size_t>(B) * T * kAux;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int o = static_cast<int>(i % kAux);
    const size_t bt = i / kAux;
    const int t = static_cast<int>(bt % T), b = static_cast<int>(bt / T);
    const float* wr = w + o * kAux * K;
    float acc = 0.f;
    for (int a = 0; a < kAux; ++a) {
      const float* cr = c + b * cs.b + a * cs.c + t * cs.t;
      for (int j = 0; j < K; ++j) acc = fmaf(wr[a * K + j], cr[j * cs.t], acc);
    }
    out[i] = acc;
  }
}

// One UpsampleNetwork stage (upsample.py:84-98,118-124): Stretch2d by s (nearest: sample u repeats frame u / s), then
// Conv2d(1, 1, (1, 2s + 1), padding (0, s)) along time, zero outside [0, lin * s).  in [B][lin][80] fp32 -> out
// [B][lin * s][80], fp32 (out32) or the fp16 GEMM operand (out16)
__global__ void k_pwg_upsample(const float* in, int lin, int s, const float* w, int B, float* out32, __half* out16) {
  const int lout = lin * s;
  const size_t n = static_cast<size_t>(B) * lout * kAux;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int a = static_cast<int>(i % kAux);
    const size_t bu = i / kAux;
    const int u = static_cast<int>(bu % lout), b = static_cast<int>(bu / lout);
    const float* src = in + static_cast<size_t>(b) * lin * kAux + a;
    float acc = 0.f;
    for (int k = 0; k <= 2 * s; ++k) {
      const int v = u + k - s;
      if (v >= 0 && v < lout) acc = fmaf(w[k], src[static_cast<size_t>(v / s) * kAux], acc);
    }
    if (out16) out16[i] = __float2half_rn(acc);
    else out32[i] = acc;
  }
}

// ---- audio rate ------------------------------------------------------------------------------------
// first_conv (Conv1d1x1(1, 64)): x = w z + b -> fp32 x and its fp16 operand copy, [rows][64]
__global__ void k_pwg_first(const float* z, const float* w, size_t rows, float* x, __half* xh) {
  const size_t n = rows * kRes;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i & (kRes - 1));
    const float v = fmaf(w[c], z[i / kRes], w[kRes + c]);
    x[i] = v;
    xh[i] = __float2half_rn(v);
  }
}

struct LayerArgs {
  const __half* w;             // the layer's pack (k_pwg_pack_layer)
  const float* b;              // b1 [128], b2 [128]
  const __half* xin;           // fp16 x [rows][64], read at rows m - d, m, m + d
  __half* xout;                // fp16 x of the next layer
  float* x;                    // fp32 residual stream [rows][64]
  float* skip;                 // fp32 skip sum [rows][64]
  const __half* cup;           // fp16 c_up [rows][80]
  int L, d, tiles_per_utt, tiles;
  int first, last;             // first: skip = s (no read); last: x and its copy are not written
};

// One residual layer (residual_block.py:94-129) over 64-row tiles; see the file comment.
__global__ void __launch_bounds__(256, 1) k_pwg_layer(const LayerArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  uint8_t* A = sm + kWBytes + wg * (kABytes + kZBytes);
  uint8_t* Z = A + kABytes;
  {
    const uint32_t dw = smem_u32(sm);
    for (int i = tid; i < (kW1Chunks + 1) * kGate * 8; i += 256) {
      const int c = i & 7, r = (i >> 3) & 127, ch = i >> 10;
      cp16(dw + ch * kChunkBytes + sw128(r, c), p.w + (static_cast<size_t>(ch) * kGate + r) * 64 + c * 8, true);
    }
    cp_commit();
  }
  // a tile's A: three taps of x (rows m0 + r + (j - 1) d, zero outside the utterance) and c_up's 80 channels (10
  // 16-byte pieces per row: 0..7 into tile 3, 8..9 into tile 4, whose other K columns are never read)
  auto load_tile = [&](int t) {
    const int b = t / p.tiles_per_utt, m0 = (t - b * p.tiles_per_utt) * kTileRows;
    const size_t base = static_cast<size_t>(b) * p.L;
    const uint32_t da = smem_u32(A);
    if (wtid == 0) {                   // the tile's fp32 x and skip rows, which its residual epilogue reads, into L2
      const uint32_t bytes = static_cast<uint32_t>(min(kTileRows, p.L - m0)) * kRes * 4;
      const uint64_t pol = l2_evict_last();
      if (!p.first) prefetch_l2_hint(p.skip + (base + m0) * kRes, bytes, pol);
      if (!p.last) prefetch_l2_hint(p.x + (base + m0) * kRes, bytes, pol);
    }
#pragma unroll 1
    for (int i = wtid; i < 3 * kTileRows * 8 + kTileRows * 10; i += 128) {
      if (i < 3 * kTileRows * 8) {
        const int c = i & 7, r = (i >> 3) & (kTileRows - 1), j = i >> 9;
        const int src = m0 + r + (j - 1) * p.d;
        const bool v = src >= 0 && src < p.L;
        cp16(da + j * kTileRows * 128 + sw128(r, c), p.xin + (base + (v ? src : 0)) * kRes + c * 8, v);
      } else {
        const int k = i - 3 * kTileRows * 8, r = k / 10, c = k - r * 10;
        const bool v = m0 + r < p.L;
        cp16(da + (3 + (c >> 3)) * kTileRows * 128 + sw128(r, c & 7), p.cup + (base + (v ? m0 + r : 0)) * kAux + c * 8,
             v);
      }
    }
    cp_commit();
  };
  const int nw = gridDim.x * 2;
  int t = blockIdx.x * 2 + wg;
  if (t < p.tiles) load_tile(t);
  cp_wait<0>();
  fence_proxy_async_smem();
  __syncthreads();                     // the weights of both warpgroups' copies, and each warpgroup's first tile
  const float* b1 = p.b;
  const float* b2 = p.b + kGate;
  constexpr float kSqrtHalf = 0.70710678118654752f;
  float acc[64];
#pragma unroll 1
  for (; t < p.tiles; t += nw) {
    const int b = t / p.tiles_per_utt, m0 = (t - b * p.tiles_per_utt) * kTileRows;
    // GEMM1: [x(m - d) | x(m) | x(m + d) | c_up] . W1
#pragma unroll
    for (int e = 0; e < 64; ++e) acc[e] = 0.f;
    wg_fence();
    const uint64_t da = wg_desc(smem_u32(A)), dw = wg_desc(smem_u32(sm));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_n128(acc, da + j * (kTileRows * 8) + 2 * k, dw + j * (kChunkBytes >> 4) + 2 * k, 1);
    }
    wgmma_n128(acc, da + 4 * (kTileRows * 8), dw + 4 * (kChunkBytes >> 4), 1);
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < 64; ++e) asm volatile("" : "+f"(acc[e])::"memory");
    wg_bar_sync();                     // A is free: the next tile's loads run under this tile's epilogues
    if (t + nw < p.tiles) load_tile(t + nw);
    // gate: columns n < 64 are xa (tanh), n + 64 xb (sigmoid); the thread holds both in acc[e] and acc[e + 32]
#pragma unroll
    for (int e = 0; e < 32; e += 2) {
      const int row = acc_row(wtid, e), n = acc_col(wtid, e);
      const float z0 = gate_acc(acc[e + 32] + __ldg(b1 + n + 64), acc[e] + __ldg(b1 + n));
      const float z1 = gate_acc(acc[e + 33] + __ldg(b1 + n + 65), acc[e + 1] + __ldg(b1 + n + 1));
      *reinterpret_cast<__half2*>(Z + sw128(row, n >> 3) + (n & 7) * 2) = __floats2half2_rn(z0, z1);
    }
    fence_proxy_async_smem();
    wg_bar_sync();
    // GEMM2: z . [W_out | W_skip]
#pragma unroll
    for (int e = 0; e < 64; ++e) acc[e] = 0.f;
    wg_fence();
    const uint64_t dz = wg_desc(smem_u32(Z)), d2 = dw + kW1Chunks * (kChunkBytes >> 4);
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_n128(acc, dz + 2 * k, d2 + 2 * k, 1);
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < 64; ++e) asm volatile("" : "+f"(acc[e])::"memory");
    // residual and skip: the thread holds out[n] in acc[e] and skip[n] in acc[e + 32]
#pragma unroll
    for (int e = 0; e < 32; e += 2) {
      const int row = acc_row(wtid, e), n = acc_col(wtid, e), m = m0 + row;
      if (m >= p.L) continue;
      const size_t idx = (static_cast<size_t>(b) * p.L + m) * kRes + n;
      float s0 = acc[e + 32] + __ldg(b2 + n + 64), s1 = acc[e + 33] + __ldg(b2 + n + 65);
      if (!p.first) {
        const float2 sv = *reinterpret_cast<const float2*>(p.skip + idx);
        s0 = sv.x + s0;
        s1 = sv.y + s1;
      }
      *reinterpret_cast<float2*>(p.skip + idx) = make_float2(s0, s1);
      if (!p.last) {
        const float2 xv = *reinterpret_cast<const float2*>(p.x + idx);
        const float x0 = (acc[e] + __ldg(b2 + n) + xv.x) * kSqrtHalf;
        const float x1 = (acc[e + 1] + __ldg(b2 + n + 1) + xv.y) * kSqrtHalf;
        *reinterpret_cast<float2*>(p.x + idx) = make_float2(x0, x1);
        *reinterpret_cast<__half2*>(p.xout + idx) = __floats2half2_rn(x0, x1);
      }
    }
    cp_wait<0>();
    fence_proxy_async_smem();
    wg_bar_sync();                     // the next tile's A has landed; this tile's Z reads are done
  }
}

// last_conv_layers (parallel_wavegan.py:124-129,167-172) after skips *= sqrt(1 / layers): one thread per sample.
// hw: [64][64] W1, [64] b1, [64] w2, [1] b2 (weight norms applied)
__global__ void __launch_bounds__(256) k_pwg_head(const float* skip, const float* hw, float scale, size_t rows,
                                                  float* wav) {
  __shared__ float sw[kSkip * kSkip + 2 * kSkip + 1];
  for (int i = threadIdx.x; i < kSkip * kSkip + 2 * kSkip + 1; i += blockDim.x) sw[i] = hw[i];
  __syncthreads();
  for (size_t r = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; r < rows;
       r += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float h[kSkip];
    const float4* src = reinterpret_cast<const float4*>(skip + r * kSkip);
#pragma unroll
    for (int q = 0; q < kSkip / 4; ++q) {
      const float4 v = src[q];
      h[4 * q] = fmaxf(v.x * scale, 0.f);
      h[4 * q + 1] = fmaxf(v.y * scale, 0.f);
      h[4 * q + 2] = fmaxf(v.z * scale, 0.f);
      h[4 * q + 3] = fmaxf(v.w * scale, 0.f);
    }
    float out = sw[kSkip * kSkip + 2 * kSkip];
#pragma unroll 4
    for (int o = 0; o < kSkip; ++o) {
      float acc = sw[kSkip * kSkip + o];
#pragma unroll
      for (int i = 0; i < kSkip; ++i) acc = fmaf(sw[o * kSkip + i], h[i], acc);
      out = fmaf(sw[kSkip * kSkip + kSkip + o], fmaxf(acc, 0.f), out);
    }
    wav[r] = out;
  }
}

unsigned grid_for(size_t n) { return static_cast<unsigned>(std::min<size_t>((n + 255) / 256, 65536)); }

}  // namespace
}  // namespace dsx

using namespace dsx;

struct dsx_pwg {
  int device = 0, sms = 1;
  dsx_pwg_config cfg{};
  int hop = 1, w = 0;
  bool loaded = false;
  __half* layer_w = nullptr;   // [layers][kLayerWeights]
  float* layer_b = nullptr;    // [layers][256]
  float* first = nullptr;      // w [64], b [64]
  float* convin = nullptr;     // [80][80][2w + 1]
  float* up = nullptr;         // per scale 2s + 1 taps, at up_off[i]
  int up_off[4] = {};
  float* head = nullptr;       // [64][64] W1, [64] b1, [64] w2, [1] b2
  float* emb = nullptr;        // [300][80], c_proj [80][160], c_proj bias [80] (use_pitch_embed)
  DevAllocs mem;               // the packs above
  GrowBuffer scale;            // weight-norm scratch
  GrowBuffer ws;               // workspace of a forward call
};

namespace {

void free_model(dsx_pwg* h) {
  h->mem.free_all();
  h->loaded = false;
}

int validate(const dsx_pwg_config* c) {
  DSX_CHECK(c, DSX_E_INVALID, "config is NULL");
  DSX_CHECK(c->residual_channels == kRes && c->gate_channels == kGate && c->skip_channels == kSkip &&
                c->aux_channels == kAux && c->kernel_size == kKernel,
            DSX_E_INVALID,
            "unsupported widths: the kernels implement residual = skip = 64, gate = 128, aux = 80 and kernel_size 3 "
            "(got residual %d, skip %d, gate %d, aux %d, kernel_size %d)",
            c->residual_channels, c->skip_channels, c->gate_channels, c->aux_channels, c->kernel_size);
  DSX_CHECK(c->layers >= 1 && c->layers <= 64, DSX_E_INVALID, "unsupported layers %d: 1..64", c->layers);
  DSX_CHECK(c->stacks >= 1 && c->layers % c->stacks == 0 && c->layers / c->stacks <= 16, DSX_E_INVALID,
            "unsupported stacks %d: layers %% stacks == 0 and layers / stacks <= 16", c->stacks);
  DSX_CHECK(c->num_scales >= 1 && c->num_scales <= 4, DSX_E_INVALID, "unsupported number of upsample_scales %d: 1..4",
            c->num_scales);
  int hop = 1;
  for (int i = 0; i < c->num_scales; ++i) {
    DSX_CHECK(c->upsample_scales[i] >= 1 && c->upsample_scales[i] <= 16, DSX_E_INVALID,
              "unsupported upsample_scales[%d] = %d: 1..16", i, c->upsample_scales[i]);
    hop *= c->upsample_scales[i];
  }
  DSX_CHECK(hop <= 1024, DSX_E_INVALID, "unsupported hop %d (the product of upsample_scales): at most 1024", hop);
  DSX_CHECK(c->aux_context_window >= 0 && c->aux_context_window <= 16, DSX_E_INVALID,
            "unsupported aux_context_window %d: 0..16", c->aux_context_window);
  DSX_CHECK(c->use_pitch_embed == 0 || c->use_pitch_embed == 1, DSX_E_INVALID, "unsupported use_pitch_embed %d: 0 or 1",
            c->use_pitch_embed);
  return DSX_OK;
}

// dst = v with the weight norm of g (rows of `inner` elements; g NULL: v as is)
int pack_wn(const float* v, const float* g, int rows, int inner, float* dst, float* scale, cudaStream_t s) {
  k_wnorm<<<rows, 256, 0, s>>>(v, g, inner, scale);
  k_pwg_scale<<<(rows * inner + 255) / 256, 256, 0, s>>>(dst, v, scale, rows * inner, inner);
  return launch_check("k_pwg_scale");
}

}  // namespace

extern "C" {

int dsx_pwg_create(int device, const dsx_pwg_config* cfg, dsx_pwg** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_TRY(validate(cfg));
  DSX_TRY(select_sm90_device(device, "PWG vocoder"));
  DSX_CUDA(cudaFuncSetAttribute(k_pwg_layer, cudaFuncAttributeMaxDynamicSharedMemorySize, kLayerSmem));
  int sms = 1;
  DSX_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
  dsx_pwg* h = new dsx_pwg();
  h->device = device;
  h->sms = sms;
  h->cfg = *cfg;
  for (int i = 0; i < cfg->num_scales; ++i) h->hop *= cfg->upsample_scales[i];
  h->w = cfg->aux_context_window;
  *out = h;
  return DSX_OK;
}

void dsx_pwg_destroy(dsx_pwg* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  free_model(h);
  h->scale.release();
  h->ws.release();
  delete h;
}

int dsx_pwg_load(dsx_pwg* h, const dsx_pwg_params* p, void* stream) {
  DSX_CHECK(h && p, DSX_E_INVALID, "null handle or params");
  const dsx_pwg_config& c = h->cfg;
  const int nl = c.layers, ns = c.num_scales, K = 2 * h->w + 1;
  DSX_CHECK(p->first_w && p->first_b && p->conv_in_w && p->up_w && p->conv_w && p->conv_b && p->aux_w && p->out_w &&
                p->out_b && p->skip_w && p->skip_b && p->last1_w && p->last1_b && p->last3_w && p->last3_b,
            DSX_E_INVALID, "missing parameters");
  for (int i = 0; i < ns; ++i) DSX_CHECK(p->up_w[i], DSX_E_INVALID, "missing upsample_net.upsample.up_layers.%d", 2 * i + 1);
  for (int l = 0; l < nl; ++l)
    DSX_CHECK(p->conv_w[l] && p->conv_b[l] && p->aux_w[l] && p->out_w[l] && p->out_b[l] && p->skip_w[l] && p->skip_b[l],
              DSX_E_INVALID, "missing parameters of conv_layers.%d", l);
  DSX_CHECK(!c.use_pitch_embed || (p->pitch_embed && p->c_proj_w && p->c_proj_b), DSX_E_INVALID,
            "use_pitch_embed needs pitch_embed and c_proj");
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_CUDA(cudaStreamSynchronize(s));   // the old packs may still be read by queued work
  free_model(h);
  DSX_TRY(h->scale.reserve(2 * (kGate + kRes) * sizeof(float), s));
  float* sc = static_cast<float*>(h->scale.ptr);
  DSX_TRY(h->mem.alloc(&h->layer_w, static_cast<size_t>(nl) * kLayerWeights * sizeof(__half)));
  DSX_TRY(h->mem.alloc(&h->layer_b, static_cast<size_t>(nl) * 2 * kGate * sizeof(float)));
  for (int l = 0; l < nl; ++l) {
    auto g = [&](const float* const* a) { return a ? a[l] : nullptr; };
    k_wnorm<<<kGate, 256, 0, s>>>(p->conv_w[l], g(p->conv_g), kRes * kKernel, sc);
    k_wnorm<<<kGate, 256, 0, s>>>(p->aux_w[l], g(p->aux_g), kAux, sc + kGate);
    k_wnorm<<<kRes, 256, 0, s>>>(p->out_w[l], g(p->out_g), kGate / 2, sc + 2 * kGate);
    k_wnorm<<<kSkip, 256, 0, s>>>(p->skip_w[l], g(p->skip_g), kGate / 2, sc + 2 * kGate + kRes);
    const LayerPackArgs a{p->conv_w[l], p->aux_w[l], p->out_w[l], p->skip_w[l], p->conv_b[l], p->out_b[l], p->skip_b[l],
                          sc, h->layer_w + static_cast<size_t>(l) * kLayerWeights, h->layer_b + l * 2 * kGate};
    k_pwg_pack_layer<<<(kLayerWeights + 255) / 256, 256, 0, s>>>(a);
    DSX_TRY(launch_check("k_pwg_pack_layer"));
  }
  DSX_TRY(h->mem.alloc(&h->first, 2 * kRes * sizeof(float)));
  DSX_TRY(pack_wn(p->first_w, p->first_g, kRes, 1, h->first, sc, s));
  DSX_CUDA(cudaMemcpyAsync(h->first + kRes, p->first_b, kRes * sizeof(float), cudaMemcpyDeviceToDevice, s));
  DSX_TRY(h->mem.alloc(&h->convin, static_cast<size_t>(kAux) * kAux * K * sizeof(float)));
  DSX_TRY(pack_wn(p->conv_in_w, p->conv_in_g, kAux, kAux * K, h->convin, sc, s));
  int taps = 0;
  for (int i = 0; i < ns; ++i) {
    h->up_off[i] = taps;
    taps += 2 * c.upsample_scales[i] + 1;
  }
  DSX_TRY(h->mem.alloc(&h->up, taps * sizeof(float)));
  for (int i = 0; i < ns; ++i)
    DSX_TRY(pack_wn(p->up_w[i], p->up_g ? p->up_g[i] : nullptr, 1, 2 * c.upsample_scales[i] + 1, h->up + h->up_off[i], sc,
                    s));
  DSX_TRY(h->mem.alloc(&h->head, (kSkip * kSkip + 2 * kSkip + 1) * sizeof(float)));
  DSX_TRY(pack_wn(p->last1_w, p->last1_g, kSkip, kSkip, h->head, sc, s));
  DSX_CUDA(cudaMemcpyAsync(h->head + kSkip * kSkip, p->last1_b, kSkip * sizeof(float), cudaMemcpyDeviceToDevice, s));
  DSX_TRY(pack_wn(p->last3_w, p->last3_g, 1, kSkip, h->head + kSkip * kSkip + kSkip, sc, s));
  DSX_CUDA(cudaMemcpyAsync(h->head + kSkip * kSkip + 2 * kSkip, p->last3_b, sizeof(float), cudaMemcpyDeviceToDevice, s));
  if (c.use_pitch_embed) {
    const size_t ne = kPitchBins * kAux, nc = 2 * kAux * kAux;
    DSX_TRY(h->mem.alloc(&h->emb, (ne + nc + kAux) * sizeof(float)));
    DSX_CUDA(cudaMemcpyAsync(h->emb, p->pitch_embed, ne * sizeof(float), cudaMemcpyDeviceToDevice, s));
    DSX_CUDA(cudaMemcpyAsync(h->emb + ne, p->c_proj_w, nc * sizeof(float), cudaMemcpyDeviceToDevice, s));
    DSX_CUDA(cudaMemcpyAsync(h->emb + ne + nc, p->c_proj_b, kAux * sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  h->loaded = true;
  return DSX_OK;
}

int dsx_pwg_forward(dsx_pwg* h, const float* z, const float* c, dsx_strides cs, const int64_t* pitch, int B, int T,
                    float* wav, void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(h->loaded, DSX_E_STATE, "dsx_pwg_load has not been called");
  DSX_CHECK(z && c && wav, DSX_E_INVALID, "z, c and wav must not be NULL");
  DSX_CHECK(B >= 1 && T >= 1, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  const dsx_pwg_config& cfg = h->cfg;
  const long long samples = static_cast<long long>(B) * T * h->hop;
  DSX_CHECK(samples <= kMaxSamples, DSX_E_INVALID, "B * T * hop = %lld samples is above the %lld a call takes", samples,
            kMaxSamples);
  DSX_CHECK(!cfg.use_pitch_embed || pitch, DSX_E_INVALID, "the generator has a pitch embedding: pitch is required");
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int L = T * h->hop, Tp = T + 2 * h->w, ns = cfg.num_scales;
  const size_t rows = static_cast<size_t>(samples);

  // workspace: fp32 x and skip, two fp16 copies of x, fp16 c_up, two fp32 stage buffers, c_proj's output
  int lmid = T;   // the longest stage input: conv_in's output or a stage before the last
  for (int i = 0; i + 1 < ns; ++i) lmid *= cfg.upsample_scales[i];
  const size_t stage_e = static_cast<size_t>(B) * lmid * kAux, cp_e = static_cast<size_t>(B) * Tp * kAux;
  DSX_TRY(h->ws.reserve(2 * align256(rows * kRes * 4) + 2 * align256(rows * kRes * 2) + align256(rows * kAux * 2) +
                            2 * align256(stage_e * 4) + (cfg.use_pitch_embed ? align256(cp_e * 4) : 0),
                        s));
  Bump ws{static_cast<uint8_t*>(h->ws.ptr)};
  float* X = ws.take<float>(rows * kRes * 4);
  float* SK = ws.take<float>(rows * kRes * 4);
  __half* XH[2] = {ws.take<__half>(rows * kRes * 2), ws.take<__half>(rows * kRes * 2)};
  __half* CUP = ws.take<__half>(rows * kAux * 2);
  float* U[2] = {ws.take<float>(stage_e * 4), ws.take<float>(stage_e * 4)};
  float* CP = cfg.use_pitch_embed ? ws.take<float>(cp_e * 4) : nullptr;

  dsx_strides in_s = cs;
  const float* in = c;
  if (cfg.use_pitch_embed) {
    const float* e = h->emb;
    k_pwg_cproj<<<grid_for(cp_e), 256, 0, s>>>(c, cs, pitch, e, e + kPitchBins * kAux, e + kPitchBins * kAux + 2 * kAux * kAux,
                                               B, Tp, CP);
    DSX_TRY(launch_check("k_pwg_cproj"));
    in = CP;
    in_s = dsx_strides{static_cast<int64_t>(Tp) * kAux, 1, kAux};
  }
  k_pwg_convin<<<grid_for(static_cast<size_t>(B) * T * kAux), 256, 0, s>>>(in, in_s, h->convin, 2 * h->w + 1, B, T, U[0]);
  DSX_TRY(launch_check("k_pwg_convin"));
  int lin = T;
  for (int i = 0; i < ns; ++i) {
    const int sc = cfg.upsample_scales[i];
    const bool last = i + 1 == ns;
    k_pwg_upsample<<<grid_for(static_cast<size_t>(B) * lin * sc * kAux), 256, 0, s>>>(
        U[i & 1], lin, sc, h->up + h->up_off[i], B, last ? nullptr : U[(i + 1) & 1], last ? CUP : nullptr);
    DSX_TRY(launch_check("k_pwg_upsample"));
    lin *= sc;
  }
  k_pwg_first<<<grid_for(rows * kRes), 256, 0, s>>>(z, h->first, rows, X, XH[0]);
  DSX_TRY(launch_check("k_pwg_first"));

  const int tpu = (L + kTileRows - 1) / kTileRows, tiles = B * tpu;
  const int ctas = std::min((tiles + 1) / 2, h->sms);
  const int lps = cfg.layers / cfg.stacks;
  for (int l = 0; l < cfg.layers; ++l) {
    LayerArgs a{};
    a.w = h->layer_w + static_cast<size_t>(l) * kLayerWeights;
    a.b = h->layer_b + l * 2 * kGate;
    a.xin = XH[l & 1];
    a.xout = XH[(l + 1) & 1];
    a.x = X;
    a.skip = SK;
    a.cup = CUP;
    a.L = L;
    a.d = 1 << (l % lps);
    a.tiles_per_utt = tpu;
    a.tiles = tiles;
    a.first = l == 0;
    a.last = l + 1 == cfg.layers;
    k_pwg_layer<<<ctas, 256, kLayerSmem, s>>>(a);
    DSX_TRY(launch_check("k_pwg_layer"));
  }
  const float scale = static_cast<float>(sqrt(1.0 / cfg.layers));
  k_pwg_head<<<grid_for(rows), 256, 0, s>>>(SK, h->head, scale, rows, wav);
  return launch_check("k_pwg_head");
}

}  // extern "C"
