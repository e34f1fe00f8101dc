// Training helpers shared by the DiffNet (dsx_train.cu), FastSpeech2 decoder (dsx_fs2train.cu), FFT denoiser
// (dsx_ffttrain.cu), duration predictor (dsx_durtrain.cu) and pitch predictor (dsx_pitchtrain.cu) training steps: the
// weight-gradient GEMM over the frame axis with its fixed-order split and reduction (run_wgrad: k_wgrad, k_wgrad_sum),
// the device-chosen power-of-two gradient scale with the tape's (B, T) check (run_scale: k_amax, k_scale), the tape
// header and dropout helpers (k_tape_hdr, hdr_drop, k_drop_masks) and the step-embedding MLP's backward (run_mlp_grad).
#pragma once
#include <algorithm>
#include <vector>

#include "dsx_internal.h"
#include "dsx_ptx.cuh"

namespace dsx {
namespace {   // every translation unit has its own copies, like dsx_conv.cuh

constexpr int kWgThreads = 256;

// ---- weight gradients: D[m][n] = sum over frames f of A[f][m] B[f + shift][n], both operands MN-major ----------------
struct WgradArgs {
  const __half* a;             // [F][lda], output rows m are its columns [0, am)
  int lda, am;
  const __half* b[4];          // per 256-column tile (blockIdx.y): source [F][ldb], shift in frames, valid columns
  int ldb[4], shift[4], bn[4];
  int F, T, fchunk;            // frames, frames per utterance, frames per split (a multiple of 64)
  float* part;                 // [splits][Mpad][Ntot]
  float* bpart;                // [splits][Mpad] column sums of A (blockIdx.y == 0), or null
  int Mpad, Ntot;
};

constexpr int kWgA = 64 * 128, kWgB = 64 * 128 * 4, kWgStage = kWgA + kWgB;
constexpr int kWgSmem = 2 * kWgStage + 1024;

__global__ void __launch_bounds__(kWgThreads) k_wgrad(const WgradArgs p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ float bsum[2][64];
  const int tid = threadIdx.x, wg = tid >> 7;
  const int mt = blockIdx.x, nt = blockIdx.y, split = blockIdx.z;
  const int f_begin = split * p.fchunk, f_end = min(p.F, f_begin + p.fchunk);
  const int chunks = (f_end - f_begin + 63) / 64;
  const __half* bsrc = p.b[nt];
  const int ldb = p.ldb[nt], shift = p.shift[nt], bn = p.bn[nt];

  auto load = [&](int s, uint8_t* buf) {
    const uint32_t da = smem_u32(buf), db = smem_u32(buf + kWgA);
    const int f0 = f_begin + s * 64;
    for (int i = tid; i < 64 * 8; i += kWgThreads) {          // A: 64 frames x 64 rows of the output
      const int k = i >> 3, c = i & 7, f = f0 + k, m = mt * 64 + c * 8;
      const bool ok = f < f_end && m < p.am;
      cp16(da + sw128(k, c), p.a + (ok ? static_cast<size_t>(f) * p.lda + m : 0), ok);
    }
    for (int i = tid; i < 64 * 32; i += kWgThreads) {         // B: 64 frames x 256 columns, four 64-column atoms
      const int k = i >> 5, c = i & 31, f = f0 + k, n = c * 8;
      bool ok = f < f_end && n < bn;
      int src = f + shift;
      if (ok && shift != 0) {
        const int t = f % p.T + shift;
        ok = t >= 0 && t < p.T;
      }
      cp16(db + (c >> 3) * 8192 + sw128(k, c & 7), bsrc + (ok ? static_cast<size_t>(src) * ldb + n : 0), ok);
    }
  };

  float acc[64];
#pragma unroll
  for (int e = 0; e < 64; ++e) acc[e] = 0.f;
  float bs = 0.f;                                              // column sum of A: thread tid < 128, row tid & 63
  if (chunks > 0) {
    load(0, smem);
    cp_commit();
  }
#pragma unroll 1
  for (int s = 0; s < chunks; ++s) {
    uint8_t* cur = smem + (s & 1) * kWgStage;
    if (s + 1 < chunks) {
      load(s + 1, smem + ((s + 1) & 1) * kWgStage);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    const uint32_t ua = smem_u32(cur), ub = smem_u32(cur + kWgA + wg * 2 * 8192);
    wg_fence();
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4)
      wgmma_n128_mn(acc, wg_desc_mn(ua + k4 * 2048, 8192), wg_desc_mn(ub + k4 * 2048, 8192), 1);
    wg_commit();
    if (p.bpart && nt == 0 && tid < 128) {
      const int m = tid & 63, k0 = (tid >> 6) * 32;
#pragma unroll 8
      for (int k = k0; k < k0 + 32; ++k)
        bs += __half2float(*reinterpret_cast<const __half*>(cur + sw128(k, m >> 3) + (m & 7) * 2));
    }
    wg_wait0();
#pragma unroll
    for (int e = 0; e < 64; ++e) asm volatile("" : "+f"(acc[e])::"memory");
    __syncthreads();
  }
  const int wtid = tid & 127;
  float* out = p.part + (static_cast<size_t>(split) * p.Mpad + mt * 64) * p.Ntot + nt * 256 + wg * 128;
#pragma unroll
  for (int e = 0; e < 64; e += 2) {
    const int r = acc_row(wtid, e), c = acc_col(wtid, e);
    *reinterpret_cast<float2*>(out + static_cast<size_t>(r) * p.Ntot + c) = make_float2(acc[e], acc[e + 1]);
  }
  if (p.bpart && nt == 0) {
    if (tid < 128) bsum[tid >> 6][tid & 63] = bs;
    __syncthreads();
    if (tid < 64) p.bpart[static_cast<size_t>(split) * p.Mpad + mt * 64 + tid] = bsum[0][tid] + bsum[1][tid];
  }
}

// Where the reduction of a wgrad's partials writes: column c < bn of B tile j of output row m goes to
// dst[j][m * ms[j] + c * cs[j]], times 1 / S unless raw[j]; the bias (the column sums of A) to db, times 1 / S unless
// db_raw, and times 1 / S to db2 (or null).  db null: no bias partials are computed.
struct WgradDst {
  float* dst[4];
  int ms[4], cs[4], raw[4];
  float *db, *db2;
  int db_raw;
};

struct WgradSumArgs {
  const float* part;           // k_wgrad's [splits][Mpad][Ntot]
  const float* bpart;          // and its [splits][Mpad] bias partials
  int splits, Mpad, Ntot, am;
  int ncol, bn[4];             // valid columns of all B tiles, of each
  WgradDst o;
  const float* scal;           // S, 1 / S
};

// each output is 0 plus the partials in split order, then times 1 / S once: no atomics, bitwise reproducible.  Thread i
// takes row m, then the tiles' columns in order, so concurrent CTAs read whole rows of the partials.
__global__ void k_wgrad_sum(const WgradSumArgs p) {
  const int total = p.am * p.ncol;
  const float is = p.scal[1];
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int m = i / p.ncol;
    int j = 0, c = i - m * p.ncol;
    while (c >= p.bn[j]) c -= p.bn[j++];
    float s = 0.f;
    for (int z = 0; z < p.splits; ++z) s += p.part[(static_cast<size_t>(z) * p.Mpad + m) * p.Ntot + j * 256 + c];
    p.o.dst[j][static_cast<size_t>(m) * p.o.ms[j] + static_cast<size_t>(c) * p.o.cs[j]] = p.o.raw[j] ? s : s * is;
  }
  if (p.o.db) {
    for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < p.am; m += gridDim.x * blockDim.x) {
      float s = 0.f;
      for (int z = 0; z < p.splits; ++z) s += p.bpart[static_cast<size_t>(z) * p.Mpad + m];
      p.o.db[m] = p.o.db_raw ? s : s * is;
      if (p.o.db2) p.o.db2[m] = s * is;
    }
  }
}

// ---- gradient scale: S from amax |g| ---------------------------------------------------------------------------------
__global__ void k_amax(const float* g, size_t n, unsigned* amax_bits) {
  float m = 0.f;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    m = fmaxf(m, fabsf(g[i]));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(amax_bits, __float_as_uint(m));   // max of non-negative floats: order-free
}

// scal[0] = S, scal[1] = 1 / S: S * amax in [2^5, 2^6); S = 1 when amax is 0 or not finite.  A backward over another
// (B, T) than its tape's (hdr non-null) would read the wrong regions: S = 1 / S = NaN then makes every gradient NaN.
__global__ void k_scale(const unsigned* amax_bits, float* scal, const Fs2TapeHdr* hdr, int B, int T) {
  if (hdr && (hdr->B != B || hdr->T != T)) {
    scal[0] = scal[1] = __int_as_float(0x7fc00000);
    return;
  }
  const float a = __uint_as_float(*amax_bits);
  int e = 0;
  if (a > 0.f && isfinite(a)) {
    frexpf(a, &e);                        // a in [2^(e-1), 2^e)
    e = min(max(6 - e, -126), 126);
  }
  scal[0] = ldexpf(1.f, e);
  scal[1] = ldexpf(1.f, -e);
}

// S from amax |g| over n values into scal (amax: a scratch word), checked against the tape's header hdr (or null)
int run_scale(const float* g, size_t n, unsigned* amax, float* scal, const Fs2TapeHdr* hdr, int B, int T,
              cudaStream_t s) {
  DSX_CUDA(cudaMemsetAsync(amax, 0, sizeof(unsigned), s));
  k_amax<<<static_cast<unsigned>(std::min<size_t>((n + 255) / 256, 1024)), 256, 0, s>>>(g, n, amax);
  DSX_TRY(launch_check("k_amax"));
  k_scale<<<1, 1, 0, s>>>(amax, scal, hdr, B, T);
  return launch_check("k_scale");
}

// ---- the tape's header and dropout ------------------------------------------------------------------------------------
__global__ void k_tape_hdr(Fs2TapeHdr* h, uint64_t seed, float p, int B, int T) {
  h->seed = seed;
  h->p = p;
  h->B = B;
  h->T = T;
}

// the dropout of site `site` as the tape's forward drew it
__device__ __forceinline__ Fs2Drop hdr_drop(const Fs2TapeHdr* h, int site) { return make_drop(h->seed, h->p, site); }

// out[f][c] = 1 where dropout d keeps element (f, c) of [F][n], else 0
__global__ void k_drop_masks(Fs2Drop d, size_t F, int n, uint8_t* out) {
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < F * n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    out[i] = dropout_scale(d, i / n, static_cast<int>(i % n)) != 0.f;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---- step-embedding MLP backward (mlp.0 -> Mish -> mlp.2 of C = residual_channels), from the saves of k_embed_table
// ([b][9 C]: sinusoid, mlp.0 output, Mish of it) and de = the gradient of the MLP's output, both scaled by S ----------
// mlp.2: dW2[c][j] = sum_b de[b][c] mish[b][j], db2 = sum_b de; dh[b][j] = (W2^T de)[j] * mish'(h[b][j]).  Thread j < 4C.
__global__ void k_mlp2_grad(const float* de, int B, int C, const float* save, const float* w2, const float* scal,
                            float* dw2, float* db2, float* dh) {
  const float is = scal[1];
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= 4 * C) return;
  for (int b = 0; b < B; ++b) {
    const float* sv = save + static_cast<size_t>(b) * 9 * C;
    float g = 0.f;
    for (int c = 0; c < C; ++c) g = fmaf(w2[static_cast<size_t>(c) * 4 * C + j], de[b * C + c], g);
    const float x = sv[C + j];
    const float sp = x > 20.f ? x : log1pf(expf(x));
    const float th = tanhf(sp);
    const float dsp = x > 20.f ? 1.f : 1.f / (1.f + expf(-x));
    dh[b * 4 * C + j] = g * (th + x * (1.f - th * th) * dsp);
  }
  if (j < C) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += de[b * C + j];
    db2[j] = s * is;
  }
  // dW2 [C][4C]: this thread's column j for every row c
  for (int c = 0; c < C; ++c) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s = fmaf(de[b * C + c], save[static_cast<size_t>(b) * 9 * C + 5 * C + j], s);
    dw2[static_cast<size_t>(c) * 4 * C + j] = s * is;
  }
}

// mlp.0: dW0[j][k] = sum_b dh[b][j] sinusoid[b][k], db0[j] = sum_b dh[b][j].  Block j, thread k.
__global__ void k_mlp0_grad(const float* dh, int B, int C, const float* save, const float* scal, float* dw0,
                            float* db0) {
  const int j = blockIdx.x, k = threadIdx.x;
  const float is = scal[1];
  float s = 0.f, sb = 0.f;
  for (int b = 0; b < B; ++b) {
    const float d = dh[b * 4 * C + j];
    s = fmaf(d, save[static_cast<size_t>(b) * 9 * C + k], s);
    sb += d;
  }
  dw0[static_cast<size_t>(j) * C + k] = s * is;
  if (k == 0) db0[j] = sb * is;
}

// both, with dh [B][4 C] as scratch (C <= 1024)
int run_mlp_grad(const float* de, int B, int C, const float* save, const float* w2, const float* scal, float* dw2,
                 float* db2, float* dh, float* dw0, float* db0, cudaStream_t s) {
  k_mlp2_grad<<<(4 * C + 255) / 256, 256, 0, s>>>(de, B, C, save, w2, scal, dw2, db2, dh);
  DSX_TRY(launch_check("k_mlp2_grad"));
  k_mlp0_grad<<<4 * C, C, 0, s>>>(dh, B, C, save, scal, dw0, db0);
  return launch_check("k_mlp0_grad");
}

int sm_count(int device) {
  int n = 0;
  cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device);
  return n > 0 ? n : 132;
}

// frames per split of a wgrad over F frames with `tiles` output tiles: about two CTAs per SM in all
int wgrad_fchunk(int F, int tiles, int device) {
  const int fch = (F + 63) / 64;
  const int sp = std::max(1, std::min(fch, (2 * sm_count(device) + tiles - 1) / tiles));
  return ((fch + sp - 1) / sp) * 64;
}

// floats of the largest partial buffer (weights, then bias) among wgrads over F frames of these (m tiles, n tiles)
size_t wgrad_part_floats(int F, const std::vector<std::pair<int, int>>& shapes, int device) {
  size_t worst = 0;
  for (const auto& [mt, nt] : shapes) {
    const int fchunk = wgrad_fchunk(F, mt * nt, device);
    const size_t sp = (F + fchunk - 1) / fchunk;
    worst = std::max(worst, sp * mt * 64 * nt * 256 + sp * mt * 64);
  }
  return worst;
}

// D[am x ntiles*256] = A^T B over a.F frames (a's operands and tiles set) into o, scaled by scal[1] as o says: k_wgrad's
// split partials in part (wgrad_part_floats), then k_wgrad_sum
int run_wgrad(WgradArgs a, int ntiles, const WgradDst& o, float* part, const float* scal, int device, cudaStream_t s) {
  const int mtiles = (a.am + 63) / 64;
  a.fchunk = wgrad_fchunk(a.F, mtiles * ntiles, device);
  const int sp = (a.F + a.fchunk - 1) / a.fchunk;
  a.part = part;
  a.Mpad = mtiles * 64;
  a.Ntot = ntiles * 256;
  a.bpart = o.db ? part + static_cast<size_t>(sp) * a.Mpad * a.Ntot : nullptr;   // the bias partials follow the weights'
  k_wgrad<<<dim3(mtiles, ntiles, sp), kWgThreads, kWgSmem, s>>>(a);
  DSX_TRY(launch_check("k_wgrad"));
  WgradSumArgs r{};
  r.part = part;
  r.bpart = a.bpart;
  r.splits = sp;
  r.Mpad = a.Mpad;
  r.Ntot = a.Ntot;
  r.am = a.am;
  for (int j = 0; j < ntiles; ++j) r.ncol += (r.bn[j] = a.bn[j]);
  r.o = o;
  r.scal = scal;
  const size_t total = static_cast<size_t>(a.am) * r.ncol;
  k_wgrad_sum<<<static_cast<unsigned>(std::min<size_t>((total + 255) / 256, 4096)), 256, 0, s>>>(r);
  return launch_check("k_wgrad_sum");
}

}  // namespace
}  // namespace dsx
