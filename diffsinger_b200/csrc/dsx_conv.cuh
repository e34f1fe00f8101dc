// Implicit-GEMM convolution core of the vocoder (dsx_hifigan.cu), the pitch extractor (dsx_pe.cu) and the FastSpeech2
// decoder (dsx_fs2dec.cu): the packed weight layout, its pack kernel and the K loop of one 64-row tile.  The epilogues
// are the callers' own.
//
// Activations are frames-major fp16 [B][L][cin], cin 80 or a multiple of 16.  Row m of the GEMM is an output position; the
// K axis is (tap j, input channel c), kk = j * cin + c, and tap j reads input row m + tap0 + j * tstep, zero outside the
// utterance's valid rows [0, valid_rows), which is the conv's zero padding.  Weights are packed fp16 [ntiles][kc][nt][64]
// (column tile, 64-wide K chunk, column, K inside the chunk), zero padded.  A CTA covers 64 rows and one column tile of NT
// columns; its WG warpgroups share the A tile and own NT / WG columns each.  Operands reach shared memory by cp.async in
// the 128-byte-swizzled layout of dsx_ptx.cuh, two stages deep: chunk s + 1 loads while chunk s runs four m64k16 wgmmas.
#pragma once
#include <algorithm>
#include <type_traits>

#include "dsx_internal.h"
#include "dsx_ptx.cuh"

namespace dsx {
namespace {   // every translation unit has its own k_pack_conv

constexpr int kConvRows = 64;   // GEMM rows per CTA

// sum over the 4 threads of an accumulator quad (they hold the same two rows)
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  return v;
}

// one convolution packed for the implicit GEMM
struct ConvGemm {
  int cin = 0;                       // input channels as stored in the operand
  int n = 0;                         // GEMM columns
  int taps = 0, tap0 = 0, tstep = 1;
  int nt = 0, ntiles = 0, kc = 0;    // columns per tile, column tiles, 64-wide K chunks
  __half* w = nullptr;               // [ntiles][kc][nt][64] fp16
  float* b = nullptr;                // [ntiles * nt], 0 past the bias
};

// the smallest tile width of 16, 32, 64, ... nt_max that holds n columns, else nt_max
inline int conv_nt(int n, int nt_max) {
  int nt = 16;
  while (nt < n && nt < nt_max) nt *= 2;
  return nt;
}

// two operand stages and the slack that aligns them to 1024 bytes
template <int NT>
constexpr int conv_smem() { return 2 * (kConvRows * 128 + NT * 128) + 1024; }

// f(std::integral_constant<int, NT>()) for tile width nt, NT instantiated for 16 .. NT_MAX
template <int NT_MAX, typename F>
int conv_dispatch(int nt, F&& f) {
  switch (nt) {
    case 16: return f(std::integral_constant<int, 16>());
    case 32: return f(std::integral_constant<int, 32>());
    case 64: return f(std::integral_constant<int, 64>());
  }
  if constexpr (NT_MAX > 128) {
    if (nt > 128) return f(std::integral_constant<int, 256>());
  }
  return f(std::integral_constant<int, 128>());
}

// opts kernel_of(integral_constant NT) in to conv_smem<NT>() bytes of dynamic shared memory for every NT up to NT_MAX
template <int NT_MAX, typename K>
int conv_opt_in(K kernel_of) {
  for (int nt = 16; nt <= NT_MAX; nt *= 2) {
    DSX_TRY(conv_dispatch<NT_MAX>(nt, [&](auto c) {
      DSX_CUDA(cudaFuncSetAttribute(kernel_of(c), cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    conv_smem<decltype(c)::value>()));
      return DSX_OK;
    }));
  }
  return DSX_OK;
}

// acc (this warpgroup's NT / WG columns) = A . B over all g.kc chunks, or acc += A . B with `accumulate` (a second
// operand pair summed into the same accumulators).  A is the 64 rows from m0 of utterance b of x [B][lx][g.cin]; B is
// column tile `tile` of g.w.  smem: conv_smem<NT>() bytes, 1024-byte aligned.
template <int NT, int WG>
__device__ __forceinline__ void conv_k_loop(const ConvGemm& g, const __half* x, int lx, int valid_rows, int b, int m0,
                                            int tile, uint8_t* smem, float (&acc)[NT / WG / 2], bool accumulate = false) {
  constexpr int NH = NT / WG, NTHR = 128 * WG, kA = kConvRows * 128, kStage = kA + NT * 128;
  const int tid = threadIdx.x, wg = WG > 1 ? tid >> 7 : 0;   // a constant 0 keeps the wgmma descriptors uniform
  auto load = [&](int s, uint8_t* buf) {
    const uint32_t da = smem_u32(buf), db = smem_u32(buf + kA);
#pragma unroll
    for (int q = 0; q < kConvRows * 8 / NTHR; ++q) {
      const int i = tid + q * NTHR, r = i >> 3, c = i & 7;
      const int kk = s * 64 + c * 8, j = kk / g.cin, ch = kk - j * g.cin;
      const int src = m0 + r + g.tap0 + j * g.tstep;
      const bool valid = j < g.taps && src >= 0 && src < valid_rows;
      cp16(da + sw128(r, c), x + (static_cast<size_t>(b) * lx + (valid ? src : 0)) * g.cin + (valid ? ch : 0), valid);
    }
    const __half* wsrc = g.w + (static_cast<size_t>(tile) * g.kc + s) * NT * 64;
    for (int i = tid; i < NT * 8; i += NTHR) {
      const int r = i >> 3, c = i & 7;
      cp16(db + sw128(r, c), wsrc + r * 64 + c * 8, true);
    }
  };

  if (!accumulate) {
#pragma unroll
    for (int e = 0; e < NH / 2; ++e) acc[e] = 0.f;
  }
  load(0, smem);
  cp_commit();
#pragma unroll 1
  for (int s = 0; s < g.kc; ++s) {
    uint8_t* cur = smem + (s & 1) * kStage;
    if (s + 1 < g.kc) {
      load(s + 1, smem + ((s + 1) & 1) * kStage);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    const uint64_t da = wg_desc(smem_u32(cur)), db = wg_desc(smem_u32(cur + kA + wg * NH * 128));
    wg_fence();
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) wgmma_f16<NH>(acc, da + 2 * k4, db + 2 * k4, 1);
    wg_commit();
    wg_wait0();
#pragma unroll
    for (int e = 0; e < NH / 2; ++e) asm volatile("" : "+f"(acc[e])::"memory");
    __syncthreads();
  }
}

// ---- weight packing ------------------------------------------------------------------------------
struct PackArgs {
  const float* v;              // Conv1d [cout][cin][k], or ConvTranspose1d [cin][cout][k] in polyphase form
  const float* scale;          // per index of dim 0 (weight norm), or null: unscaled
  const float* bias;           // [cout], or null: no bias
  int cin, cout, cout_p, k, u, transposed;   // cout_p: columns per ConvTranspose1d phase (column n = r cout_p + o)
};

// W (* scale) -> g.w, zero padded; bias -> g.b
__global__ void k_pack_conv(const ConvGemm g, const PackArgs p) {
  const size_t total = static_cast<size_t>(g.ntiles) * g.kc * g.nt * 64;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(i & 63);
    size_t t = i >> 6;
    const int rr = static_cast<int>(t % g.nt);
    t /= g.nt;
    const int s = static_cast<int>(t % g.kc);
    const int tile = static_cast<int>(t / g.kc);
    const int n = tile * g.nt + rr, kk = s * 64 + q, j = kk / g.cin, c = kk - j * g.cin;
    float val = 0.f;
    if (n < g.n && j < g.taps && c < p.cin) {
      if (p.transposed) {
        const int r = n / p.cout_p, o = n - r * p.cout_p;
        if (o < p.cout) {
          val = p.v[(static_cast<size_t>(c) * p.cout + o) * p.k + r + j * p.u];
          if (p.scale) val *= p.scale[c];
        }
      } else if (n < p.cout) {
        val = p.v[(static_cast<size_t>(n) * p.cin + c) * p.k + j];
        if (p.scale) val *= p.scale[n];
      }
    }
    g.w[i] = __float2half_rn(val);
    if (i < static_cast<size_t>(g.ntiles) * g.nt) {
      const int nn = static_cast<int>(i), o = nn % p.cout_p;
      g.b[nn] = (nn < g.n && o < p.cout && p.bias) ? p.bias[o] : 0.f;
    }
  }
}

// Sizes g's tiles (g.cin, g.n and g.taps set, tile width at most nt_max) and allocates its packs in mem.
inline int conv_alloc(DevAllocs& mem, ConvGemm& g, int nt_max) {
  g.nt = conv_nt(g.n, nt_max);
  g.ntiles = (g.n + g.nt - 1) / g.nt;
  g.kc = (g.taps * g.cin + 63) / 64;
  DSX_TRY(mem.alloc(&g.w, static_cast<size_t>(g.ntiles) * g.kc * g.nt * 64 * sizeof(__half)));
  return mem.alloc(&g.b, static_cast<size_t>(g.ntiles) * g.nt * sizeof(float));
}

// (Re)fills g's allocated packs on the stream.
inline int conv_repack(const ConvGemm& g, const PackArgs& a, cudaStream_t s) {
  const size_t nw = static_cast<size_t>(g.ntiles) * g.kc * g.nt * 64;
  const int blocks = static_cast<int>(std::min<size_t>((nw + 255) / 256, 4096));
  k_pack_conv<<<blocks, 256, 0, s>>>(g, a);
  return launch_check("k_pack_conv");
}

// conv_alloc, then conv_repack.
inline int conv_pack(DevAllocs& mem, ConvGemm& g, int nt_max, const PackArgs& a, cudaStream_t s) {
  DSX_TRY(conv_alloc(mem, g, nt_max));
  return conv_repack(g, a, s);
}

}  // namespace
}  // namespace dsx
