// Counter-based noise generator shared by the sampler kernels.
#pragma once
#include <stdint.h>

namespace dsx {

// ------------------------------------------------------------------------------------------
// Philox4x32-10 + Box-Muller (perf-mode noise; distribution-equal to torch.randn, not stream-equal)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}
__device__ __forceinline__ float2 box_muller(uint32_t a, uint32_t b) {
  // u1 in (0,1], u2 in [0,1)
  float u1 = (static_cast<float>(a) + 1.0f) * 2.3283064365386963e-10f;
  float u2 = static_cast<float>(b) * 2.3283064365386963e-10f;
  // fast intrinsics (MUFU.LG2 / SIN / COS): |error| ~1e-6, far below what a sampler can resolve
  // (sqrt.approx: one MUFU; sqrtf() with IEEE rounding is a 15-instruction sequence with a slow-path call, per draw)
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(-2.0f * __logf(u1)));
  float s, c;
  __sincosf(6.283185307179586f * u2, &s, &c);
  return make_float2(r * c, r * s);
}
__device__ __forceinline__ float philox_normal(uint64_t seed, uint64_t offset, size_t i) {
  uint4 ctr = make_uint4(static_cast<uint32_t>(i >> 2), static_cast<uint32_t>((i >> 2) >> 32),
                         static_cast<uint32_t>(offset), static_cast<uint32_t>(offset >> 32));
  uint4 r = philox4x32_10(ctr, make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)));
  float2 n01 = box_muller(r.x, r.y), n23 = box_muller(r.z, r.w);
  switch (i & 3) {
    case 0: return n01.x;
    case 1: return n01.y;
    case 2: return n23.x;
    default: return n23.y;
  }
}


// Four normals from one Philox block.  Sampler noise for mel element (b, m, t) of a [B][M][T] tensor is lane (m & 3)
// of block ((b * (M/4) + m/4) * T + t), so a thread that owns one frame draws four bins per call.
__device__ __forceinline__ float4 philox_normal4(uint64_t seed, uint64_t offset, size_t blk) {
  uint4 ctr = make_uint4(static_cast<uint32_t>(blk), static_cast<uint32_t>(blk >> 32),
                         static_cast<uint32_t>(offset), static_cast<uint32_t>(offset >> 32));
  uint4 r = philox4x32_10(ctr, make_uint2(static_cast<uint32_t>(seed), static_cast<uint32_t>(seed >> 32)));
  float2 n01 = box_muller(r.x, r.y), n23 = box_muller(r.z, r.w);
  return make_float4(n01.x, n01.y, n23.x, n23.y);
}
__device__ __forceinline__ size_t mel_noise_block(int b, int m, int t, int M, int T) {
  return (static_cast<size_t>(b) * (M >> 2) + (m >> 2)) * T + t;
}

// ------------------------------------------------------------------------------------------
// Dropout masks of the training steps: element (frame, channel) of dropout site `site` is kept when the 24-bit uniform u
// of lane channel % 4 of the Philox4x32-10 block (channel / 4, frame, site, 0) under key seed is >= p, so
// P(keep) = 1 - p to 2^-24 (torch's distribution, not its stream).  Kept elements are scaled by inv_keep = 1 / (1 - p).
// ------------------------------------------------------------------------------------------
struct Fs2Drop {
  uint64_t seed = 0;
  float p = 0.f, inv_keep = 1.f;
  int site = -1;                 // < 0: no dropout (scale 1)
};
__host__ __device__ __forceinline__ Fs2Drop make_drop(uint64_t seed, float p, int site) {
  Fs2Drop d;
  d.seed = seed;
  d.p = p;
  d.inv_keep = 1.f / (1.f - p);
  d.site = site;
  return d;
}
__device__ __forceinline__ uint4 dropout_block(const Fs2Drop& d, size_t frame, int channel) {
  const uint4 ctr = make_uint4(static_cast<uint32_t>(channel >> 2), static_cast<uint32_t>(frame),
                               static_cast<uint32_t>(d.site), static_cast<uint32_t>(frame >> 32));
  return philox4x32_10(ctr, make_uint2(static_cast<uint32_t>(d.seed), static_cast<uint32_t>(d.seed >> 32)));
}
__device__ __forceinline__ float dropout_lane(const Fs2Drop& d, const uint4& r, int lane) {
  const uint32_t v = lane == 0 ? r.x : lane == 1 ? r.y : lane == 2 ? r.z : r.w;
  return static_cast<float>(v >> 8) * 5.9604644775390625e-8f >= d.p ? d.inv_keep : 0.f;
}
// the factor of element (frame, channel): 0 or inv_keep, or 1 without dropout
__device__ __forceinline__ float dropout_scale(const Fs2Drop& d, size_t frame, int channel) {
  if (d.site < 0) return 1.f;
  return dropout_lane(d, dropout_block(d, frame, channel), channel & 3);
}
// the factors of channels c and c + 1 (c even)
__device__ __forceinline__ float2 dropout_scale2(const Fs2Drop& d, size_t frame, int c) {
  if (d.site < 0) return make_float2(1.f, 1.f);
  const uint4 r = dropout_block(d, frame, c);
  return make_float2(dropout_lane(d, r, c & 3), dropout_lane(d, r, (c & 3) + 1));
}

}  // namespace dsx
