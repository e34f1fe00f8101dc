// SSIM mel loss on sm_90a: the reference's ssim(img1, img2, window_size=11) (modules/commons/ssim.py:319-391) over
// single-channel [B, 1, H, W] images, forward and backward, in fp32 on CUDA cores.
//
// The 11 x 11 window is the outer product of the 1-D Gaussian g (sigma 1.5), so every blur runs as an 11-tap vertical
// pass and an 11-tap horizontal one, both zero-padded by 5.  Each CTA owns whole rows (W <= 256) of one image for a tile
// of TH rows; everything between the two global reads and the global write stays in shared memory.
//   k_ssim_fwd   rows [h0, h0 + TH): the vertical pass of x, y, x^2, y^2, xy from global, then the horizontal pass and
//                the SSIM formula -> map
//   k_ssim_bwd   the five moments on rows [h0 - 5, h0 + TH + 5) (inputs from rows h0 - 10 .. h0 + TH + 9), from them
//                and d_map the per-pixel partials a1 = d dS/dmu1, a2 = d dS/dmu2, b = 2 d dS/ds11 (= 2 d dS/ds22) and
//                c = d dS/ds12, then their blur (the window is symmetric and zero padding transposes to zero padding):
//                d_x = G*a1 + x G*b + y G*c, d_y = G*a2 + y G*b + x G*c
// No workspace, atomics or handle.  Every output pixel is computed by the same sequence of operations whatever the tile,
// the batch or the call, so results are bitwise reproducible and a batch gives each image's bits alone.  The moments are
// not shifted: the caller's bias (6 for mels) leaves s11 = G*(x^2) near 36, whose fp32 rounding (~4e-6) sits well below
// C2 = 9e-4; TF32's (~4e-2) would not.
#include "dsx_internal.h"

namespace dsx {
namespace {

constexpr int kHalf = 5;
constexpr int kThreads = 256;
constexpr int kMaxW = 256;
constexpr int kSmemFloats = 24576;      // 96 KB per CTA, two CTAs per SM, for the tile sizes below
constexpr int kMinRows = 8, kMaxRows = 64;
constexpr float kC1 = static_cast<float>(0.01 * 0.01);
constexpr float kC2 = static_cast<float>(0.03 * 0.03);

// gaussian(11, 1.5) as the reference computes it: exp() in double, rounded to float32, divided by the float32 sum
__constant__ float kG[2 * kHalf + 1] = {0x1.0d956cp-10f, 0x1.f1fe02p-8f, 0x1.26eb18p-5f, 0x1.bff0fep-4f,
                                        0x1.b43c3ep-3f,  0x1.106560p-2f, 0x1.b43c3ep-3f, 0x1.bff0fep-4f,
                                        0x1.26eb18p-5f,  0x1.f1fe02p-8f, 0x1.0d956cp-10f};

// vertical 11-tap pass of x, y, x^2, y^2, xy at (r, w) of one image, zero outside rows [0, H)
__device__ __forceinline__ void vblur(const float* __restrict__ x, const float* __restrict__ y, int r, int w, int H,
                                      int W, float v[5]) {
#pragma unroll
  for (int k = 0; k < 5; ++k) v[k] = 0.f;
#pragma unroll
  for (int j = 0; j <= 2 * kHalf; ++j) {
    const int rr = r + j - kHalf;
    if (rr < 0 || rr >= H) continue;
    const size_t o = static_cast<size_t>(rr) * W + w;
    const float a = __ldg(x + o), c = __ldg(y + o), g = kG[j];
    v[0] += g * a;
    v[1] += g * c;
    v[2] += g * (a * a);
    v[3] += g * (c * c);
    v[4] += g * (a * c);
  }
}

// horizontal 11-tap pass at column w of N fields (row pointer `row`, field stride fs), zero outside columns [0, W)
template <int N>
__device__ __forceinline__ void hblur(const float* row, int fs, int w, int W, float out[N]) {
#pragma unroll
  for (int k = 0; k < N; ++k) out[k] = 0.f;
#pragma unroll
  for (int j = 0; j <= 2 * kHalf; ++j) {
    const int c = w + j - kHalf;
    if (c < 0 || c >= W) continue;
    const float g = kG[j];
#pragma unroll
    for (int k = 0; k < N; ++k) out[k] += g * row[k * fs + c];
  }
}

// the reference's _ssim formula (ssim.py:335-346) on the moments m = (mu1, mu2, G*x^2, G*y^2, G*xy).  The products are
// rounded before they are subtracted, as in the reference, not fused: then x = y gives A1 = B1 and A2 = B2 bit for bit,
// and the map exactly 1, where a fused multiply-add on one side only would leave the rounding of mu^2 in sigma^2.
struct SsimTerms {
  float mu1, mu2, A1, A2, B1, B2;
  __device__ __forceinline__ explicit SsimTerms(const float m[5]) : mu1(m[0]), mu2(m[1]) {
    const float mu1_sq = __fmul_rn(mu1, mu1), mu2_sq = __fmul_rn(mu2, mu2), mu1_mu2 = __fmul_rn(mu1, mu2);
    A1 = 2.f * mu1_mu2 + kC1;
    A2 = 2.f * (m[4] - mu1_mu2) + kC2;
    B1 = mu1_sq + mu2_sq + kC1;
    B2 = (m[2] - mu1_sq) + (m[3] - mu2_sq) + kC2;
  }
  __device__ __forceinline__ float value() const { return (A1 * A2) / (B1 * B2); }
};

__global__ void __launch_bounds__(kThreads) k_ssim_fwd(const float* __restrict__ x, const float* __restrict__ y, int H,
                                                       int W, int TH, int tiles, float* __restrict__ map) {
  extern __shared__ float sm[];                      // [5][TH][W] vertical passes
  const int h0 = (blockIdx.x % tiles) * TH;
  const size_t img = static_cast<size_t>(blockIdx.x / tiles) * H * W;
  const int fs = TH * W, n = min(TH, H - h0) * W;
  x += img;
  y += img;
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const int r = i / W, w = i - r * W;
    float v[5];
    vblur(x, y, h0 + r, w, H, W, v);
#pragma unroll
    for (int k = 0; k < 5; ++k) sm[k * fs + i] = v[k];
  }
  __syncthreads();
  map += img + static_cast<size_t>(h0) * W;
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const int r = i / W, w = i - r * W;
    float m[5];
    hblur<5>(sm + r * W, fs, w, W, m);
    map[i] = SsimTerms(m).value();
  }
}

__global__ void __launch_bounds__(kThreads) k_ssim_bwd(const float* __restrict__ x, const float* __restrict__ y,
                                                       const float* __restrict__ dmap, int H, int W, int TH, int tiles,
                                                       float* __restrict__ dx, float* __restrict__ dy) {
  extern __shared__ float sm[];                      // V [5][R][W] moments, P [4][R][W] partials; Q [4][TH][W] over V
  const int h0 = (blockIdx.x % tiles) * TH;
  const size_t img = static_cast<size_t>(blockIdx.x / tiles) * H * W;
  const int R = TH + 2 * kHalf, fs = R * W, base = h0 - kHalf;   // smem row i holds image row base + i
  float* V = sm;
  float* P = sm + 5 * fs;
  x += img;
  y += img;
  dmap += img;
  const int lo = max(base, 0), n1 = (min(h0 + TH + kHalf, H) - lo) * W;
  for (int i = threadIdx.x; i < n1; i += kThreads) {
    const int r = lo + i / W, w = i % W;
    float v[5];
    vblur(x, y, r, w, H, W, v);
#pragma unroll
    for (int k = 0; k < 5; ++k) V[k * fs + (r - base) * W + w] = v[k];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n1; i += kThreads) {
    const int r = lo + i / W, w = i % W;
    const int o = (r - base) * W + w;
    float m[5];
    hblur<5>(V + (r - base) * W, fs, w, W, m);
    const SsimTerms t(m);
    const float D = t.B1 * t.B2, S = (t.A1 * t.A2) / D;
    const float e = (t.A2 - t.A1) / D, q = S * (1.f / t.B1 - 1.f / t.B2);
    const float d = dmap[static_cast<size_t>(r) * W + w];
    P[o] = d * (2.f * (t.mu2 * e - t.mu1 * q));        // dS/dmu1
    P[fs + o] = d * (2.f * (t.mu1 * e - t.mu2 * q));   // dS/dmu2
    P[2 * fs + o] = d * (-2.f * S / t.B2);             // 2 dS/ds11 = 2 dS/ds22
    P[3 * fs + o] = d * (2.f * t.A1 / D);              // dS/ds12
  }
  __syncthreads();
  const int fq = TH * W, n2 = min(TH, H - h0) * W;
  for (int i = threadIdx.x; i < n2; i += kThreads) {
    const int r = h0 + i / W, w = i % W;
    float q[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j <= 2 * kHalf; ++j) {
      const int rr = r + j - kHalf;
      if (rr < 0 || rr >= H) continue;
      const float g = kG[j];
#pragma unroll
      for (int k = 0; k < 4; ++k) q[k] += g * P[k * fs + (rr - base) * W + w];
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) V[k * fq + i] = q[k];
  }
  __syncthreads();
  const size_t out = static_cast<size_t>(h0) * W;
  for (int i = threadIdx.x; i < n2; i += kThreads) {
    const int r = i / W, w = i - r * W;
    float q[4];
    hblur<4>(V + r * W, fq, w, W, q);
    const float a = x[out + i], c = y[out + i];
    if (dx) dx[img + out + i] = q[0] + a * q[2] + c * q[3];
    if (dy) dy[img + out + i] = q[1] + c * q[2] + a * q[3];
  }
}

int ssim_check(const float* x, const float* y, int B, int H, int W) {
  DSX_CHECK(x && y, DSX_E_INVALID, "x and y must not be NULL");
  DSX_CHECK(B >= 1 && H >= 1 && W >= 1 && W <= kMaxW, DSX_E_INVALID,
            "ssim needs B >= 1, H >= 1 and 1 <= W <= %d (got B %d, H %d, W %d)", kMaxW, B, H, W);
  return DSX_OK;
}

// rows per tile: as many as kSmemFloats holds (at least kMinRows, at most kMaxRows and H)
int tile_rows(int fields, int halo, int W, int H) {
  return min(H, max(kMinRows, min(kMaxRows, kSmemFloats / (fields * W) - halo)));
}

int launch_grid(int B, int H, int TH, int* tiles, unsigned* grid) {
  *tiles = (H + TH - 1) / TH;
  const long long n = static_cast<long long>(B) * *tiles;
  DSX_CHECK(n <= 0x7fffffffll, DSX_E_INVALID, "ssim: B * ceil(H / %d) = %lld tiles is above the launch grid's limit", TH,
            n);
  *grid = static_cast<unsigned>(n);
  return DSX_OK;
}

}  // namespace
}  // namespace dsx

using namespace dsx;

extern "C" {

int dsx_ssim_forward(const float* x, const float* y, int B, int H, int W, float* map, void* stream) {
  DSX_TRY(ssim_check(x, y, B, H, W));
  DSX_CHECK(map, DSX_E_INVALID, "map must not be NULL");
  const int TH = tile_rows(5, 0, W, H);
  int tiles;
  unsigned grid;
  DSX_TRY(launch_grid(B, H, TH, &tiles, &grid));
  const size_t smem = sizeof(float) * 5 * TH * W;
  DSX_CUDA(cudaFuncSetAttribute(k_ssim_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  k_ssim_fwd<<<grid, kThreads, smem, static_cast<cudaStream_t>(stream)>>>(x, y, H, W, TH, tiles, map);
  return launch_check("k_ssim_fwd");
}

int dsx_ssim_backward(const float* x, const float* y, const float* d_map, int B, int H, int W, float* d_x, float* d_y,
                      void* stream) {
  DSX_TRY(ssim_check(x, y, B, H, W));
  DSX_CHECK(d_map, DSX_E_INVALID, "d_map must not be NULL");
  if (!d_x && !d_y) return DSX_OK;
  const int TH = tile_rows(9, 2 * kHalf, W, H);
  int tiles;
  unsigned grid;
  DSX_TRY(launch_grid(B, H, TH, &tiles, &grid));
  const size_t smem = sizeof(float) * 9 * (TH + 2 * kHalf) * W;
  DSX_CUDA(cudaFuncSetAttribute(k_ssim_bwd, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  k_ssim_bwd<<<grid, kThreads, smem, static_cast<cudaStream_t>(stream)>>>(x, y, d_map, H, W, TH, tiles, d_x, d_y);
  return launch_check("k_ssim_bwd");
}

}  // extern "C"
