// Tensor-core path of the dsx sampler for Hopper (sm_90a): warpgroup MMA (wgmma.mma_async, fp16 operands from shared
// memory, fp32 accumulators in registers).  Two kernels:
//   k_hp_step<NWG>   residual layers [l0, l1) of one DiffNet evaluation (usr/diff/net.py:58-78) and, optionally, what
//                    follows them in a diffusion step: skip / output projections, the DDPM or PNDM update and the next
//                    evaluation's input projection (net.py:115-130, shallow_diffusion_tts.py:134-199).  Persistent and
//                    cooperative: every CTA walks over the frame tiles of a layer, and a tile starts layer l+1 once its
//                    neighbour tiles, whose conv input it reads, have published layer l (wait_layer).
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
// Operands reach shared memory in the 128-byte-swizzled K-major layout wgmma reads (dsx_ptx.cuh) through a ring of R
// stages: one stage = a 256-row x 64-k weight tile (32 KB, shared by the warpgroups), packed already swizzled and moved
// by one bulk copy, + the A operands that are not resident: 64 x 64 activation blocks per warpgroup, copied by cp.async
// (zero-filled outside [0, T)).  Each slot has a full barrier (the bulk copy's bytes and one arrival per thread, after
// its cp.async if it copied a block) and an empty barrier (one arrival per warpgroup when its MMAs of the slot are done).
// The ring runs on across GEMM phases: before an epilogue starts, the first R stages of the next phase are issued, so
// the weight stream does not stop while the epilogues run.  With P <= 2 (R = 3) GEMM1's taps are not streamed: the
// tile's conv input, frames t0 - 8 .. t0 + 64 NWG + 8, is copied once into a resident window, and tap j's A descriptor
// starts (j - 1) d rows away from the warpgroup's rows.  Both chunks read it, so each element of y crosses L2 -> SM once
// per layer instead of six times.  fp16x3 (R = 2) reads y's lo plane too and keeps streaming its taps.
// Each warpgroup's rows go through the same instruction sequence whatever NWG is, so 64- and 128-frame CTAs give
// bit-identical results.  While GEMM1 runs, the warpgroup prefetches the CP rows its gate epilogues read into L2,
// and the epilogues issue their global loads in batches ahead of their stores: every operand of a batch, including the
// residual and skip epilogues' bias and FiLM pairs, is loaded before the batch's first store.
//
// Precision (MMA passes P per k-block): P = 1 fp16 operands; P = 2 adds a W_lo pass (weights as hi+lo fp16 pairs);
// P = 3 accumulates A_hi*W_hi + A_hi*W_lo + A_lo*W_hi (~2^-22 relative).  The conditioner projection is always 3-pass.
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "dsx_internal.h"
#include "dsx_ptx.cuh"
#include "dsx_rng.cuh"

namespace dsx {

constexpr int kC = 256;                   // residual / conditioner channels supported by this path
constexpr int kRowsPerLayer = 80 * 256;    // wpack rows (of 64 fp16) per layer: 64 W1 tiles + 16 W2 tiles of 256 rows
constexpr int kSrRowsPerLayer = 32 * 256;  // rows per layer of one stochastically rounded weight set: 24 W1 + 8 W2 tiles
constexpr int kWBytes = 256 * 128;         // one weight tile: 256 rows x 64 fp16
constexpr int kABytes = 64 * 128;          // one activation block: 64 rows x 64 fp16
constexpr int kZBytes = 4 * kABytes;       // one plane (4 k-blocks) of a warpgroup's z / h / x_in operand
constexpr int kEpiBatch = 8;               // accumulator pairs whose global loads a layer epilogue issues at once

constexpr int kHalo = 8;                   // conv-input window rows beyond each end of a tile: the largest dilation
                                           // (dilation_cycle_length <= 4 on this path, dsx_load_diffnet)

// Shared memory of k_hp_step<NWG, R> from a 1024-aligned base (the dynamic allocation adds 1 KB for the alignment):
//   R ring slots of STAGE bytes | full[R], empty[R], window[4] mbarriers (1 KB, keeps what follows aligned) | ...
// WIN (R = 3; P <= 2: fp16, fp16x2, fp16s): GEMM1 reads its three taps from one conv-input window per tile, so the ring
// carries weight tiles only.  After the barriers:
//   W, NWG x 40 KB: in the layers the window, 4 channel blocks of WROWS = 64 NWG + 2 kHalo rows (frames t0 - kHalo ..
//     t0 + 64 NWG + kHalo of the tile), NWG x 8 + 2 KB each.  Once every warpgroup is done with GEMM1 chunk 1, its first
//     NWG x 16 KB take z hi k-blocks 2-3 (the window is reloaded only after GEMM2).  In the head, z hi k-blocks 2-3 and
//     then R activation slots of NWG x 8 KB for H1's A blocks; h's lo k-blocks 0..2 live in them (H2 and the input
//     projection carry weights only).
//   z hi k-blocks 0-1, NWG x 16 KB | LO: z lo k-block 3 (the layers never read z lo; the head does, HP = 3), NWG x 8 KB
// !WIN (R = 2, fp16x3, P = 3 inside the layers; and the conditioner projection): a ring slot also holds one 64 x 64
//   activation block per warpgroup, copied with the stage, and z is whole: hi plane NWG x 32 KB | LO plane NWG x 32 KB.
template <int NWG, int R, bool WIN = (R == 3)>
struct StepCfg {
  static_assert(R == 2 || R == 3, "ring depth");
  static constexpr int THREADS = NWG * 128;
  static constexpr int STAGE = kWBytes + (WIN ? 0 : NWG * kABytes);
  static constexpr int BARS = R * STAGE;
  static constexpr int W = BARS + 1024;
  static constexpr int WROWS = 64 * NWG + 2 * kHalo;
  static constexpr int WBLK = WROWS * 128;
  static constexpr int ZHI23 = 2 * kABytes;                       // z hi k-blocks 2-3 of one warpgroup, in W
  static constexpr int ASLOT = NWG * ZHI23;                       // the head's activation slots, in W
  static constexpr int WSIZE = WIN ? std::max(4 * WBLK, ASLOT + R * NWG * kABytes) : 0;
  static constexpr int ZHI = W + WSIZE;
  static constexpr int ZHI_WG = WIN ? 2 * kABytes : kZBytes;      // z hi bytes per warpgroup at ZHI
  static constexpr int ZLO = ZHI + NWG * ZHI_WG;
  static constexpr int SMEM = 1024 + ZLO + NWG * (R == 2 ? kZBytes : kABytes);
  static_assert(WBLK % 1024 == 0 && ASLOT % 1024 == 0, "window blocks and activation slots start 1024-aligned");
  static_assert(!WIN || NWG * ZHI23 <= WSIZE, "z hi k-blocks 2-3 fit in W");
  // NWG = 2: 1 + 3 x 32 + 1 + 80 (window 72) + 32 + 16 KB (R = 3) or 1 + 2 x 48 + 1 + 64 + 64 KB (R = 2) = 226 KB, of
  // 227 KB.  NWG = 1, R = 3: 1 + 96 + 1 + 40 + 16 + 8 = 162 KB.
  static_assert(SMEM <= 232448, "shared memory budget (227 KB per block on sm_90)");
};
// the conditioner projection: the ring (with activation blocks) and its barriers only
constexpr int kCondSmem = 1024 + StepCfg<2, 3, false>::BARS + 2 * 3 * 8;

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
  long long* trace;          // dsx_debug_trace buffer [trace_ctas][DSX_TRACE_SLOTS], or nullptr
  int trace_ctas;
  unsigned* flags;           // [2][units] per-tile progress in this launch, zeroed before it: layers done | layers whose
                             // GEMM1 and gates are done (paired tiles only)
};

// phase stamp of dsx_debug_trace (layout in dsx.h); one uniform branch when tracing is off
__device__ __forceinline__ void stamp(const HpParams& p, int slot) {
  if (p.trace != nullptr && threadIdx.x == 0 && slot < DSX_TRACE_SLOTS && static_cast<int>(blockIdx.x) < p.trace_ctas) {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)::"memory");
    p.trace[static_cast<size_t>(blockIdx.x) * DSX_TRACE_SLOTS + slot] = t;
  }
}
__device__ __forceinline__ int layer_slot(const HpParams& p, int l, int k) { return 1 + 9 * (l - p.l0) + k; }
__device__ __forceinline__ int head_slot(const HpParams& p, int k) { return 1 + 9 * (p.l1 - p.l0) + k; }

// ------------------------------------------------------------------------------------------
// ordering between tiles
// ------------------------------------------------------------------------------------------
// Layer l of a tile reads y of layer l - 1 from its own frames and at most kHalo frames into its neighbour tiles of the
// same utterance; x, skip, CP and S16 of a tile are read by that tile only, and windows zero-fill frames outside [0, T),
// so tiles of different utterances never read each other.  So instead of a grid-wide barrier between layers, every
// tile publishes p.flags[u] = layers done (after its residual epilogue wrote y) and a tile waits only for its
// neighbours.  Waiting for the neighbours to finish layer l - 1 also means they have read Y buffer (l + 1) & 1 for the
// last time before the tile overwrites it in layer l.
//
// Deadlock freedom: every CTA is resident (cooperative launch) and visits (layer, tile) in layer-major order, and a
// wait at layer l is only ever for layer l - 1 or, between paired tiles, for an earlier point of layer l.  The CTA that
// owns the awaited point is either past it or itself waiting at a strictly earlier point, and the earliest waiting
// point of all waits for nothing that is not already done.
//
// Pairing: when every tile has its own CTA, tile j of utterance 2k + 1 starts layer l only after tile j of utterance
// 2k has finished GEMM1 and the gates of layer l (p.flags[units + u]).  The two groups then run half a layer apart, so
// one group's L2-bound GEMMs overlap the other's HBM-bound epilogues.  This is scheduling only: the tiles share no data.
template <int NWG>
__device__ __forceinline__ int partner_tile(const HpParams& p, int u) {
  if (p.units > static_cast<int>(gridDim.x) || p.B < 2) return -1;
  const int tpu = p.Tp / (64 * NWG), b = u / tpu;
  if (b & 1) return u - tpu;
  return b + 1 < p.B ? u + tpu : -1;
}

// thread 0: spins until the neighbours of tile u in its utterance have published n layers
template <int NWG>
__device__ __forceinline__ void wait_neighbours(const HpParams& p, int u, unsigned n) {
  const int tpu = p.Tp / (64 * NWG);
  if (u % tpu != 0) wait_geq(p.flags + u - 1, n);
  if ((u + 1) % tpu != 0) wait_geq(p.flags + u + 1, n);
}

// Holds the CTA until tile u may start layer l.  Thread 0's acquire loads, followed by the __syncthreads, order the
// neighbours' y writes before every thread's later reads of them: the window and the streamed taps are non-bulk
// cp.async, which reads through the generic proxy.  (A bulk copy of the window would need a proxy fence after this.)
template <int NWG>
__device__ __forceinline__ void wait_layer(const HpParams& p, int l, int u) {
  if (threadIdx.x == 0) {
    const unsigned n = l - p.l0;
    if (n > 0) wait_neighbours<NWG>(p, u, n);
    const int pu = partner_tile<NWG>(p, u);
    if (pu >= 0 && pu < u) wait_geq(p.flags + p.units + pu, n + 1);
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------------
// operand loads and the GEMM loop
// ------------------------------------------------------------------------------------------
// 256 (NROWS) weight rows of an unswizzled tile -> swizzled tile; row r comes from src0 (r < 128) or src1 (r >= 128).
// Only the self-test uses it, to check the layout against a host product; the kernels bulk-copy pre-swizzled tiles.
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
// outside [0, T) read as zero.  Called by the 128 threads of one warpgroup.  (Unlike the window, a streamed tap is read
// again by the layer's other taps and chunk, so it carries no eviction hint.)
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
// One channel block of a conv-input window: rows r < rows hold frame t_first + r of one utterance (utt: its [Tp][256]
// frames), channels [ch0, ch0 + 64); frames outside [0, T) read as zero.  dst is 1024-aligned, so a wgmma descriptor
// started at any row reads 64 consecutive frames.  Called by the NT threads of the CTA.  The lines leave L2 first: a layer
// reads its conv input once per tile (the neighbour tiles' halo rows aside) and the layer after overwrites it.
template <int NT>
__device__ __forceinline__ void load_wblock(uint8_t* dst, const __half* utt, int t_first, int ch0, int rows, int T, int tid) {
  const uint32_t d = smem_u32(dst);
#pragma unroll 1
  for (int i = tid; i < rows * 8; i += NT) {
    const int r = i >> 3, c = i & 7, t = t_first + r;
    const bool valid = t >= 0 && t < T;
    cp16_hint(d + sw128(r, c), utt + static_cast<size_t>(valid ? t : 0) * kC + ch0 + c * 8, valid, l2_evict_first());
  }
}

template <int N>
__device__ __forceinline__ void fence_acc(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

struct NoPrefetch {
  __device__ __forceinline__ void operator()(int) const {}
};

__device__ __forceinline__ uint8_t* smem_base() {
  extern __shared__ uint8_t smem_raw[];
  return reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
}

// The shared memory of one CTA, laid out as StepCfg says (the conditioner projection has no z): the operand ring, its
// barriers, and this warpgroup's z operand.  Addresses are recomputed from the base where they are used, so only n and
// nw stay live: the stages consumed so far in the launch, and the conv-input windows.  Every thread runs the same GEMM
// phases, so both are the same in all of them; ring stage i uses slot i % R in barrier phase i / R, window j completes
// phase j of the window barriers.
template <int NWG, int R, bool WIN = (R == 3)>
struct Smem {
  using Cfg = StepCfg<NWG, R, WIN>;
  uint32_t n, nw;
  __device__ __forceinline__ uint8_t* slot(uint32_t i) const { return smem_base() + (i % R) * Cfg::STAGE; }
  __device__ __forceinline__ uint32_t full(uint32_t i) const { return smem_u32(smem_base() + Cfg::BARS) + (i % R) * 8; }
  __device__ __forceinline__ uint32_t empty(uint32_t i) const { return full(i) + R * 8; }
  __device__ __forceinline__ uint32_t parity(uint32_t i) const { return (i / R) & 1; }
  // channel block c of the conv-input window (WIN) and its barrier
  __device__ __forceinline__ uint8_t* wblk(int c) const { return smem_base() + Cfg::W + c * Cfg::WBLK; }
  __device__ __forceinline__ uint32_t wbar(int c) const { return full(0) + 2 * R * 8 + c * 8; }
  // warpgroup wg's activation block in slot j
  __device__ __forceinline__ uint8_t* ablk(int j, int wg) const {
    if (WIN) return smem_base() + Cfg::W + Cfg::ASLOT + j * NWG * kABytes + wg * kABytes;
    return smem_base() + j * Cfg::STAGE + kWBytes + wg * kABytes;
  }
  // k-block kb of z plane 0 (hi) or 1 (lo).  With WIN, hi k-blocks 2-3 share W with the window, and the lo plane may
  // only be used while no activation block is in flight in the ring (the head's H2 and input projection, StepCfg).
  __device__ __forceinline__ uint8_t* zblk(int plane, int kb) const {
    const int wg = threadIdx.x >> 7;
    if (plane == 0) {
      if (WIN && kb >= 2) return smem_base() + Cfg::W + wg * Cfg::ZHI23 + (kb - 2) * kABytes;
      return smem_base() + Cfg::ZHI + wg * Cfg::ZHI_WG + kb * kABytes;
    }
    if (!WIN) return smem_base() + Cfg::ZLO + wg * kZBytes + kb * kABytes;
    return kb < R ? ablk(kb, wg) : smem_base() + Cfg::ZLO + wg * kABytes;
  }
  // (row r, channel k) of z plane `plane`
  __device__ __forceinline__ uint8_t* zat(int plane, int r, int k) const {
    return zblk(plane, k >> 6) + sw128(r, (k & 63) >> 3) + (k & 7) * 2;
  }
  __device__ __forceinline__ void init() {
    n = 0;
    nw = 0;
    if (threadIdx.x == 0) {
      for (int j = 0; j < R; ++j) {
        mbar_init(full(j), 1 + NWG * 128);     // the bulk copy's arrive.expect_tx + one arrival per thread
        mbar_init(empty(j), NWG);              // one release per warpgroup
      }
      if (WIN)
        for (int c = 0; c < 4; ++c) mbar_init(wbar(c), NWG * 128);   // every thread's cp.async arrival
      fence_mbar_init();
    }
    __syncthreads();
  }
};

// A GEMM phase of one tile; the stages of a phase are its k-blocks times MMA passes
enum PhaseKind { PH_NONE, PH_G1, PH_G2, PH_H1, PH_H2, PH_IN, PH_COND };
struct Phase {
  int kind, l, u, hq;   // layer, tile, GEMM1 chunk / GEMM2 half / conditioner-projection chunk
};
// the first GEMM phase of the head of tile u (none past the last tile)
__device__ __forceinline__ Phase head_phase(const HpParams& p, int u) {
  const int kind = u >= p.units ? PH_NONE : (p.head_flags & TC_HEAD) ? PH_H1 : (p.head_flags & TC_INPROJ) ? PH_IN : PH_NONE;
  return Phase{kind, 0, u, 0};
}
// what this CTA runs after layer l: the next layer or the head, from its first tile
__device__ __forceinline__ Phase after_layer(const HpParams& p, int l) {
  const int u0 = blockIdx.x;
  if (l + 1 < p.l1) return Phase{PH_G1, l + 1, u0, 0};
  return p.head_flags ? head_phase(p, u0) : Phase{PH_NONE, 0, 0, 0};
}

// The operands of one stage for this thread's warpgroup
struct StageSrc {
  const __half* w0;   // packed weight tile, or its rows 0..127 when w1 is set
  const __half* w1;   // rows 128..255 from a second 128-row tile, or nullptr
  uint32_t wbytes;    // bytes of each weight copy
  const __half* a;    // plane whose 64 x 64 block is copied into the slot; nullptr: the A operand is z or the window
  int b, at, ach;     // that block: utterance, first frame (may lie outside [0, T)), first channel
  int wrow;           // >= 0: the A operand is window block ach / 64 from this row on (GEMM1 with WIN)
  int zplane, zkb;    // otherwise the plane and k-block of z
};

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

__device__ __forceinline__ int phase_passes(const HpParams& p, int kind) {
  return kind == PH_COND ? 3 : (kind >= PH_H1 ? p.HP : p.P);
}
__device__ __forceinline__ int phase_stages(const HpParams& p, const Phase& ph) {
  // k-blocks: GEMM1 3 taps x 256 channels, input projection 128 mel bins, the others 256 channels
  const int kbs = ph.kind == PH_G1 ? 12 : ph.kind == PH_IN ? 2 : ph.kind == PH_NONE ? 0 : 4;
  return kbs * phase_passes(p, ph.kind);
}

template <int NWG, bool WIN>
__device__ __forceinline__ StageSrc stage_src(const HpParams& p, const Phase& ph, int s) {
  const int frame0 = ph.u * 64 * NWG;
  const int P = phase_passes(p, ph.kind);
  const int kb = s / P, ps = s % P, wp = pass_wplane(ps), ap = pass_aplane(ps);
  StageSrc st;
  st.w1 = nullptr;
  st.wbytes = kWBytes;
  st.a = nullptr;
  st.b = frame0 / p.Tp;
  st.at = frame0 % p.Tp + (threadIdx.x >> 7) * 64;
  st.ach = kb * 64;
  st.wrow = -1;
  st.zplane = ap;
  st.zkb = kb;
  switch (ph.kind) {
    case PH_G1: {  // [y(t-d) | y(t) | y(t+d)]: k-block kb = tap * 4 + channel block
      const int shift = ((kb >> 2) - 1) * (1 << (ph.l % p.cycle));
      st.w0 = w1_tile(p, ph.l, wp, ph.hq, kb);
      st.ach = (kb & 3) * 64;
      if (WIN) {   // P <= 2: every pass reads y's hi plane, resident in the window
        st.wrow = kHalo + (threadIdx.x >> 7) * 64 + shift;
      } else {
        st.a = p.Y + static_cast<size_t>(ph.l & 1) * 2 * p.plane + ap * p.plane;
        st.at += shift;
      }
      break;
    }
    case PH_G2:
      st.w0 = w2_tile(p, ph.l, wp, ph.hq, kb);
      break;
    case PH_H1:
      st.w0 = whead_tile(p, wp * 8 + kb);
      st.w1 = whead_tile(p, wp * 8 + 4 + kb);
      st.wbytes = kWBytes / 2;
      st.a = p.S16 + ap * p.plane;
      break;
    case PH_H2:   // N = 128: one 128-row tile
      st.w0 = whead_tile(p, 16 + wp * 4 + kb);
      st.wbytes = kWBytes / 2;
      break;
    case PH_IN:
      st.w0 = whead_tile(p, 24 + wp * 4 + kb);
      st.w1 = whead_tile(p, 24 + wp * 4 + 2 + kb);
      st.wbytes = kWBytes / 2;
      break;
    default:      // PH_COND: the conditioner k-blocks 12..15 of W1 chunk hq
      st.w0 = p.w + (static_cast<size_t>(ph.l) * kRowsPerLayer + ((wp * 2 + ph.hq) * 16 + 12 + kb) * 256) * 64;
      st.a = p.CONDH + ap * p.plane;
      break;
  }
  return st;
}

enum { kIssueW = 1, kIssueA = 2 };
// Issues the parts of ring stage i: the weight tile (thread 0, once the slot's previous stage is released by every
// warpgroup) and this warpgroup's activation block (every thread; its own MMAs of the slot's previous stage are done).
// Every thread arrives on the full barrier with its A part, block or not, so the stage completes only when both parts
// have landed.  With WIN a thread without a block arrives at once, so the stage does not wait for the window it may
// have in flight.
template <int NWG, int R, bool WIN>
__device__ __forceinline__ void issue(const HpParams& p, const Smem<NWG, R, WIN>& sm, const StageSrc& st, uint32_t i,
                                      int parts) {
  const uint32_t full = sm.full(i);
  uint8_t* slot = sm.slot(i);
  if ((parts & kIssueW) && threadIdx.x == 0) {
    mbar_wait(sm.empty(i), sm.parity(i) ^ 1);
    mbar_arrive_expect_tx(full, st.w1 ? 2 * st.wbytes : st.wbytes);
    bulk_g2s(smem_u32(slot), st.w0, st.wbytes, full);
    if (st.w1) bulk_g2s(smem_u32(slot) + st.wbytes, st.w1, st.wbytes, full);
  }
  if (parts & kIssueA) {
    if (st.a) load_a(sm.ablk(i % R, threadIdx.x >> 7), st.a, st.b, st.at, st.ach, p.T, p.Tp, threadIdx.x & 127);
    if (WIN && !st.a) mbar_arrive(full);
    else cp_arrive_noinc(full);
  }
}

// The conv input of both GEMM1 chunks of tile u in layer l, into the window (StepCfg), copied by every thread of the
// CTA.  Each channel block completes on its own barrier, so the first MMAs wait for block 0 only.
template <int NWG, int R, bool WIN>
__device__ __forceinline__ void load_window(const HpParams& p, const Smem<NWG, R, WIN>& sm, int l, int u) {
  const int frame0 = u * 64 * NWG;
  const __half* utt = p.Y + static_cast<size_t>(l & 1) * 2 * p.plane + static_cast<size_t>(frame0 / p.Tp) * p.Tp * kC;
#pragma unroll 1
  for (int c = 0; c < 4; ++c) {
    load_wblock<NWG * 128>(sm.wblk(c), utt, frame0 % p.Tp - kHalo, c * 64, StepCfg<NWG, R, WIN>::WROWS, p.T, threadIdx.x);
    cp_arrive_noinc(sm.wbar(c));
  }
}

// Issues parts of the first R stages of phase ph, the next one the ring will run (all its slots are released).  With
// WIN, the A part of GEMM1 chunk 0 is the tile's window; the caller makes sure no warpgroup still reads z from W.
template <int NWG, int R, bool WIN>
__device__ __forceinline__ void fill(const HpParams& p, const Smem<NWG, R, WIN>& sm, const Phase& ph, int parts) {
  if (WIN && ph.kind == PH_G1 && ph.hq == 0 && (parts & kIssueA)) load_window(p, sm, ph.l, ph.u);
  const int n = min(R, phase_stages(p, ph));
#pragma unroll 1
  for (int j = 0; j < n; ++j) issue(p, sm, stage_src<NWG, WIN>(p, ph, j), sm.n + j, parts);
}

// c0 (weight rows 0..127) [and c1 (rows 128..255) when NH == 2] = sum over the stages s of phase ph of A_s . W_s^T.  The
// first R stages were issued by fill(); stage s + R - 1 is issued once the MMAs of stage s - 1 are done, which keeps one
// wgmma group in flight behind the copies.  pre(s) runs after that (L2 prefetches of what the epilogues read, paced so
// that they queue behind the operand copies).  Every thread of the CTA runs it; it ends with the accumulators complete
// and every slot released by this warpgroup.
template <int NH, int NWG, int R, bool WIN, class Pre = NoPrefetch>
__device__ __forceinline__ void gemm(float (&c0)[64], float (&c1)[64], Smem<NWG, R, WIN>& sm, const HpParams& p,
                                     const Phase& ph, Pre pre = Pre()) {
  const int nst = phase_stages(p, ph);
  const int wg = threadIdx.x >> 7;
  // the epilogue before this phase wrote z with st.shared: visible to the warpgroup's wgmmas from here
  fence_proxy_async_smem();
  wg_bar_sync();
  fence_acc(c0);
  if (NH == 2) fence_acc(c1);
#pragma unroll 1
  for (int s = 0; s < nst; ++s) {
    const uint32_t i = sm.n + s;
    const StageSrc st = stage_src<NWG, WIN>(p, ph, s);
    mbar_wait(sm.full(i), sm.parity(i));
    if (WIN && st.wrow >= 0) mbar_wait(sm.wbar(st.ach >> 6), sm.nw & 1);
    fence_proxy_async_smem();   // the cp.async writes of the activation block or window -> the async proxy of wgmma
    uint8_t* slot = sm.slot(i);
    // (without WIN, ablk is slot + kWBytes + wg * kABytes; spelled out from slot, the R = 2 form spills less)
    const uint8_t* aop = WIN && st.wrow >= 0 ? sm.wblk(st.ach >> 6) + st.wrow * 128
                         : st.a ? (WIN ? sm.ablk(i % R, wg) : slot + kWBytes + wg * kABytes)
                                : sm.zblk(st.zplane, st.zkb);
    const uint64_t a = wg_desc(smem_u32(aop));
    const uint64_t w = wg_desc(smem_u32(slot));
    wg_fence();
#pragma unroll
    for (int k4 = 0; k4 < 4; ++k4) {
      const int acc = (s > 0 || k4 > 0) ? 1 : 0;
      wgmma_n128(c0, a + 2 * k4, w + 2 * k4, acc);
      if (NH == 2) wgmma_n128(c1, a + 2 * k4, w + (16384 >> 4) + 2 * k4, acc);
    }
    wg_commit();
    if (s > 0) {
      wg_wait1();
      if ((threadIdx.x & 127) == 0) mbar_arrive(sm.empty(i - 1));
      if (s - 1 + R < nst) issue(p, sm, stage_src<NWG, WIN>(p, ph, s - 1 + R), i - 1 + R, kIssueW | kIssueA);
    }
    pre(s);
  }
  wg_wait0();
  fence_acc(c0);
  if (NH == 2) fence_acc(c1);
  if ((threadIdx.x & 127) == 0) mbar_arrive(sm.empty(sm.n + nst - 1));
  sm.n += nst;
}

// ------------------------------------------------------------------------------------------
// one residual layer of one tile
// ------------------------------------------------------------------------------------------
template <int NWG, int R, bool WIN>
__device__ __forceinline__ void layer_tile(const HpParams& p, int l, int u, Smem<NWG, R, WIN>& sm) {
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  const int frame0 = u * 64 * NWG;
  const int b = frame0 / p.Tp, t0 = frame0 % p.Tp + wg * 64;
  const size_t fbase = static_cast<size_t>(b) * p.Tp + t0;     // global frame of row 0 of this warpgroup
  const int P = p.P;
  const size_t NF = p.plane / kC;
  float c0[64], c1[64];

  // ---- GEMM1 + gate, chunk by chunk ----
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    // L2 prefetch of this warpgroup's CP rows (64 x 2 KB, both chunks) during chunk 0, 16 KB per stage.  They are
    // marked evict_last so that the weight stream and the other group's epilogue traffic do not push chunk 1's rows out
    // before its gate epilogue reads them; that read (ld_stream_f2, evict_first) releases them.  x and skip are not
    // prefetched: with the CP rows held, a chunk-1 prefetch of them cost more than it saved (DESIGN.md).
    auto pre = [&](int s) {
      if (wtid != 0 || s >= 8 || h != 0) return;
      prefetch_l2_hint(p.CP + (static_cast<size_t>(l) * NF + fbase) * 512 + s * 4096, 16384, l2_evict_last());
    };
    gemm<2>(c0, c1, sm, p, Phase{PH_G1, l, u, h}, pre);
    // chunk 1's weights and taps do not depend on this epilogue; GEMM2's weights do not depend on either
    fill(p, sm, h == 0 ? Phase{PH_G1, l, u, 1} : Phase{PH_G2, l, u, 0}, kIssueW | kIssueA);
    if (WIN && h == 1) {
      // the window is spent; z hi k-blocks 2-3, which this epilogue writes, overlap it, and the other warpgroup's
      // rows of it may still be read
      sm.nw++;
      __syncthreads();
    }
    stamp(p, layer_slot(p, l, 2 * h));
    const float* cp = p.CP + (static_cast<size_t>(l) * NF + fbase) * 512 + h * 256;
    // the loads of kEpiBatch accumulator pairs are issued together, ahead of the stores that use them
#pragma unroll
    for (int e0 = 0; e0 < 64; e0 += 2 * kEpiBatch) {
      float2 cgv[kEpiBatch], cfv[kEpiBatch];
#pragma unroll
      for (int j = 0; j < kEpiBatch; ++j) {
        const int e = e0 + 2 * j, r = acc_row(wtid, e), n = acc_col(wtid, e);
        cgv[j] = ld_stream_f2(cp + static_cast<size_t>(r) * 512 + n);
        cfv[j] = ld_stream_f2(cp + static_cast<size_t>(r) * 512 + 128 + n);
      }
#pragma unroll
      for (int j = 0; j < kEpiBatch; ++j) {
        const int e = e0 + 2 * j, r = acc_row(wtid, e), n = acc_col(wtid, e);
        float z0, z1;
        if (p.fast_gate) {
          z0 = gate_fast(c0[e] + cgv[j].x, c1[e] + cfv[j].x);
          z1 = gate_fast(c0[e + 1] + cgv[j].y, c1[e + 1] + cfv[j].y);
        } else {
          z0 = gate_acc(c0[e] + cgv[j].x, c1[e] + cfv[j].x);
          z1 = gate_acc(c0[e + 1] + cgv[j].y, c1[e + 1] + cfv[j].y);
        }
        const __half2 hh = __floats2half2_rn(z0, z1);
        *reinterpret_cast<__half2*>(sm.zat(0, r, 128 * h + n)) = hh;
        if (R == 2 && P == 3) {
          const float2 hf = __half22float2(hh);
          *reinterpret_cast<__half2*>(sm.zat(1, r, 128 * h + n)) = __floats2half2_rn(z0 - hf.x, z1 - hf.y);
        }
      }
    }
    stamp(p, layer_slot(p, l, 2 * h + 1));
    // an even-utterance tile lets its partner start layer l (wait_layer)
    if (h == 1 && tid == 0 && partner_tile<NWG>(p, u) > u) st_release_gpu(p.flags + p.units + u, l - p.l0 + 1);
  }

  // ---- GEMM2 + residual / skip epilogues ----
  const bool last = (l + 1 == p.L);
  const float* dnext = last ? nullptr : p.dtab + static_cast<size_t>(b) * p.d_row_stride + static_cast<size_t>(l + 1) * kC;
  __half* Yout = p.Y + static_cast<size_t>((l + 1) & 1) * 2 * p.plane;
#pragma unroll 1
  for (int q = 0; q < 2; ++q) {
    gemm<2>(c0, c1, sm, p, Phase{PH_G2, l, u, q});
    if (q == 0) fill(p, sm, Phase{PH_G2, l, u, 1}, kIssueW | kIssueA);
    else if (u + static_cast<int>(gridDim.x) < p.units) {
      const Phase next{PH_G1, l, u + static_cast<int>(gridDim.x), 0};
      fill(p, sm, next, kIssueW);
      // the wait ends in a __syncthreads, which also keeps the next tile's window off the z k-blocks the other
      // warpgroup may still read
      wait_layer<NWG>(p, l, next.u);
      fill(p, sm, next, kIssueA);
    } else {
      fill(p, sm, after_layer(p, l), kIssueW);   // its activation blocks or window are issued after the next wait
    }
    stamp(p, layer_slot(p, l, 4 + 2 * q));
    // This thread's accumulators cover rows row0 and row0 + 8 and columns colb + 8 i + {0, 1} of each 128-column half
    // (acc_row / acc_col), so every address below is a per-thread base plus a compile-time offset; with the offsets
    // folded the unrolled loops hold no 64-bit address per element.
    const int row0 = acc_row(wtid, 0), colb = acc_col(wtid, 0);
    const bool ok0 = t0 + row0 < p.T, ok8 = t0 + row0 + 8 < p.T;
    const size_t tb = (fbase + row0) * kC + colb;
    const float* bias = p.b2 + static_cast<size_t>(l) * 512 + q * 256 + colb;
    const float* dn = last ? nullptr : dnext + colb;
    const float* src = (q == 0 ? p.X : p.SKIP) + tb;
    float* dst = (q == 0 ? p.X : p.SKIP) + tb;
    __half* yo = Yout + tb;
    __half* so = p.S16 + tb;
    const bool read_old = q == 0 || l > 0;
    const bool read_d = q == 0 && !last;
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
      for (int e0 = 0; e0 < 64; e0 += 2 * kEpiBatch) {
        // the batch's x or skip pairs, and the bias and FiLM pairs of its kEpiBatch / 2 columns (shared by rows row0 and
        // row0 + 8), all ahead of the stores: loaded in the element loop, each bias or FiLM pair would be a round trip
        // that the element's stores wait for
        float2 old[kEpiBatch], bbv[kEpiBatch / 2], dvv[kEpiBatch / 2];
#pragma unroll
        for (int j = 0; j < kEpiBatch; ++j) {
          const int e = e0 + 2 * j, o = ((e & 2) ? 8 * kC : 0) + hh * 128 + (e >> 2) * 8;
          old[j] = make_float2(0.f, 0.f);
          if (read_old && ((e & 2) ? ok8 : ok0)) old[j] = *reinterpret_cast<const float2*>(src + o);
        }
#pragma unroll
        for (int i = 0; i < kEpiBatch / 2; ++i) {
          const int c = hh * 128 + ((e0 >> 2) + i) * 8;
          bbv[i] = __ldg(reinterpret_cast<const float2*>(bias + c));
          dvv[i] = make_float2(0.f, 0.f);
          if (read_d) dvv[i] = __ldg(reinterpret_cast<const float2*>(dn + c));
        }
#pragma unroll
        for (int j = 0; j < kEpiBatch; ++j) {
          const int e = e0 + 2 * j, c = hh * 128 + (e >> 2) * 8, o = ((e & 2) ? 8 * kC : 0) + c;
          if (!((e & 2) ? ok8 : ok0)) continue;
          const float a0 = hh ? c1[e] : c0[e], a1 = hh ? c1[e + 1] : c0[e + 1];
          const float2 bb = bbv[j >> 1];
          if (q == 0) {
            float2 xv = old[j];
            xv.x = (xv.x + (a0 + bb.x)) * 0.70710678118654752440f;
            xv.y = (xv.y + (a1 + bb.y)) * 0.70710678118654752440f;
            *reinterpret_cast<float2*>(dst + o) = xv;
            if (!last) {
              const float2 dv = dvv[j >> 1];
              const float ya = xv.x + dv.x, yb = xv.y + dv.y;
              const __half2 hy = __floats2half2_rn(ya, yb);
              *reinterpret_cast<__half2*>(yo + o) = hy;
              if (p.ylo) {
                const float2 hf = __half22float2(hy);
                *reinterpret_cast<__half2*>(yo + p.plane + o) = __floats2half2_rn(ya - hf.x, yb - hf.y);
              }
            }
          } else {
            float2 sk = make_float2(a0 + bb.x, a1 + bb.y);
            if (l > 0) {
              sk.x = old[j].x + sk.x;
              sk.y = old[j].y + sk.y;
            }
            *reinterpret_cast<float2*>(dst + o) = sk;
            if (last) {
              const float sa = sk.x * p.inv_sqrt_l, sb = sk.y * p.inv_sqrt_l;
              const __half2 hs = __floats2half2_rn(sa, sb);
              const float2 hf = __half22float2(hs);
              *reinterpret_cast<__half2*>(so + o) = hs;
              *reinterpret_cast<__half2*>(so + p.plane + o) = __floats2half2_rn(sa - hf.x, sb - hf.y);
            }
          }
        }
      }
    }
    stamp(p, layer_slot(p, l, 5 + 2 * q));
    if (q == 0) {
      // y of layer l is written: publish it to the neighbours
      __syncthreads();
      if (tid == 0) st_release_gpu(p.flags + u, l - p.l0 + 1);
    }
  }
}

// ------------------------------------------------------------------------------------------
// head of one tile: eps = W_out . relu(W_s . s16 + b_s) + b_out, sampler update, next input projection
// ------------------------------------------------------------------------------------------
template <int NWG, int R>
__device__ __forceinline__ void head_tile(const HpParams& p, int u, Smem<NWG, R>& sm) {
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  const int frame0 = u * 64 * NWG;
  const int b = frame0 / p.Tp, t0 = frame0 % p.Tp + wg * 64;
  const size_t fbase = static_cast<size_t>(b) * p.Tp + t0;
  const int flags = p.head_flags;
  const bool do_head = flags & TC_HEAD, do_in = flags & TC_INPROJ;
  float c0[64], c1[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) c0[i] = 0.f;

  if (do_head) {
    // H1: h = relu(s16 . W_s^T + b_s) -> fp16 hi / lo operand.  H2 carries weights only, so h's lo plane may take the
    // activation slots (StepCfg).
    gemm<2>(c0, c1, sm, p, Phase{PH_H1, 0, u, 0});
    fill(p, sm, Phase{PH_H2, 0, u, 0}, kIssueW | kIssueA);
    stamp(p, head_slot(p, 0));
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
      for (int e = 0; e < 64; e += 2) {
        const int r = acc_row(wtid, e), col = hh * 128 + acc_col(wtid, e);
        const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bs + col));
        const float a0 = fmaxf((hh ? c1[e] : c0[e]) + bb.x, 0.f), a1 = fmaxf((hh ? c1[e + 1] : c0[e + 1]) + bb.y, 0.f);
        const __half2 hv = __floats2half2_rn(a0, a1);
        *reinterpret_cast<__half2*>(sm.zat(0, r, col)) = hv;
        const float2 hf = __half22float2(hv);
        *reinterpret_cast<__half2*>(sm.zat(1, r, col)) = __floats2half2_rn(a0 - hf.x, a1 - hf.y);
      }
    }
    stamp(p, head_slot(p, 1));
    // H2: eps (before bias) = h . W_out^T, N = 128 (rows >= M of the packed tile are zero)
    gemm<1>(c0, c1, sm, p, Phase{PH_H2, 0, u, 0});
    fill(p, sm, do_in ? Phase{PH_IN, 0, u, 0} : head_phase(p, u + gridDim.x), kIssueW | kIssueA);
    stamp(p, head_slot(p, 2));
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
      *reinterpret_cast<__half2*>(sm.zat(0, r, m)) = hv;
      const float2 hf = __half22float2(hv);
      *reinterpret_cast<__half2*>(sm.zat(1, r, m)) = __floats2half2_rn(xv[0] - hf.x, xv[1] - hf.y);
    }
  }
  stamp(p, head_slot(p, 3));
  if (!do_in) return;

  // ---- input projection: x0 = relu(x_in . W_in^T + b_in) -> X ; y0 = split(x0 + d_0) -> Y buffer 0 ----
  gemm<2>(c0, c1, sm, p, Phase{PH_IN, 0, u, 0});
  fill(p, sm, head_phase(p, u + gridDim.x), kIssueW | kIssueA);
  stamp(p, head_slot(p, 4));
  if (p.l1 > p.l0) {
    // Y buffer 0, written below, is the conv input of layer L - 1 when L is odd: the neighbours must be done with it
    if (tid == 0) wait_neighbours<NWG>(p, u, p.l1 - p.l0);
    __syncthreads();
  }
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
  stamp(p, head_slot(p, 5));
}

template <int NWG, int R>
__global__ void __launch_bounds__(NWG * 128, 1) k_hp_step(const __grid_constant__ HpParams p) {
  Smem<NWG, R> sm;
  sm.init();
  stamp(p, 0);
  const int u0 = blockIdx.x;
  fill(p, sm, p.l0 < p.l1 ? Phase{PH_G1, p.l0, u0, 0} : head_phase(p, u0), kIssueW);
  for (int l = p.l0; l < p.l1; ++l) {
    // every thread gets here with its ring copies issued and none of its barrier waits pending
    wait_layer<NWG>(p, l, u0);
    if (l > p.l0) stamp(p, layer_slot(p, l - 1, 8));
    fill(p, sm, Phase{PH_G1, l, u0, 0}, kIssueA);
    for (int u = u0; u < p.units; u += gridDim.x) layer_tile<NWG, R>(p, l, u, sm);
  }
  if (p.head_flags) {
    // the head reads the tile's own S16 rows, written by other threads of the CTA
    __syncthreads();
    if (p.l0 < p.l1) stamp(p, layer_slot(p, p.l1 - 1, 8));
    fill(p, sm, head_phase(p, u0), kIssueA);
    for (int u = u0; u < p.units; u += gridDim.x) head_tile<NWG, R>(p, u, sm);
  }
}

// CP[l][frame][h * 256 + n] = cond . W1cond^T (hi / lo operands, 3 passes) + dilated_conv.bias + conditioner_projection.bias,
// for job (tile of 128 frames, layer) = (blockIdx.x, blockIdx.y)
__global__ void __launch_bounds__(256, 1) k_hp_condproj(const __grid_constant__ HpParams p) {
  Smem<2, 3, false> sm;   // the ring only, activation blocks included: no z operand, no window
  sm.init();
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  const int u = blockIdx.x, l = blockIdx.y;
  const int frame0 = u * 128;
  const int b = frame0 / p.Tp, t0 = frame0 % p.Tp + wg * 64;
  const size_t fbase = static_cast<size_t>(b) * p.Tp + t0;
  const size_t NF = p.plane / kC;
  float c0[64], c1[64];
  fill(p, sm, Phase{PH_COND, l, u, 0}, kIssueW | kIssueA);
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    gemm<2>(c0, c1, sm, p, Phase{PH_COND, l, u, h});
    if (h == 0) fill(p, sm, Phase{PH_COND, l, u, 1}, kIssueW | kIssueA);
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
// weight packing (tiles of 64 fp16 per row, in the order the K loops consume them).  Each row is stored in the
// 128-byte-swizzled order of its shared-memory slot (sw128_elem), so one bulk copy moves a tile.
// ------------------------------------------------------------------------------------------
// whead tile order (128 rows x 64 k each): skip_projection [plane][row half][kb 0..3] (16 tiles),
// output_projection [plane][kb 0..3] with rows >= M zero (8 tiles), input_projection [plane][row half][kb 0..1]
// with k >= M zero (8 tiles).
__global__ void k_pack_whead(const float* __restrict__ skip_w, const float* __restrict__ fin_w,
                             const float* __restrict__ in_w, __half* __restrict__ whead, int M) {
  const int tileidx = blockIdx.x, n = threadIdx.x;   // 128 threads = rows
  int plane;
  __half* dst = whead + static_cast<size_t>(tileidx) * 128 * 64;
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
    dst[sw128_elem(n, kk)] = plane == 0 ? hi : __float2half_rn(v - __half2float(hi));
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
  __half* dst = wpack + (static_cast<size_t>(l) * kRowsPerLayer + static_cast<size_t>(tileidx) * 256) * 64;
  for (int kk = 0; kk < 64; ++kk) {
    const float v = src[kk];
    const __half hi = __float2half_rn(v);
    dst[sw128_elem(n, kk)] = plane == 0 ? hi : __float2half_rn(v - __half2float(hi));
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
  __half* dst = wsr + ((static_cast<size_t>(set) * L + l) * 32 + tileidx) * 256 * 64;
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
      dst[sw128_elem(n, k4 * 4 + e)] = (uu < pr) ? ho : hn;
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
  DSX_TRY(h->mem.alloc(&wpack, rows * 64 * sizeof(__half)));
  DSX_TRY(h->mem.alloc(&b1p, static_cast<size_t>(h->m.L) * 512 * sizeof(float)));
  k_pack_wtc<<<dim3(kRowsPerLayer / 256, h->m.L), 256, 0, s>>>(h->m.w1f, h->m.w2f, h->m.b1f, wpack, b1p);
  DSX_TRY(counted_launch(h, "k_pack_wtc"));
  h->m.wpack = wpack;
  h->m.b1p = b1p;
  __half* whead;
  DSX_TRY(h->mem.alloc(&whead, static_cast<size_t>(32) * 128 * 64 * sizeof(__half)));
  k_pack_whead<<<32, 128, 0, s>>>(h->m.skip_w, h->m.fin_w, h->m.in_w, whead, h->m.M);
  DSX_TRY(counted_launch(h, "k_pack_whead"));
  h->m.whead = whead;
  h->m.wsr = nullptr;
  h->m.wsr_sets = 0;
  if (h->precision == DSX_PREC_FP16S) {
    const int R = std::max(1, h->sr_sets);
    __half* wsr;
    const size_t srows = static_cast<size_t>(R) * h->m.L * kSrRowsPerLayer;
    DSX_TRY(h->mem.alloc(&wsr, srows * 64 * sizeof(__half)));
    k_pack_wsr<<<dim3(32, h->m.L, R), 256, 0, s>>>(h->m.w1f, h->m.w2f, wsr, h->m.L, h->sr_seed);
    DSX_TRY(counted_launch(h, "k_pack_wsr"));
    h->m.wsr = wsr;
    h->m.wsr_sets = R;
  }
  return DSX_OK;
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// co-resident CTAs of k_hp_step<NWG, R> on this device (cached per handle)
template <int NWG, int R>
static int step_capacity(dsx_handle* h) {
  int& cache = h->step_occ[NWG == 1 ? 0 : R == 3 ? 1 : 2];
  if (cache == 0) {
    using Cfg = StepCfg<NWG, R>;
    cudaFuncSetAttribute(k_hp_step<NWG, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM);
    int n = 0;
    cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, k_hp_step<NWG, R>, Cfg::THREADS, Cfg::SMEM);
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
  prm.trace = h->trace_on ? reinterpret_cast<long long*>(h->trace_dev) : nullptr;
  prm.trace_ctas = 2 * h->sm_count;
  prm.flags = h->ws.FLAGS;
  return prm;
}

static void set_head(dsx_handle* h, HpParams& prm, const HeadArgs& a) {
  prm.head_flags = a.flags;
  prm.x = a.x;
  prm.xs = a.xs;
  prm.eps = a.eps;
  prm.noise = a.noise;
  prm.seed = a.seed;
  prm.offset = a.offset;
  prm.b_off = h->batch_offset;
  prm.c = a.c;
  if (a.plms) prm.pl = *a.plms;
  prm.d0 = h->ws.DTAB + static_cast<size_t>(a.next_row0) * h->m.L * kC;
  prm.d0_row_stride = a.row_per_b * h->m.L * kC;
}

template <int NWG, int R>
static int launch_step(dsx_handle* h, const HpParams& prm, cudaStream_t s) {
  const int cap = step_capacity<NWG, R>(h);
  DSX_CHECK(cap > 0, DSX_E_CUDA, "k_hp_step<%d, %d> cannot be resident on this device", NWG, R);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(std::min(prm.units, cap)));
  cfg.blockDim = dim3(StepCfg<NWG, R>::THREADS);
  cfg.dynamicSmemBytes = StepCfg<NWG, R>::SMEM;
  cfg.stream = s;
  // The progress flags count from zero in every launch that runs layers.  A memset on the stream, rather than an epoch
  // kept by the host, stays right under graph replay and when the batch geometry changes between calls.
  if (prm.l1 > prm.l0) DSX_CUDA(cudaMemsetAsync(prm.flags, 0, 2 * static_cast<size_t>(prm.units) * sizeof(unsigned), s));
  // cooperative: tiles spin-wait on the progress flags of other CTAs (wait_layer), so every CTA must be resident
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  DSX_CUDA(cudaLaunchKernelEx(&cfg, k_hp_step<NWG, R>, prm));
  return counted_launch(h, "k_hp_step");
}

// Layers that read z's lo plane (P = 3) keep it out of the ring and run a two-stage ring; every other launch runs three.
static int launch_step(dsx_handle* h, const HpParams& prm, int rows, cudaStream_t s) {
  if (prm.P == 3) {
    DSX_CHECK(rows == 128, DSX_E_INVALID, "three-pass layers run in 128-frame tiles");
    return launch_step<2, 2>(h, prm, s);
  }
  return rows == 64 ? launch_step<1, 3>(h, prm, s) : launch_step<2, 3>(h, prm, s);
}

static int gate_mode(const dsx_handle* h, int P) { return h->gate_approx >= 0 ? h->gate_approx : (P == 3 ? 0 : 1); }

// CP for the conditioner currently packed in ws.CONDH (called once per API call, after launch_pack_cond).
int launch_tc_condproj(dsx_handle* h, const Geom& g, cudaStream_t s) {
  if (!h->attr_cond) {
    DSX_CUDA(cudaFuncSetAttribute(k_hp_condproj, cudaFuncAttributeMaxDynamicSharedMemorySize, kCondSmem));
    h->attr_cond = true;
  }
  HpParams prm = base_params(h, g, 128);
  prm.w = h->m.wpack;
  k_hp_condproj<<<dim3(static_cast<unsigned>(prm.units), static_cast<unsigned>(h->m.L)), 256, kCondSmem, s>>>(prm);
  return counted_launch(h, "k_hp_condproj");
}

// Frames per CTA for this call: 64 (one warpgroup per CTA, twice the CTAs) whenever the whole batch then has a CTA per
// tile at once, i.e. for small batches that would otherwise leave most SMs idle; 128 otherwise.
static int stack_rows(dsx_handle* h, const Geom& g) {
  if (h->stack_rows == 64 || h->stack_rows == 128) return h->stack_rows;      // DSX_OPT_STACK_ROWS
  const int cap64 = step_capacity<1, 3>(h);
  return (cap64 > 0 && g.frames_padded() / 64 <= static_cast<size_t>(cap64)) ? 64 : 128;
}

// The stack form: every layer of an evaluation in one launch at stack_rows, one weight plane per MMA pass (fp16s: the
// stochastically rounded set of the table row).  It takes FP16 / FP16X2 / FP16S under DSX_OPT_STACK_KERNEL and
// DSX_OPT_STACK_MODE; every other layer launch uses the hi / lo planes at 128 rows.
static bool stack_form(const dsx_handle* h) {
  return h->stack_kernel && h->stack_mode &&
         (h->precision == DSX_PREC_FP16 || h->precision == DSX_PREC_FP16X2 || h->precision == DSX_PREC_FP16S);
}

bool tc_fuse_head(const dsx_handle* h) { return stack_form(h) && h->fused_head && h->profile != 2; }

int launch_tc_step(dsx_handle* h, const Geom& g, int l0, int l1, int row0, int row_per_b, const HeadArgs* head,
                   cudaStream_t s) {
  const ModelDev& m = h->m;
  const bool layers = l1 > l0, stack = layers && stack_form(h);
  if (!layers && !head) return DSX_OK;
  DSX_CHECK(!layers || !head || (stack && l0 == 0 && l1 == m.L), DSX_E_INVALID,
            "the head shares a launch only with all layers in the stack form");
  const int rows = stack ? stack_rows(h, g) : 128;
  HpParams prm = base_params(h, g, rows);
  if (head) set_head(h, prm, *head);
  if (!layers) return launch_step(h, prm, rows, s);
  if (stack) {
    const bool sr = (h->precision == DSX_PREC_FP16S);
    prm.w_sr = sr ? 1 : 0;
    prm.w = sr ? m.wsr + static_cast<size_t>(row0 % std::max(1, m.wsr_sets)) * m.L * kSrRowsPerLayer * 64 : m.wpack;
    prm.P = (h->precision == DSX_PREC_FP16X2) ? 2 : 1;
  } else {
    prm.w = m.wpack;
    prm.P = (h->precision == DSX_PREC_FP16S) ? 2 : h->precision;   // DSX_PREC_FP16 = 1, FP16X2 = 2, FP16X3 = 3 == MMA passes
  }
  prm.fast_gate = gate_mode(h, prm.P);
  prm.dtab = h->ws.DTAB + static_cast<size_t>(row0) * m.L * kC;
  prm.d_row_stride = row_per_b * m.L * kC;
  const int per_launch = h->stack_mode ? l1 - l0 : 1;   // DSX_OPT_STACK_MODE = 0: one launch per layer
  for (int l = l0; l < l1; l += per_launch) {
    prm.l0 = l;
    prm.l1 = l + per_launch;
    DSX_TRY(launch_step(h, prm, rows, s));
  }
  if (stack) {
    h->stack_launches++;
    h->stack_rows_used = rows;
  }
  return DSX_OK;
}

// ------------------------------------------------------------------------------------------
// self-test: the operand loads (swizzle, row shift, zero fill) and the wgmma descriptors against a host GEMM
// ------------------------------------------------------------------------------------------
struct SelfParams {
  const __half* a;   // [T][256] fp16, one utterance
  const __half* w;   // [256 rows][64], plain (BULK = false) or packed as the kernels' weights (sw128_elem)
  float* out;        // [64][256] ([128][256] for the window)
  int t0, T;
  int off;           // window: row offset of the A operand from row kHalo + 64 wg (a tap's frame shift)
};

// GEMM1's conv-input window as k_hp_step<2, 3> holds it: channel block 1 of the window of the 128-frame tile at t0,
// copied by all 256 threads onto an mbarrier that the packed weight tile's bulk copy also completes.  Warpgroup wg
// multiplies the 64 rows from window row kHalo + 64 wg + off, a descriptor start that is not 1024-aligned.
__global__ void __launch_bounds__(256, 1) k_selftest_window(const __grid_constant__ SelfParams p) {
  uint8_t* base = smem_base();
  uint8_t* win = base + kWBytes;
  const uint32_t full = smem_u32(win + StepCfg<2, 3>::WBLK);
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127;
  float c0[64], c1[64];
  if (tid == 0) {
    mbar_init(full, 1 + 256);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_arrive_expect_tx(full, kWBytes);
    bulk_g2s(smem_u32(base), p.w, kWBytes, full);
  }
  load_wblock<256>(win, p.a, p.t0 - kHalo, 64, StepCfg<2, 3>::WROWS, p.T, tid);
  cp_arrive_noinc(full);
  mbar_wait(full, 0);
  fence_proxy_async_smem();
  const uint64_t a = wg_desc(smem_u32(win + (kHalo + wg * 64 + p.off) * 128)), w = wg_desc(smem_u32(base));
  wg_fence();
#pragma unroll
  for (int k4 = 0; k4 < 4; ++k4) {
    wgmma_n128(c0, a + 2 * k4, w + 2 * k4, k4 > 0);
    wgmma_n128(c1, a + 2 * k4, w + (16384 >> 4) + 2 * k4, k4 > 0);
  }
  wg_commit();
  wg_wait0();
  fence_acc(c0);
  fence_acc(c1);
  for (int e = 0; e < 64; ++e) {
    const int r = wg * 64 + acc_row(wtid, e), n = acc_col(wtid, e);
    p.out[r * 256 + n] = c0[e];
    p.out[r * 256 + 128 + n] = c1[e];
  }
}

// BULK = false: cp.async of the plain tile into the swizzled layout; true: one bulk copy of the packed tile, completing
// on an mbarrier together with the activation block's cp.async, as in the kernels' ring
template <bool BULK>
__global__ void __launch_bounds__(128, 1) k_selftest(const __grid_constant__ SelfParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int wtid = threadIdx.x;
  float c0[64], c1[64];
  if (BULK) {
    const uint32_t full = smem_u32(base + kWBytes + kABytes);
    if (wtid == 0) {
      mbar_init(full, 1 + 128);
      fence_mbar_init();
    }
    __syncthreads();
    if (wtid == 0) {
      mbar_arrive_expect_tx(full, kWBytes);
      bulk_g2s(smem_u32(base), p.w, kWBytes, full);
    }
    load_a(base + kWBytes, p.a, 0, p.t0, 0, p.T, p.T, wtid);
    cp_arrive_noinc(full);
    mbar_wait(full, 0);
    fence_proxy_async_smem();
  } else {
    load_w<128>(base, p.w, p.w + 128 * 64, 256, wtid);
    load_a(base + kWBytes, p.a, 0, p.t0, 0, p.T, p.T, wtid);
    cp_commit();
    cp_wait<0>();
    fence_proxy_async_smem();
    __syncthreads();
  }
  const uint64_t a = wg_desc(smem_u32(base + kWBytes)), w = wg_desc(smem_u32(base));
  wg_fence();
#pragma unroll
  for (int k4 = 0; k4 < 4; ++k4) {
    wgmma_n128(c0, a + 2 * k4, w + 2 * k4, k4 > 0);
    wgmma_n128(c1, a + 2 * k4, w + (16384 >> 4) + 2 * k4, k4 > 0);
  }
  wg_commit();
  wg_wait0();
  fence_acc(c0);
  fence_acc(c1);
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
  std::vector<__half> ha(static_cast<size_t>(T) * 256), hw(256 * 64), hwp(256 * 64);
  for (int t = 0; t < T; ++t)
    for (int c = 0; c < 256; ++c) ha[static_cast<size_t>(t) * 256 + c] = __float2half(aval(t, c));
  for (int n = 0; n < 256; ++n)
    for (int k = 0; k < 64; ++k) {
      hw[static_cast<size_t>(n) * 64 + k] = __float2half(wval(n, k));
      hwp[sw128_elem(n, k)] = __float2half(wval(n, k));
    }
  __half *da = nullptr, *dw = nullptr, *dwp = nullptr;
  float* dout = nullptr;
  DSX_CUDA(cudaMalloc(&da, ha.size() * 2));
  DSX_CUDA(cudaMalloc(&dw, hw.size() * 2));
  DSX_CUDA(cudaMalloc(&dwp, hwp.size() * 2));
  DSX_CUDA(cudaMalloc(&dout, 128 * 256 * 4));
  DSX_CUDA(cudaMemcpy(da, ha.data(), ha.size() * 2, cudaMemcpyHostToDevice));
  DSX_CUDA(cudaMemcpy(dw, hw.data(), hw.size() * 2, cudaMemcpyHostToDevice));
  DSX_CUDA(cudaMemcpy(dwp, hwp.data(), hwp.size() * 2, cudaMemcpyHostToDevice));
  const int smem = 1024 + kWBytes + kABytes + 8;
  DSX_CUDA(cudaFuncSetAttribute(k_selftest<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  DSX_CUDA(cudaFuncSetAttribute(k_selftest<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int failures = 0;
  const int starts[] = {0, -8, 37, 120};     // interior, leading zero fill, unaligned, trailing zero fill
  for (int bulk = 0; bulk < 2; ++bulk)
    for (int t0 : starts) {
      SelfParams prm{da, bulk ? dwp : dw, dout, t0, T};
      DSX_CUDA(cudaMemset(dout, 0xff, 64 * 256 * 4));
      if (bulk) k_selftest<true><<<1, 128, smem>>>(prm);
      else k_selftest<false><<<1, 128, smem>>>(prm);
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
      snprintf(line, sizeof(line), "wgmma_m64n128k16 %s t0=%d: bad=%d/16384 maxerr=%.3g\n",
               bulk ? "bulk-copied packed tile" : "cp.async tile", t0, bad, maxerr);
      report += line;
      if (bad) failures++;
    }
  // the window: tile at 0 of a 130-frame utterance (zero rows before frame 0 and from frame 130 on) and tile at 128 of
  // the 150-frame one (real rows before the tile, zero rows after the utterance); taps at +-d for every dilation
  const int wsmem = 1024 + kWBytes + StepCfg<2, 3>::WBLK + 8;
  DSX_CUDA(cudaFuncSetAttribute(k_selftest_window, cudaFuncAttributeMaxDynamicSharedMemorySize, wsmem));
  const int wins[2][2] = {{0, 130}, {128, T}};
  const int offs[] = {-8, -4, -2, -1, 0, 1, 2, 4, 8};
  for (const auto& wt : wins) {
    int bad = 0;
    double maxerr = 0;
    for (int off : offs) {
      SelfParams prm{da, dwp, dout, wt[0], wt[1], off};
      DSX_CUDA(cudaMemset(dout, 0xff, 128 * 256 * 4));
      k_selftest_window<<<1, 256, wsmem>>>(prm);
      DSX_CUDA(cudaGetLastError());
      DSX_CUDA(cudaDeviceSynchronize());
      std::vector<float> out(128 * 256);
      DSX_CUDA(cudaMemcpy(out.data(), dout, out.size() * 4, cudaMemcpyDeviceToHost));
      for (int m = 0; m < 128; ++m)
        for (int n = 0; n < 256; ++n) {
          double ref = 0;
          const int t = wt[0] + m + off;
          if (t >= 0 && t < wt[1])
            for (int k = 0; k < 64; ++k) ref += static_cast<double>(aval(t, 64 + k)) * wval(n, k);
          const double e = fabs(ref - out[static_cast<size_t>(m) * 256 + n]);
          if (!(e <= 1e-4)) bad++;
          if (e > maxerr || e != e) maxerr = e;
        }
    }
    char line[160];
    snprintf(line, sizeof(line), "wgmma_m64n128k16 window t0=%d T=%d rows 8+-{0,1,2,4,8}, 2 warpgroups: bad=%d/294912 maxerr=%.3g\n",
             wt[0], wt[1], bad, maxerr);
    report += line;
    if (bad) failures++;
  }
  cudaFree(da);
  cudaFree(dw);
  cudaFree(dwp);
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
