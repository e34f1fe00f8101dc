// FastSpeech2 encoder on sm_90a: txt_tokens [B, T] (+ the MIDI addends) -> encoder_out [B, T, H]
// (FastspeechEncoder, modules/fastspeech/tts_modules.py:310-347; FastspeechMIDIEncoder, modules/diffsinger_midi/fs2.py:11-36),
// in eval mode, and the length regulator (LengthRegulator, tts_modules.py:159-189).
//
// Encoder, per call 1 (relative positions) or 2 (sinusoidal) + 5 L launches over frames-major buffers:
//   k_pos_scan_tokens   make_positions(txt_tokens) (dsx_posemb.cuh), sinusoidal mode only
//   k_fs2enc_embed      one warp per token: x = sqrt(H) E[tok], ((x + midi) + midi_dur) + slur, the position term,
//                       x * !pad (pad = tok == 0) -> fp32 X and PAD, and layer 0's layer_norm1 -> fp16 A
//   fs2_layers_run      the FastSpeech2 decoder's L layers and final LayerNorm * !pad (dsx_fs2dec.cu) -> fp32 out
// The encoder's FFTBlocks have no position embedding of their own and no pos_embed_alpha (use_pos_embed=False in
// FastspeechEncoder.__init__), so the decoder's entry (k_pos_scan over channel 0 + k_fs2_embed) is not run.
//
// Length regulator, two calls because T_mel depends on the data:
//   k_lr_totals   one block per utterance: d = rint(float(dur) * alpha) * !pad, its inclusive int64 scan, the total and a
//                 flag for a negative d
//   k_lr_fill     one thread per output frame: binary search of the frame in the utterance's scan
#include <math.h>
#include <stdio.h>

#include "dsx_conv.cuh"
#include "dsx_internal.h"
#include "dsx_posemb.cuh"

namespace dsx {
namespace {

constexpr float kEncLnEps = 1e-5f;   // nn.LayerNorm of EncSALayer

struct EncAddends {
  const float* p[3];          // midi_embedding, midi_dur_embedding, slur_embedding, or NULL
  dsx_strides s[3];
};

// row t of RelPositionalEncoding's reversed table (espnet_positional_embedding.py:23-45): position P - 1 - t, sin at even
// and cos at odd channels of div_term[c / 2] = exp(2 (c / 2) * neg), neg = -ln(1e4) / H
__device__ __forceinline__ float rel_table(int ps, int c, float neg) {
  const float div = expf(static_cast<float>(c & ~1) * neg);
  const float arg = static_cast<float>(ps) * div;
  return (c & 1) ? cosf(arg) : sinf(arg);
}

// One warp per token, H / 32 <= 8 channels per lane.  mode 0: x + table[pos] (sinusoidal, pos from k_pos_scan_tokens);
// mode 1: x * sqrt(H) + rel_table(P - 1 - t).  An id outside [0, vocab) reads a zero row.  Training (the encoder training
// step, dsx_fs2enctrain.cu): dropout site `drop` before the * !pad, and X copied to xsave.
__global__ void k_fs2enc_embed(const int64_t* tok, int rows, int T, int H, const float* E, int vocab, float scale,
                               EncAddends add, int mode, const int* pos, float neg_emb, int rel_len, float rel_neg,
                               const float* ln_w, const float* ln_b, float* X, uint8_t* PAD, __half* A, Fs2Drop drop,
                               float* xsave) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows) return;
  const int b = warp / T, t = warp - b * T, per = H / 32;
  const int64_t id = tok[warp];
  const bool keep = id != 0, in_range = id >= 0 && id < vocab;
  const float* er = E + (in_range ? id : 0) * static_cast<int64_t>(H);
  float* xr = X + static_cast<size_t>(warp) * H;
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    if (i >= per) break;
    const int c = lane + 32 * i;
    float x = scale * (in_range ? er[c] : 0.f);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (add.p[k]) x = x + add.p[k][b * add.s[k].b + c * add.s[k].c + t * add.s[k].t];
    }
    x = mode == 0 ? x + pos_table(pos[warp], c, H, neg_emb) : x * scale + rel_table(rel_len - 1 - t, c, rel_neg);
    if (drop.site >= 0) x *= dropout_scale(drop, warp, c);
    v[i] = keep ? x : 0.f;
    xr[c] = v[i];
    if (xsave) xsave[static_cast<size_t>(warp) * H + c] = v[i];
  }
  if (lane == 0) PAD[warp] = keep ? 0 : 1;
  warp_row_ln16(v, per, H, kEncLnEps, ln_w, ln_b, A + static_cast<size_t>(warp) * H);
}

// ---- length regulator ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kScanThreads) k_lr_totals(const int64_t* dur, const uint8_t* pad, int B, int T,
                                                            float alpha, int64_t* cum, int64_t* totals) {
  __shared__ long long sh[kScanThreads];
  __shared__ int neg;
  if (threadIdx.x == 0) neg = 0;
  __syncthreads();
  const size_t row = static_cast<size_t>(blockIdx.x) * T;
  // torch.round(dur.float() * alpha).long() * (1 - dur_padding.long())
  auto val = [&](int t) -> long long {
    if (pad && pad[row + t]) return 0;
    return static_cast<long long>(rintf(__ll2float_rn(dur[row + t]) * alpha));
  };
  block_scan<long long>(sh, T, val, [&](int t, long long s, long long d) {
    cum[row + t] = s;
    if (d < 0) neg = 1;
    if (t == T - 1) totals[blockIdx.x] = s;
  });
  __syncthreads();
  if (threadIdx.x == 0 && neg) totals[B] = 1;   // zeroed before the launch
}

// mel2ph[b][f] = 1 + the first t with cum[b][t] > f, for f < totals[b]; else 0
__global__ void k_lr_fill(const int64_t* cum, const int64_t* totals, int B, int T, int Tm, int64_t* mel2ph) {
  const size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<size_t>(B) * Tm) return;
  const int b = static_cast<int>(i / Tm);
  const long long f = static_cast<long long>(i - static_cast<size_t>(b) * Tm);
  if (f >= totals[b]) {
    mel2ph[i] = 0;
    return;
  }
  const int64_t* c = cum + static_cast<size_t>(b) * T;
  int lo = 0, hi = T - 1;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (c[mid] > f) {
      hi = mid;
    } else {
      lo = mid + 1;
    }
  }
  mel2ph[i] = lo + 1;
}

}  // namespace

int fs2enc_entry(const dsx_fs2dec* stack, int pos_mode, const float* E, int vocab, const int64_t* tokens, int B, int T,
                 const float* const* add, const dsx_strides* as, int rel_len, const Fs2Bufs& w, __half* A,
                 const Fs2Drop& drop, float* xsave, cudaStream_t s) {
  EncAddends ad{};
  for (int k = 0; k < 3; ++k) {
    ad.p[k] = add ? add[k] : nullptr;
    if (ad.p[k]) {
      DSX_CHECK(as, DSX_E_INVALID, "addend %d has no strides", k);
      ad.s[k] = as[k];
    }
  }
  const int H = fs2_config(stack).hidden;
  if (pos_mode == 0) {
    k_pos_scan_tokens<<<B, kScanThreads, 0, s>>>(tokens, T, w.POS);
    DSX_TRY(launch_check("k_pos_scan_tokens"));
  }
  const float* ln_w;
  const float* ln_b;
  fs2_first_ln(stack, &ln_w, &ln_b);
  const size_t frames = static_cast<size_t>(B) * T;
  k_fs2enc_embed<<<static_cast<unsigned>((frames * 32 + 255) / 256), 256, 0, s>>>(
      tokens, static_cast<int>(frames), T, H, E, vocab, static_cast<float>(sqrt(static_cast<double>(H))), ad, pos_mode,
      w.POS, pos_neg_emb(H), rel_len, -static_cast<float>(log(10000.0) / H), ln_w, ln_b, w.X, w.PAD, A, drop, xsave);
  return launch_check("k_fs2enc_embed");
}

}  // namespace dsx

using namespace dsx;

struct dsx_fs2enc {
  int device = 0;
  dsx_fs2enc_config cfg{};
  dsx_fs2dec* stack = nullptr;   // the FFTBlocks layers and final LayerNorm (packed by fs2_load)
  float* embed = nullptr;        // embed_tokens.weight [vocab][H]
  bool loaded = false;
  DevAllocs mem;
  GrowBuffer ws;
};

extern "C" {

int dsx_fs2enc_create(int device, const dsx_fs2enc_config* cfg, dsx_fs2enc** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_CHECK(cfg, DSX_E_INVALID, "config is NULL");
  DSX_CHECK(cfg->vocab >= 1, DSX_E_INVALID, "unsupported vocab %d: at least 1 row of embed_tokens", cfg->vocab);
  DSX_CHECK(cfg->pos == 0 || cfg->pos == 1, DSX_E_INVALID, "unsupported pos %d: 0 (sinusoidal) or 1 (relative)",
            cfg->pos);
  dsx_fs2dec* stack = nullptr;
  DSX_TRY(dsx_fs2dec_create(device, &cfg->stack, &stack));
  dsx_fs2enc* h = new dsx_fs2enc();
  h->device = device;
  h->cfg = *cfg;
  h->stack = stack;
  *out = h;
  return DSX_OK;
}

void dsx_fs2enc_destroy(dsx_fs2enc* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  dsx_fs2dec_destroy(h->stack);
  h->mem.free_all();
  h->ws.release();
  delete h;
}

int dsx_fs2enc_load(dsx_fs2enc* h, const dsx_fs2enc_params* p, void* stream) {
  DSX_CHECK(h && p, DSX_E_INVALID, "null handle or params");
  DSX_CHECK(p->embed_w, DSX_E_INVALID, "missing embed_tokens.weight");
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  h->loaded = false;
  DSX_TRY(fs2_load(h->stack, &p->stack, stream));   // synchronises s before it frees the old packs
  h->mem.free_all();
  const size_t n = static_cast<size_t>(h->cfg.vocab) * h->cfg.stack.hidden;
  DSX_TRY(h->mem.alloc(&h->embed, n * sizeof(float)));
  DSX_CUDA(cudaMemcpyAsync(h->embed, p->embed_w, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
  h->loaded = true;
  return DSX_OK;
}

int dsx_fs2enc_forward(dsx_fs2enc* h, const int64_t* tokens, int B, int T, const float* const* add, const dsx_strides* as,
                       int rel_len, float* out, void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(h->loaded, DSX_E_STATE, "dsx_fs2enc_load has not been called");
  DSX_CHECK(tokens && out, DSX_E_INVALID, "tokens and out must not be NULL");
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(B <= 65535, DSX_E_INVALID, "B = %d utterances per call is above the 65535 the launch grid holds", B);
  DSX_CHECK(h->cfg.pos == 0 || rel_len >= T, DSX_E_INVALID, "rel_len %d is shorter than T = %d", rel_len, T);
  const int Tp = (T + kConvRows - 1) / kConvRows * kConvRows;
  DSX_CHECK(static_cast<long long>(B) * Tp * 4 * h->cfg.stack.hidden < (1ll << 31), DSX_E_INVALID,
            "B * T = %lld tokens is too large", static_cast<long long>(B) * T);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_TRY(h->ws.reserve(fs2_workspace_bytes(h->stack, B, T), s));
  const Fs2Bufs w = fs2_carve(h->stack, h->ws.ptr, B, T);
  DSX_TRY(fs2enc_entry(h->stack, h->cfg.pos, h->embed, h->cfg.vocab, tokens, B, T, add, as, rel_len, w, w.A, Fs2Drop{},
                       nullptr, s));
  return fs2_layers_run(h->stack, w, B, T, out, nullptr, s);
}

int dsx_length_totals(const int64_t* dur, const uint8_t* pad, int B, int T, float alpha, int64_t* cum, int64_t* totals,
                      void* stream) {
  DSX_CHECK(dur && cum && totals, DSX_E_INVALID, "dur, cum and totals must not be NULL");
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(alpha > 0.f, DSX_E_INVALID, "alpha must be positive (got %g)", static_cast<double>(alpha));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_CUDA(cudaMemsetAsync(totals + B, 0, sizeof(int64_t), s));
  k_lr_totals<<<B, kScanThreads, 0, s>>>(dur, pad, B, T, alpha, cum, totals);
  return launch_check("k_lr_totals");
}

int dsx_length_regulate(const int64_t* cum, const int64_t* totals, int B, int T, int T_mel, int64_t* mel2ph,
                        void* stream) {
  DSX_CHECK(cum && totals, DSX_E_INVALID, "cum and totals must not be NULL");
  DSX_CHECK(B > 0 && T > 0 && T_mel >= 0, DSX_E_INVALID, "bad sizes B %d, T %d, T_mel %d", B, T, T_mel);
  if (T_mel == 0) return DSX_OK;
  DSX_CHECK(mel2ph, DSX_E_INVALID, "mel2ph must not be NULL");
  const size_t n = static_cast<size_t>(B) * T_mel;
  k_lr_fill<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(cum, totals, B, T,
                                                                                                   T_mel, mel2ph);
  return launch_check("k_lr_fill");
}

}  // extern "C"
