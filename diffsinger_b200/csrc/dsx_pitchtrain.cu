// Pitch and energy predictors on sm_90a: PitchPredictor.forward (modules/fastspeech/tts_modules.py:192-240) in eval mode
// and as a training step with a saved tape and the exact backward.  P = chans, F = B T frames.
//
// The predictor is the duration predictor's stack (dsx_pe.cu, dsx_durtrain.cu) with four differences: the position term
// at the input, no mask, a head of odim <= 16 outputs, and the gradient of pos_embed_alpha.  So both handles wrap the
// duration predictor's (a dsx_durpred for eval, a dsx_durpred_train for training) and add only those:
//   forward   k_pos_scan and k_pos_add (dsx_posemb.cuh): x + alpha table[pos] -> layer 0's fp16 operand; dp_stack_run
//             without a mask: each layer's k_pe_conv, the last one writing its output (after dropout) in fp32; k_ppt_head:
//             Linear(P, odim), one warp per frame.  Training adds k_tape_hdr (the tape's header) and the duration
//             predictor's conv weight pack (without its head), and saves the positions, the layers' inputs and the head's input to the tape.
//   backward  dpt_backward with no mask and odim outputs (the head's backward, then per layer wgrad and the transposed
//             conv with the layer below's backward in its epilogue), always down to d_in, the gradient at layer 0's
//             input (= d_x); then k_ppt_alpha_part and k_ppt_alpha_sum: d alpha = sum d_in . table[pos] over a fixed
//             grid, summed in order.
// The eval forward runs the same kernels as the training forward (k_pe_conv's eval instantiation, whose results equal
// the training one's at p = 0), so the training forward at p = 0 gives the eval forward's bits.
#include <math.h>

#include <algorithm>

#include "dsx_conv.cuh"
#include "dsx_internal.h"
#include "dsx_posemb.cuh"
#include "dsx_wgrad.cuh"

namespace dsx {
namespace {

constexpr int kPpMaxOdim = 16;
constexpr int kAlphaBlocks = 256;   // CTAs of k_ppt_alpha_part: fixed, so the partial sums have a fixed order

// out[f][o] = b[o] + sum_c hin[f][c] W[o][c] (tts_modules.py:234), one warp per frame, P <= 256
__global__ void __launch_bounds__(256) k_ppt_head(const float* hin, const float* W, const float* b, int F, int P, int od,
                                                  float* out) {
  const int f = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (f >= F) return;
  const float* row = hin + static_cast<size_t>(f) * P;
  float h[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) h[i] = lane + 32 * i < P ? row[lane + 32 * i] : 0.f;
  for (int o = 0; o < od; ++o) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      if (lane + 32 * i < P) s += h[i] * W[o * P + lane + 32 * i];
#pragma unroll
    for (int k = 16; k > 0; k >>= 1) s += __shfl_xor_sync(0xffffffffu, s, k);
    if (lane == 0) out[static_cast<size_t>(f) * od + o] = s + b[o];
  }
}

// d alpha partials: CTA z sums d_in[i] table[pos[i / n]][i % n] over i = z * 256 + tid + k * kAlphaBlocks * 256, then
// over its threads in a fixed tree
__global__ void __launch_bounds__(256) k_ppt_alpha_part(const float* din, const int* pos, size_t F, int n, float neg_emb,
                                                        float* part) {
  __shared__ float red[256];
  float s = 0.f;
  const size_t total = F * n;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % n);
    s += din[i] * pos_table(pos[i / n], c, n, neg_emb);
  }
  red[threadIdx.x] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = red[0];
}

__global__ void k_ppt_alpha_sum(const float* part, int n, float* out) {
  float s = 0.f;
  for (int i = 0; i < n; ++i) s += part[i];
  out[0] = s;
}

inline dsx_durpred_config dp_config(const dsx_pitchpred_config& c) {
  dsx_durpred_config d{};
  d.idim = c.idim;
  d.chans = c.chans;
  d.layers = c.layers;
  d.kernel = c.kernel;
  d.padding = c.padding;
  d.offset = 1.f;   // out2dur's; the pitch predictor has no duration head
  return d;
}

inline dsx_durpred_params dp_params(const dsx_pitchpred_params& p) {
  return dsx_durpred_params{p.conv_w, p.conv_b, p.ln_w, p.ln_b, p.linear_w, p.linear_b};
}

int pp_validate(const dsx_pitchpred_config* c) {
  DSX_CHECK(c, DSX_E_INVALID, "config is NULL");
  DSX_CHECK(c->odim >= 1 && c->odim <= kPpMaxOdim, DSX_E_INVALID, "unsupported odim %d: 1..%d", c->odim, kPpMaxOdim);
  return DSX_OK;   // the rest is the duration predictor's check
}

int pp_check_geom(const dsx_pitchpred_config& c, int B, int T) {
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(B <= 65535, DSX_E_INVALID, "B = %d utterances per call is above the 65535 the launch grid holds", B);
  const long long Tp = (T + kConvRows - 1) / kConvRows * kConvRows;
  DSX_CHECK(static_cast<long long>(B) * Tp * std::max(c.idim, c.chans) < (1ll << 31), DSX_E_INVALID,
            "B * T = %lld frames is too large", static_cast<long long>(B) * T);
  return DSX_OK;
}

int pp_check_params(const dsx_pitchpred_params* p, int L, const char* what) {
  DSX_CHECK(p, DSX_E_INVALID, "%s is NULL", what);
  DSX_CHECK(p->conv_w && p->conv_b && p->ln_w && p->ln_b && p->linear_w && p->linear_b && p->pos_embed_alpha,
            DSX_E_INVALID, "a pointer of %s is NULL", what);
  for (int l = 0; l < L; ++l)
    DSX_CHECK(p->conv_w[l] && p->conv_b[l] && p->ln_w[l] && p->ln_b[l], DSX_E_INVALID,
              "a pointer of layer %d of %s is NULL", l, what);
  return DSX_OK;
}

// the position term: pos over channel 0 of x [B][T][idim], then fp16(x + alpha table[pos]) -> a0.  2 launches.
int pp_entry(const float* x, const float* alpha, int B, int T, int idim, int* pos, __half* a0, cudaStream_t s) {
  k_pos_scan<<<B, kScanThreads, 0, s>>>(x, T, idim, pos);
  DSX_TRY(launch_check("k_pos_scan"));
  const size_t ne = static_cast<size_t>(B) * T * idim;
  k_pos_add<<<static_cast<unsigned>((ne + 255) / 256), 256, 0, s>>>(x, pos, alpha, B * T, idim, pos_neg_emb(idim), a0);
  return launch_check("k_pos_add");
}

int pp_head(const float* hin, const float* W, const float* b, int F, int P, int od, float* out, cudaStream_t s) {
  k_ppt_head<<<static_cast<unsigned>((static_cast<size_t>(F) * 32 + 255) / 256), 256, 0, s>>>(hin, W, b, F, P, od, out);
  return launch_check("k_ppt_head");
}

struct PpTape {
  DurTape d;                   // d.pad is NULL: nothing is masked
  int* pos;                    // [F] int32
};

// every region of the tape for (config, B, T), in order; bytes of the whole tape
size_t pp_tape_carve(const dsx_pitchpred_config& c, int B, int T, uint8_t* base, PpTape* t) {
  const size_t F = static_cast<size_t>(B) * T, P = c.chans;
  const int L = c.layers;
  size_t n = 0;
  auto take = [&](size_t bytes) {
    uint8_t* q = base ? base + n : nullptr;
    n += align256(bytes);
    return q;
  };
  PpTape dummy;
  PpTape& tp = t ? *t : dummy;
  tp.d.hdr = reinterpret_cast<Fs2TapeHdr*>(take(sizeof(Fs2TapeHdr)));
  tp.d.pad = nullptr;
  tp.pos = reinterpret_cast<int*>(take(4 * F));
  tp.d.tr.a.resize(L);
  tp.d.tr.r.resize(L);
  tp.d.tr.a[0] = reinterpret_cast<__half*>(take(2 * F * c.idim));
  for (int l = 0; l < L; ++l) tp.d.tr.r[l] = reinterpret_cast<float*>(take(4 * F * P));
  for (int l = 1; l < L; ++l) tp.d.tr.a[l] = reinterpret_cast<__half*>(take(2 * F * P));
  tp.d.tr.hin = reinterpret_cast<float*>(take(4 * F * P));
  return n;
}

}  // namespace
}  // namespace dsx

using namespace dsx;

struct dsx_pitchpred {
  int device = 0;
  dsx_pitchpred_config cfg{};
  dsx_durpred* dp = nullptr;   // the convolutions' packs and LayerNorm affines
  bool loaded = false;
  float* head = nullptr;       // linear.weight [odim][P], bias [odim]
  float* alpha = nullptr;      // pos_embed_alpha [1]
  DevAllocs mem;
  GrowBuffer ws;
};

struct dsx_pitchpred_train {
  int device = 0;
  dsx_pitchpred_config cfg{};
  dsx_durpred_train* dp = nullptr;   // the duration predictor's step: packs, kernels and backward
};

namespace {

size_t pp_ws_bytes(const dsx_pitchpred_train* h, int B, int T) {
  const size_t F = static_cast<size_t>(B) * T;
  return dpt_workspace_bytes(h->dp, B, T, h->cfg.odim) + align256(4 * F * h->cfg.idim) + align256(4 * kAlphaBlocks);
}

}  // namespace

extern "C" {

int dsx_pitchpred_create(int device, const dsx_pitchpred_config* cfg, dsx_pitchpred** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_TRY(pp_validate(cfg));
  const dsx_durpred_config dc = dp_config(*cfg);
  dsx_durpred* dp = nullptr;
  DSX_TRY(dsx_durpred_create(device, &dc, &dp));   // validates the rest and selects the device
  dsx_pitchpred* h = new dsx_pitchpred();
  h->device = device;
  h->cfg = *cfg;
  h->dp = dp;
  *out = h;
  return DSX_OK;
}

void dsx_pitchpred_destroy(dsx_pitchpred* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  h->mem.free_all();
  h->ws.release();
  dsx_durpred_destroy(h->dp);
  delete h;
}

int dsx_pitchpred_load(dsx_pitchpred* h, const dsx_pitchpred_params* p, void* stream) {
  DSX_CHECK(h && p, DSX_E_INVALID, "null handle or params");
  DSX_CHECK(p->linear_w && p->linear_b && p->pos_embed_alpha, DSX_E_INVALID, "missing linear or pos_embed_alpha");
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const dsx_durpred_params dpp = dp_params(*p);
  DSX_TRY(dsx_durpred_load(h->dp, &dpp, stream));   // synchronises s before it frees the old packs
  h->mem.free_all();
  h->loaded = false;
  const int P = h->cfg.chans, od = h->cfg.odim;
  DSX_TRY(h->mem.alloc(&h->head, (od * P + od) * sizeof(float)));
  DSX_TRY(h->mem.alloc(&h->alpha, sizeof(float)));
  DSX_CUDA(cudaMemcpyAsync(h->head, p->linear_w, od * P * sizeof(float), cudaMemcpyDeviceToDevice, s));
  DSX_CUDA(cudaMemcpyAsync(h->head + od * P, p->linear_b, od * sizeof(float), cudaMemcpyDeviceToDevice, s));
  DSX_CUDA(cudaMemcpyAsync(h->alpha, p->pos_embed_alpha, sizeof(float), cudaMemcpyDeviceToDevice, s));
  h->loaded = true;
  return DSX_OK;
}

int dsx_pitchpred_forward(dsx_pitchpred* h, const float* x, int B, int T, float* out, void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(h->loaded, DSX_E_STATE, "dsx_pitchpred_load has not been called");
  DSX_CHECK(x && out, DSX_E_INVALID, "x and out must not be NULL");
  const dsx_pitchpred_config& c = h->cfg;
  DSX_TRY(pp_check_geom(c, B, T));
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t F = static_cast<size_t>(B) * T;
  const int P = c.chans, C = std::max(c.idim, P);
  DSX_TRY(h->ws.reserve(align256(4 * F) + 2 * align256(2 * F * C) + align256(4 * F * P), s));
  Bump ws{static_cast<uint8_t*>(h->ws.ptr)};
  int* pos = ws.take<int>(4 * F);
  __half* A[2] = {ws.take<__half>(2 * F * C), ws.take<__half>(2 * F * C)};
  float* hin = ws.take<float>(4 * F * P);
  DSX_TRY(pp_entry(x, h->alpha, B, T, c.idim, pos, A[0], s));
  DSX_TRY(dp_stack_run(h->dp, A, nullptr, B, T, nullptr, nullptr, nullptr, hin, s));
  return pp_head(hin, h->head, h->head + c.odim * P, static_cast<int>(F), P, c.odim, out, s);
}

int dsx_pitchpred_train_create(int device, const dsx_pitchpred_config* cfg, dsx_pitchpred_train** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_TRY(pp_validate(cfg));
  const dsx_durpred_config dc = dp_config(*cfg);
  dsx_durpred_train* dp = nullptr;
  DSX_TRY(dsx_durpred_train_create(device, &dc, &dp));   // validates the rest and selects the device
  dsx_pitchpred_train* h = new dsx_pitchpred_train();
  h->device = device;
  h->cfg = *cfg;
  h->dp = dp;
  *out = h;
  return DSX_OK;
}

void dsx_pitchpred_train_destroy(dsx_pitchpred_train* h) {
  if (!h) return;
  dsx_durpred_train_destroy(h->dp);
  delete h;
}

int dsx_pitchpred_train_tape_bytes(dsx_pitchpred_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  DSX_TRY(pp_check_geom(h->cfg, B, T));
  *out = pp_tape_carve(h->cfg, B, T, nullptr, nullptr);
  return DSX_OK;
}

int dsx_pitchpred_train_workspace_bytes(dsx_pitchpred_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  DSX_TRY(pp_check_geom(h->cfg, B, T));
  *out = pp_ws_bytes(h, B, T);
  return DSX_OK;
}

int dsx_pitchpred_train_forward(dsx_pitchpred_train* h, const dsx_pitchpred_params* w, const float* x, int B, int T,
                                float p_drop, uint64_t seed, void* tape, size_t tape_bytes, void* workspace,
                                size_t workspace_bytes, float* out, void* stream) {
  (void)workspace;   // the forward writes only the tape and out
  (void)workspace_bytes;
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  const dsx_pitchpred_config& c = h->cfg;
  DSX_TRY(pp_check_geom(c, B, T));
  DSX_TRY(pp_check_params(w, c.layers, "the parameters"));
  DSX_CHECK(x && tape && out, DSX_E_INVALID, "x, tape and out must not be NULL");
  DSX_CHECK(p_drop >= 0.f && p_drop < 1.f, DSX_E_INVALID, "dropout p = %g is outside [0, 1)", static_cast<double>(p_drop));
  const size_t need = pp_tape_carve(c, B, T, nullptr, nullptr);
  DSX_CHECK(tape_bytes >= need, DSX_E_INVALID, "tape of %zu bytes is below the %zu this (B, T) needs", tape_bytes, need);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PpTape tp;
  pp_tape_carve(c, B, T, static_cast<uint8_t*>(tape), &tp);
  tp.d.tr.seed = seed;
  tp.d.tr.p = p_drop;
  k_tape_hdr<<<1, 1, 0, s>>>(tp.d.hdr, seed, p_drop, B, T);
  DSX_TRY(launch_check("k_tape_hdr"));
  dsx_durpred* fwd = dpt_forward_handle(h->dp);
  const dsx_durpred_params dpp = dp_params(*w);
  DSX_TRY(durpred_train_pack(fwd, &dpp, s, false));
  DSX_TRY(pp_entry(x, w->pos_embed_alpha, B, T, c.idim, tp.pos, tp.d.tr.a[0], s));
  DSX_TRY(dp_stack_run(fwd, nullptr, nullptr, B, T, nullptr, nullptr, &tp.d.tr, tp.d.tr.hin, s));
  return pp_head(tp.d.tr.hin, w->linear_w, w->linear_b, B * T, c.chans, c.odim, out, s);
}

int dsx_pitchpred_train_backward(dsx_pitchpred_train* h, const dsx_pitchpred_params* w, const void* tape,
                                 const float* d_out, const dsx_pitchpred_params* grads, float* d_x, int B, int T,
                                 void* workspace, size_t workspace_bytes, void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  const dsx_pitchpred_config& c = h->cfg;
  DSX_TRY(pp_check_geom(c, B, T));
  DSX_TRY(pp_check_params(w, c.layers, "the parameters"));
  DSX_TRY(pp_check_params(grads, c.layers, "the gradients"));
  DSX_CHECK(tape && d_out && workspace, DSX_E_INVALID, "tape, d_out and workspace must not be NULL");
  const size_t wneed = pp_ws_bytes(h, B, T);
  DSX_CHECK(workspace_bytes >= wneed, DSX_E_INVALID, "workspace of %zu bytes is below the %zu this (B, T) needs",
            workspace_bytes, wneed);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PpTape tp;
  pp_tape_carve(c, B, T, static_cast<uint8_t*>(const_cast<void*>(tape)), &tp);
  const size_t F = static_cast<size_t>(B) * T;
  Bump extra{static_cast<uint8_t*>(workspace) + dpt_workspace_bytes(h->dp, B, T, c.odim)};
  float* din_ws = extra.take<float>(4 * F * c.idim);
  float* apart = extra.take<float>(4 * kAlphaBlocks);
  float* din = d_x ? d_x : din_ws;   // d alpha needs the input gradient whether or not the caller does
  const dsx_durpred_params dw = dp_params(*w), dg = dp_params(*grads);
  DSX_TRY(dpt_backward(h->dp, &dw, tp.d, d_out, c.odim, &dg, din, B, T, workspace, s));
  k_ppt_alpha_part<<<kAlphaBlocks, 256, 0, s>>>(din, tp.pos, F, c.idim, pos_neg_emb(c.idim), apart);
  DSX_TRY(launch_check("k_ppt_alpha_part"));
  k_ppt_alpha_sum<<<1, 1, 0, s>>>(apart, kAlphaBlocks, const_cast<float*>(grads->pos_embed_alpha));
  return launch_check("k_ppt_alpha_sum");
}

int dsx_pitchpred_train_masks(dsx_pitchpred_train* h, uint64_t seed, float p_drop, int B, int T, uint8_t* const* out,
                              void* stream) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  return dsx_durpred_train_masks(h->dp, seed, p_drop, B, T, out, stream);
}

}  // extern "C"
