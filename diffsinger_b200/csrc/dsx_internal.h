// Internal declarations shared by the dsx translation units (not part of the C ABI).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/dsx.h"
#include "dsx_rng.cuh"

namespace dsx {

void set_error(const char* fmt, ...);
#define DSX_CUDA(expr)                                                                        \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      ::dsx::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return DSX_E_CUDA;                                                                      \
    }                                                                                         \
  } while (0)
#define DSX_CHECK(cond, code, ...)     \
  do {                                 \
    if (!(cond)) {                     \
      ::dsx::set_error(__VA_ARGS__);   \
      return (code);                   \
    }                                  \
  } while (0)
#define DSX_TRY(expr)          \
  do {                         \
    int _r = (expr);           \
    if (_r != DSX_OK) return _r; \
  } while (0)

// ---- handle plumbing ------------------------------------------------------------------------------
// the error of the last launch, if any, as DSX_E_CUDA naming the kernel
inline int launch_check(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return DSX_E_CUDA;
  }
  return DSX_OK;
}

// cudaMalloc of at least one byte; out of memory is DSX_E_NOMEM, any other failure DSX_E_CUDA
inline int checked_malloc(void** p, size_t bytes) {
  cudaError_t e = cudaMalloc(p, bytes ? bytes : 1);
  if (e != cudaSuccess) {
    set_error("cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    return e == cudaErrorMemoryAllocation ? DSX_E_NOMEM : DSX_E_CUDA;
  }
  return DSX_OK;
}

// device allocations freed together (a model's packed weights)
struct DevAllocs {
  std::vector<void*> ptrs;
  template <typename T>
  int alloc(T** p, size_t bytes) {
    DSX_TRY(checked_malloc(reinterpret_cast<void**>(p), bytes));
    ptrs.push_back(*p);
    return DSX_OK;
  }
  void free_all() {
    for (void* p : ptrs) cudaFree(p);
    ptrs.clear();
  }
};

// grow-only device buffer: when `need` bytes do not fit, waits for the queued work on s that may still read it, frees
// it and allocates need + need / 8
struct GrowBuffer {
  void* ptr = nullptr;
  size_t cap = 0;
  int reserve(size_t need, cudaStream_t s) {
    if (cap >= need) return DSX_OK;
    if (ptr) {
      DSX_CUDA(cudaStreamSynchronize(s));
      cudaFree(ptr);
    }
    ptr = nullptr;
    cap = 0;
    DSX_TRY(checked_malloc(&ptr, need + need / 8));
    cap = need + need / 8;
    return DSX_OK;
  }
  // reserve that zero-fills a buffer it (re)allocated, on s
  int reserve_zeroed(size_t need, cudaStream_t s) {
    if (cap >= need) return DSX_OK;
    DSX_TRY(reserve(need, s));
    DSX_CUDA(cudaMemsetAsync(ptr, 0, cap, s));
    return DSX_OK;
  }
  void release() {
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    cap = 0;
  }
};

// a GrowBuffer that reads as a T*
template <typename T>
struct Buf : GrowBuffer {
  operator T*() const { return static_cast<T*>(ptr); }
};

inline size_t align256(size_t bytes) { return (bytes + 255) & ~size_t(255); }

// hands out consecutive 256-byte-aligned pieces of a buffer of at least the sum of their align256 sizes
struct Bump {
  uint8_t* p;
  template <typename T>
  T* take(size_t bytes) {
    T* q = reinterpret_cast<T*>(p);
    p += align256(bytes);
    return q;
  }
};

// makes `device` current after checking that it exists; its properties to *prop
inline int select_device(int device, cudaDeviceProp* prop) {
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    set_error("no CUDA device available (%s); dsx has no CPU fallback", cudaGetErrorString(e));
    return DSX_E_CUDA;
  }
  DSX_CHECK(device >= 0 && device < ndev, DSX_E_INVALID, "device %d out of range (%d devices)", device, ndev);
  DSX_CUDA(cudaGetDeviceProperties(prop, device));
  DSX_CUDA(cudaSetDevice(device));
  return DSX_OK;
}

// select_device for the kernels of `what`, whose only target is sm_90
inline int select_sm90_device(int device, const char* what) {
  cudaDeviceProp prop;
  DSX_TRY(select_device(device, &prop));
  DSX_CHECK(prop.major == 9 && prop.minor == 0, DSX_E_CUDA, "the %s's kernels are built for sm_90a; device %d is sm_%d%d",
            what, device, prop.major, prop.minor);
  return DSX_OK;
}

constexpr int kTile = 128;  // frames per tile: the frame axis of every utterance is padded to a multiple of it

// Geometry of one call: B utterances of T frames, stored frames-major with the frame axis
// padded to a multiple of the tile so tiles never straddle utterances.
struct Geom {
  int B = 0, T = 0, Tp = 0, tiles_per_utt = 0, tiles = 0;
  void set(int b, int t) {
    B = b;
    T = t;
    tiles_per_utt = (t + kTile - 1) / kTile;
    Tp = tiles_per_utt * kTile;
    tiles = B * tiles_per_utt;
  }
  size_t frames_padded() const { return static_cast<size_t>(B) * Tp; }
};

// Device-side model description handed to kernels.
struct ModelDev {
  int M, C, H, L, cycle;
  // fp32, SIMT layouts
  const float* in_w;   // [C][M]
  const float* in_b;   // [C]
  const float* mlp0_w; // [4C][C]
  const float* mlp0_b;
  const float* mlp2_w; // [C][4C]
  const float* mlp2_b;
  const float* dif_w;  // [L][C][C]
  const float* dif_b;  // [L][C]
  const float* w1f;    // [L][2C][3C+H]   k = tap*C + c | 3C + h
  const float* b1f;    // [L][2C]         dil_b + cond_b
  const float* w2f;    // [L][2C][C]
  const float* b2f;    // [L][2C]
  const float* skip_w; // [C][C]
  const float* skip_b;
  const float* fin_w;  // [M][C]
  const float* fin_b;
  // tensor-core packs (fp16, 128-byte rows of 64 k-values, each row in its 128-byte-swizzled order; see dsx_hopper.cu
  // for the tile order)
  const __half* wpack; // [L][20480 rows][64]
  const float* b1p;    // [L][2 chunks][256]  gate(128) | filter(128) per chunk
  const __half* whead; // [32 tiles][128 rows][64]: skip_projection, output_projection, input_projection packs
  const __half* wsr;   // [R][L][8192 rows][64] stochastically rounded weight sets (DSX_PREC_FP16S), or nullptr
  int wsr_sets;        // R
};

// Grow-only buffers of the sampler, each its own allocation: growth of one leaves the others, and what they hold, in place
struct Workspace {
  Geom g;               // geometry (B, T) of the last call
  int rows_cap = 0;     // step-table rows
  Buf<float> X;         // [B][Tp][C] residual stream
  Buf<float> SKIP;      // [B][Tp][C]
  Buf<float> CONDF;     // [B][Tp][H] fp32 (SIMT path)
  Buf<float> G1;        // [B][Tp][simt_g1_cols] SIMT GEMM output scratch: a layer's 2C columns, or the head's M
  Buf<float> Zf;        // [B][Tp][C]  SIMT gate output
  Buf<__half> Y;        // [2 buffers][2 planes][B][Tp][C]
  Buf<__half> CONDH;    // [2 planes][B][Tp][H]
  Buf<float> CP;        // [L][B][Tp][512] conditioner projection + bias of every layer (tensor-core path)
  Buf<__half> S16;      // [2 planes][B][Tp][C] skip_sum / sqrt(L), operand of the head GEMM
  Buf<unsigned> FLAGS;  // [2][B * Tp / 64] per-tile progress flags of the step kernel (tensor-core path)
  Buf<float> DTAB;      // [rows][L][C]
  Buf<float> EMB;       // [rows][C] scratch (mlp output)
  Buf<int64_t> TVALS;   // [rows]
  Buf<float> EPS;       // [5][B][M][T] current + PLMS history ring
  Buf<float> XTMP;      // [B][M][T] PLMS warm-up state
  Buf<float> XSTATE;    // [B][M][T] mel state of dsx_infer
  // f(GrowBuffer&) on every buffer: the one list of them, behind bytes() and release()
  template <typename F>
  void each(F f) {
    f(X); f(SKIP); f(CONDF); f(G1); f(Zf); f(Y); f(CONDH); f(CP); f(S16); f(FLAGS); f(DTAB); f(EMB); f(TVALS); f(EPS);
    f(XTMP); f(XSTATE);
  }
  size_t bytes() {   // DSX_INFO_WORKSPACE_BYTES
    size_t n = 0;
    each([&](GrowBuffer& b) { n += b.cap; });
    return n;
  }
  void release() {
    each([](GrowBuffer& b) { b.release(); });
    g = Geom();
    rows_cap = 0;
  }
};

struct FftDenoiser;   // dsx_fftdiff.cu

}  // namespace dsx

struct dsx_handle {
  int device = 0;
  int sm_count = 0;
  bool loaded = false;
  int precision = DSX_PREC_FP32_SIMT;
  int tc_group = 0;             // 2 when the tensor-core path (sm_90 wgmma kernels) is available on the device, else 0
  int layer_limit = -1;
  int64_t launches = 0;
  int64_t stack_launches = 0;   // one-launch-per-step launches of k_hp_step (layers + fused head)
  dsx::ModelDev m{};
  dsx::DevAllocs mem;         // device allocations of the model
  int sched_T = 0;
  std::vector<float> sched[DSX_SCH_COUNT];
  dsx::Workspace ws;
  int* status_dev = nullptr;   // kernel watchdog / self-check word
  int* status_host = nullptr;  // pinned mirror
  int profile = 0;
  dsx::GrowBuffer stage[7];    // dsx_infer_host device staging
  int stack_kernel = 1;                // DSX_OPT_STACK_KERNEL: 1 = layers and head of a step in one launch where it applies
  int step_occ[3] = {};                // co-resident CTAs of k_hp_step<NWG, R> <1, 3> / <2, 3> / <2, 2> on the device (0 unknown, -1 none)
  int fused_head = 1;                  // DSX_OPT_FUSED_HEAD: the head / sampler update / next input projection run inside the stack launch
  int stack_rows = 0;                  // DSX_OPT_STACK_ROWS: 0 = automatic, 64 / 128 forced
  int stack_rows_used = 0;             // rows per CTA of the last stack launch
  int sr_sets = 64;                    // DSX_OPT_SR_SETS: weight sets of DSX_PREC_FP16S (takes effect at the next dsx_load_diffnet)
  unsigned long long sr_seed = 0x5DEECE66Dull;
  bool cond_ready = false;             // CONDH / CP (or CONDF) hold the conditioner of dsx_set_cond for geometry cond_geom
  dsx::Geom cond_geom;
  int gate_approx = -1;                // DSX_OPT_GATE_APPROX: -1 = default (tanh.approx gate), 0 / 1 forced
  int batch_offset = 0;                // DSX_OPT_BATCH_OFFSET: global index of utterance 0 in the Philox noise counters
  bool attr_cond = false;
  int stack_mode = 1;               // 1: all residual layers of an evaluation in one launch
  std::vector<cudaEvent_t> prof_events;   // pairs (start, stop), prof_used of them recorded
  size_t prof_used = 0;
  int64_t* trace_dev = nullptr;     // dsx_debug_trace: [2 * sm_count][DSX_TRACE_SLOTS] phase stamps of the step kernel
  bool trace_on = false;
  dsx::FftDenoiser* fft = nullptr;  // dsx_load_fft: the denoiser is the FFT (m holds only M and H), else DiffNet
};

namespace dsx {

// launch_check of a launch (or the last of n) that DSX_INFO_KERNEL_LAUNCHES counts
inline int counted_launch(dsx_handle* h, const char* what, int n = 1) {
  h->launches += n;
  return launch_check(what);
}

// ---- dsx_simt.cu -------------------------------------------------------------------------
// Largest M and C of the fp32 path: k_inproj stages 16 frames x M and k_embed_table 5 C floats in the default 48 KB of
// dynamic shared memory (dsx_load_diffnet refuses larger models)
constexpr int kSimtMaxM = 768;
constexpr int kSimtMaxC = 2448;
// row stride of ws.G1: each layer's gate / filter and residual / skip GEMMs write 2C columns, the head's output projection M
inline int simt_g1_cols(const ModelDev& m) { return m.M > 2 * m.C ? m.M : 2 * m.C; }
int simt_pack_model(dsx_handle* h, const dsx_diffnet_params* p, cudaStream_t s);
int launch_embed_table(dsx_handle* h, const int64_t* t_dev, int rows, cudaStream_t s);
// emb[row] = mlp(SinusoidalPosEmb(m.C)(t[row])) for `rows` rows (m: C and the mlp weights)
int launch_embed_mlp(dsx_handle* h, const ModelDev& m, const int64_t* t_dev, int rows, float* emb, cudaStream_t s);
// the same, also saving each row's sinusoid, mlp.0 output and its Mish to save [rows][9 C] (the training step's tape)
int launch_embed_saved(const ModelDev& m, const int64_t* t_dev, int rows, float* emb, float* save, cudaStream_t s);
int launch_pack_cond(dsx_handle* h, const float* cond, dsx_strides cs, const Geom& g, cudaStream_t s);
int launch_inproj(dsx_handle* h, const float* x, dsx_strides xs, const Geom& g, int row0, int row_per_b,
                  cudaStream_t s);
int launch_simt_layer(dsx_handle* h, int layer, const Geom& g, int row0, int row_per_b, cudaStream_t s);
int launch_head(dsx_handle* h, const Geom& g, float* eps, cudaStream_t s);
struct DdpmCoef { float A, Bc, c1, c2, sigma; };
int launch_ddpm_update(dsx_handle* h, float* x, const float* eps, const float* noise, uint64_t seed,
                       uint64_t offset, DdpmCoef c, size_t n, int T, cudaStream_t s);
struct PlmsCoef { float kx, ke, a_diff, denom, w0, w1, w2, w3; };   // see k_plms_update
int launch_plms_update(dsx_handle* h, float* x_out, const float* x_in, const float* e0, const float* e1,
                       const float* e2, const float* e3, PlmsCoef c, size_t n, cudaStream_t s);
int launch_prologue(dsx_handle* h, float* x, const float* fs2_mel, const float* start_noise, uint64_t seed,
                    const float* spec_min, const float* spec_max, float sa, float s1a, int B, int T, int M,
                    cudaStream_t s);
int launch_epilogue(dsx_handle* h, const float* x, const int64_t* mel2ph, const float* spec_min,
                    const float* spec_max, float* mel_out, int B, int T, int M, cudaStream_t s);

// ---- dsx_hopper.cu -----------------------------------------------------------------------
int tc_pack_model(dsx_handle* h, cudaStream_t s);
int launch_tc_condproj(dsx_handle* h, const Geom& g, cudaStream_t s);
// Head / tail of DiffNet on tensor cores.  flags: 1 = head (skip -> eps), 2 = write eps, 4 = DDPM update of x,
// 8 = input projection of x (after the update if any) for the evaluation that uses table row (next_row0, row_per_b).
enum { TC_HEAD = 1, TC_WRITE_EPS = 2, TC_UPDATE = 4, TC_INPROJ = 8, TC_PLMS = 16 };
// PNDM update fused into the head kernel (TC_PLMS): eps' = (w0 eps_t + w1 h1 + w2 h2 + w3 h3) / denom, x_out = phi(x, eps', t)
// (usr/diff/shallow_diffusion_tts.py:174-199); eps_t is also stored to `eps_store` (history ring) when non-null.
struct PlmsFuse {
  PlmsCoef c;
  const float* h1;
  const float* h2;
  const float* h3;   // earlier eps, most recent first, contiguous [B][M][T] (or null)
  float* eps_store;  // this evaluation's eps -> history ring slot (or null)
  float* x_out;      // result; null: in place
};
bool tc_supported(const dsx_handle* h);

// What follows the residual stack of an evaluation: eps, a sampler update and the next evaluation's input projection
struct HeadArgs {
  int flags = 0;            // TC_* (0: no head)
  float* x = nullptr;       // mel state
  dsx_strides xs{};
  float* eps = nullptr;     // TC_WRITE_EPS
  const float* noise = nullptr;
  uint64_t seed = 0, offset = 0;
  DdpmCoef c{};
  int next_row0 = 0, row_per_b = 0;   // FiLM table row of the NEXT evaluation (TC_INPROJ)
  const PlmsFuse* plms = nullptr;
};
// Whether the head of an evaluation of all layers runs inside the layers' launch: the stack form with DSX_OPT_FUSED_HEAD,
// except under DSX_OPT_PROFILE = 2, which times the head as a launch of its own.
bool tc_fuse_head(const dsx_handle* h);
// k_hp_step for layers [l0, l1) of the evaluation at FiLM table row (row0, row_per_b), followed in the same launch by
// `head` (only with all layers where tc_fuse_head allows it); with no layers, `head` alone at 128 rows.
int launch_tc_step(dsx_handle* h, const Geom& g, int l0, int l1, int row0, int row_per_b, const HeadArgs* head,
                   cudaStream_t s);

int ensure_workspace(dsx_handle* h, const Geom& g, int rows, cudaStream_t s);
int check_status(dsx_handle* h, cudaStream_t s, const char* what);

// ---- dsx_fs2dec.cu: the FFTBlocks stack of a loaded decoder handle, shared by the FastSpeech2 decoder and the FFT
// denoiser ----------------------------------------------------------------------------------------------------------
struct Fs2Bufs {
  float* X;          // [B][T][H] fp32 residual stream: the stack's input on entry
  __half *A, *O, *Q, *K, *F, *VT;
  uint8_t* PAD;      // [B][T] padding flags, set on entry
  int* POS;
};
size_t fs2_workspace_bytes(const dsx_fs2dec* h, int B, int T);
Fs2Bufs fs2_carve(const dsx_fs2dec* h, void* ws, int B, int T);   // ws: fs2_workspace_bytes(h, B, T) bytes
// the decoder's entry -- positions over channel 0, X = (X + alpha * table[pos]) * !pad and LN1 of layer 0 -> A -- then
// fs2_layers_run.  2 + 5 L launches.
// What the training step's forward (dsx_fs2train.cu) saves, and its dropout: site 0 at the entry, then per layer i sites
// 1 + 3 i (after out_proj), 2 + 3 i (after the FFN activation) and 3 + 3 i (after ffn_2).  Every pointer is a tape region.
struct Fs2Train {
  uint64_t seed = 0;
  float p = 0.f;
  std::vector<float*> xin;                          // LayerNorm inputs [F][H]: LN1 of layer i at 2 i, LN2 at 2 i + 1,
                                                    // the final LayerNorm at 2 L
  std::vector<__half*> a1, a2, q, k, v, o, z, hd;   // per layer: LN1 and LN2 outputs [F][H]; Q (scaled), K, V
                                                    // [B][heads][T][D]; attention output [F][H]; ffn_1 output * k^-0.5
                                                    // before the activation and the ffn_2 input after dropout [F][4H]
  std::vector<float*> lse;                          // per layer: softmax log-sum-exp [B][heads][T] (+inf: no key)
  Fs2Drop drop(int site) const { return make_drop(seed, p, site); }
};
// the first region of a dsx_fs2dec_train tape: the forward's dropout, so that the backward draws the same masks from the
// tape alone, and its (B, T), which the backward checks on the device
struct Fs2TapeHdr {
  uint64_t seed;
  float p;
  int B, T;
};
int fs2_stack_run(const dsx_fs2dec* h, const Fs2Bufs& w, int B, int T, float* out, __half* out16, cudaStream_t s,
                  const Fs2Train* tr = nullptr);
// k_fs2_pack of x (any strides) into w.X and w.PAD, then fs2_stack_run
int fs2_forward_run(const dsx_fs2dec* h, const float* x, dsx_strides xs, int B, int T, const Fs2Bufs& w, float* out,
                    cudaStream_t s, const Fs2Train* tr = nullptr);
// The training step's packs: fs2_train_alloc sizes and allocates them once; fs2_train_pack refills them from the
// caller's fp32 weights on the stream (no allocation, no synchronisation) and points the LayerNorm affines and
// pos_embed_alpha at the caller's arrays.
int fs2_train_alloc(dsx_fs2dec* h);
int fs2_train_pack(dsx_fs2dec* h, const dsx_fs2dec_params* p, cudaStream_t s);
const dsx_fs2dec_config& fs2_config(const dsx_fs2dec* h);
// the L layers from X (masked), PAD and A = LN1 of layer 0 (fp16), then the final LayerNorm * !pad: to out [B][T][H] fp32,
// or (out == NULL) to out16 as fp16.  5 L launches.
int fs2_layers_run(const dsx_fs2dec* h, const Fs2Bufs& w, int B, int T, float* out, __half* out16, cudaStream_t s,
                   const Fs2Train* tr = nullptr);
int fs2_layers(const dsx_fs2dec* h);
void fs2_first_ln(const dsx_fs2dec* h, const float** w, const float** b);   // layer 0's layer_norm1 (device)
// dsx_fs2dec_load with pos_embed_alpha optional (the encoder's FFTBlocks have none)
int fs2_load(dsx_fs2dec* h, const dsx_fs2dec_params* p, void* stream);

// ---- dsx_fs2enc.cu: the encoder's entry, shared by the eval forward and the encoder training step ----------------------
// Positions (pos_mode 0, to w.POS), then x = sqrt(H) E[tok] + the addends + the position term, * dropout(drop) (site < 0:
// none), * !pad -> w.X, w.PAD, xsave (or NULL) and layer 0's layer_norm1 of the stack -> A (fp16).  2 launches, 1 for
// pos_mode 1.
int fs2enc_entry(const dsx_fs2dec* stack, int pos_mode, const float* E, int vocab, const int64_t* tokens, int B, int T,
                 const float* const* add, const dsx_strides* as, int rel_len, const Fs2Bufs& w, __half* A,
                 const Fs2Drop& drop, float* xsave, cudaStream_t s);

// ---- dsx_fs2train.cu: the decoder training step's stack, which the encoder training step (dsx_fs2enctrain.cu) also
// drives -----------------------------------------------------------------------------------------------------------------
// the regions of a dsx_fs2dec_train tape
struct Fs2TrainTape {
  Fs2TapeHdr* hdr;
  uint8_t* pad;                // [F] padding flags
  int* pos;                    // [F] positions of the decoder's entry (unused by the encoder step)
  Fs2Train tr;
};
dsx_fs2dec* fs2t_stack(dsx_fs2dec_train* h);   // the forward's packs and kernels
// dsx_fs2dec_train_tape_bytes for a (B, T) the caller has checked; with base, the regions of the tape at base to *t
size_t fs2t_tape_carve(const dsx_fs2dec_train* h, int B, int T, void* base, Fs2TrainTape* t);
// DSX_E_INVALID when a pointer of p is NULL (pos_embed_alpha only when alpha)
int fs2t_check_params(const dsx_fs2dec_params* p, int L, int alpha, const char* what);
// the training forward's steps before the stack's entry: packs w (forward and transposed backward packs), carves the tape
// to *tp and writes its header (seed, p, B, T).  No allocation, no synchronisation.
int fs2t_begin(dsx_fs2dec_train* h, const dsx_fs2dec_params* w, int B, int T, float p_drop, uint64_t seed, void* tape,
               cudaStream_t s, Fs2TrainTape* tp);
// The backward of dsx_fs2dec_train_backward from d_out through the final LayerNorm and the L layers, with the tape's PAD
// as the forward wrote it: every stack gradient through grads (pos_embed_alpha not read), d_x = the gradient at the entry's
// dropout input, * !pad, * dropout(0) (or NULL), and d_alpha = sum d_x . table[pos] over the tape's positions (or NULL:
// not computed).  workspace: dsx_fs2dec_train_workspace_bytes(B, T); B and T checked by the caller.
int fs2t_backward(dsx_fs2dec_train* h, const dsx_fs2dec_params* w, const void* tape, const float* d_out,
                  const dsx_fs2dec_params* grads, float* d_x, float* d_alpha, int B, int T, void* workspace,
                  cudaStream_t s);

// ---- dsx_pe.cu: the duration predictor's layers, shared by its eval forward and its training step (dsx_durtrain.cu) ---
// What the training forward saves, every pointer a tape region: layer i's fp16 input operand a[i] ([F][idim] for i = 0,
// else [F][chans]; a[0] is the packed x), its LayerNorm input r[i] (conv + bias, ReLU; fp32 [F][chans]) and the head's
// input hin (the last layer's output after dropout and * !mask, fp32 [F][chans]).  Dropout site i is layer i's.
struct DurTrain {
  uint64_t seed = 0;
  float p = 0.f;
  std::vector<__half*> a;
  std::vector<float*> r;
  float* hin = nullptr;
  Fs2Drop drop(int site) const { return make_drop(seed, p, site); }
};
// The training step's forward packs live in a dsx_durpred handle: durpred_train_alloc sizes them once (the handle then
// counts as loaded), durpred_train_pack refills them from the caller's fp32 weights on the stream (no allocation, no
// synchronisation) and points the LayerNorm affines at the caller's arrays; head = false leaves out the duration head's
// weights (the pitch predictor's stack has a head of its own).
int durpred_train_alloc(dsx_durpred* h);
int durpred_train_pack(dsx_durpred* h, const dsx_durpred_params* p, cudaStream_t s, bool head = true);
// x (any strides) -> tr.a[0], then the layers in training form (k_pe_conv<NT, true>): xs [B][T], 0 on padding.
// 1 + n_layers launches.
int durpred_train_run(const dsx_durpred* h, const float* x, dsx_strides xs_, const uint8_t* mask, int B, int T,
                      const DurTrain& tr, float* xs, cudaStream_t s);
// DurationPredictor._forward's layers from layer 0's fp16 operand: eval (tr == NULL) from A[0], alternating A[0] and A[1];
// training (tr) from tr->a[0], as durpred_train_run.  With a mask, the duration head follows -> xs, dur (see
// dsx_durpred_forward).  mask == NULL is the pitch predictor's stack (tts_modules.py:222-235, dsx_pitchtrain.cu): nothing
// is masked, and the last layer's output after dropout goes to hin [F][chans] fp32 instead of a head.  n_layers launches.
int dp_stack_run(const dsx_durpred* h, __half* const* A, const uint8_t* mask, int B, int T, float* xs, int64_t* dur,
                 const DurTrain* tr, float* hin, cudaStream_t s);

// ---- dsx_durtrain.cu: the duration predictor step's backward, shared with the pitch predictor step (dsx_pitchtrain.cu)
// the regions of a training tape the backward reads
struct DurTape {
  Fs2TapeHdr* hdr;
  uint8_t* pad;                // [F] the forward's mask, or NULL: no mask
  DurTrain tr;
};
dsx_durpred* dpt_forward_handle(dsx_durpred_train* h);   // the forward's packs and kernels
// workspace bytes of dpt_backward over (B, T) with a head of od outputs (1..16)
size_t dpt_workspace_bytes(const dsx_durpred_train* h, int B, int T, int od);
// The backward from d_out [F][od] (unscaled) through a head Linear(chans, od) (* !mask when tp.pad) and the layers:
// every gradient through grads (linear_w [od][chans], linear_b [od]) and d_x [F][idim] (or NULL), all written.  S is
// the power of two from amax |d_out * !mask| over every column.  B, T and the pointers are checked by the caller.
// 4 + 4 L launches for k <= 4; no allocation, no synchronisation.
int dpt_backward(dsx_durpred_train* h, const dsx_durpred_params* w, const DurTape& tp, const float* d_out, int od,
                 const dsx_durpred_params* grads, float* d_x, int B, int T, void* workspace, cudaStream_t s);

// ---- dsx_fftdiff.cu: the FFT denoiser of the sampler handle ---------------------------------------------------------
int fft_create(int device, const dsx_fft_config* c, const dsx_fft_params* p, cudaStream_t s, FftDenoiser** out);
void fft_destroy(FftDenoiser* f);
// per-(B, T) buffers and `rows` step-table rows; a moved cond-part buffer clears h->cond_ready
int fft_workspace(dsx_handle* h, const Geom& g, int rows, cudaStream_t s);
int fft_set_cond(dsx_handle* h, const float* cond, dsx_strides cs, const Geom& g, cudaStream_t s);
int fft_embed_table(dsx_handle* h, const int64_t* t_dev, int rows, cudaStream_t s);
// eps (contiguous [B,1,M,T]) of x (any strides), utterance b at table row row0 + b * row_per_b
int fft_eval(dsx_handle* h, const float* x, dsx_strides xs, const Geom& g, int row0, int row_per_b, float* eps,
             cudaStream_t s);

}  // namespace dsx
