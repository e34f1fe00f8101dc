// FastSpeech2 encoder training step on sm_90a: FastspeechEncoder.forward / FastspeechMIDIEncoder.forward in training mode
// (modules/fastspeech/tts_modules.py:310-347, modules/diffsinger_midi/fs2.py:11-36), with what the backward needs saved
// to a caller-owned tape, and the exact backward to every encoder parameter, embed_tokens.weight included, and to the sum
// of the MIDI addends.  H = hidden, F = B T tokens, V = vocab.
//
// The FFTBlocks layers are a dsx_fs2dec_train handle (dsx_fs2train.cu) driven through its internal entries on this
// step's tape and workspace; its tape comes first, so the tape starts with its header (seed, p, B, T), and the tokens
// follow it.  Dropout is the decoder step's: site 0 at the entry, 1 + 3 i, 2 + 3 i, 3 + 3 i in layer i, keyed by
// (seed, site, frame, channel).
//
// Forward:
//   fs2t_begin        the stack's fp16 packs of this step's weights, its transposed backward packs, the tape header
//   tokens -> tape    one device copy
//   fs2enc_entry      the eval encoder's entry (dsx_fs2enc.cu) in its training form: positions, then x = sqrt(H) E[tok] +
//                     addends + the position term, * dropout(0), * !pad -> X, the tape's PAD and LayerNorm input xin[0],
//                     and layer 0's LN1 operand a1[0]
//   fs2_layers_run    the L layers with their training hooks and the final LayerNorm -> out fp32 [F][H]
//
// Backward:
//   fs2t_backward     every stack gradient and g = the gradient at the entry's dropout input (fp32 [F][H], * !pad,
//                     * dropout(0)); the decoder step's backward runs the same code
//   k_et_keys         key (token << 32 | frame) per frame; padding and out-of-range ids count as token 0
//   k_et_sort_block / k_et_sort_step   bitonic sort of the keys: stages up to 1024 keys in shared memory, longer strides
//                     one launch each.  The keys are distinct, so the order is the stable order of frames by token.
//   k_et_bounds       the run [start, end) of every token in the sorted keys
//   k_et_partial      per chunk of 64 sorted frames: d_add = g (sinusoidal) or sqrt(H) g (rel) of each frame, and the sum
//                     of sqrt(H) d_add over each run's piece in the chunk, in sorted order
//   k_et_rows         one CTA per embedding row: the sum of its run's piece sums in chunk order; rows without a frame and
//                     row 0 (padding_idx) get 0
// The embedding gradient costs O(F log^2 F) for the sort and O(F H + V H) for the sums, whatever the vocabulary; no atomics
// touch a result, so two backwards of one tape are bitwise equal.  Every gradient is the stack's fp32 g (already divided by
// its power-of-two scale) times constants, so 2^k d_out gives exactly 2^k times every gradient.
#include <math.h>

#include <algorithm>

#include "dsx_conv.cuh"
#include "dsx_internal.h"

namespace dsx {
namespace {

constexpr int kSortBlock = 1024;   // keys per CTA of k_et_sort_block
constexpr int kSegRows = 64;       // sorted frames per chunk of k_et_partial
using Key = unsigned long long;

__device__ __forceinline__ bool tape_other(const Fs2TapeHdr* h, int B, int T) { return h->B != B || h->T != T; }

__global__ void k_et_keys(const int64_t* tok, int F, int N, int vocab, Key* keys) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (i < F) {
    const int64_t id = tok[i];
    const Key v = (id > 0 && id < vocab) ? static_cast<Key>(id) : 0ull;
    keys[i] = (v << 32) | static_cast<Key>(i);
  } else {
    keys[i] = ~0ull;
  }
}

// the pair (i, i + j) of compare-exchange t at stride j (a power of two), ascending where (global i) & k == 0
__device__ __forceinline__ void bitonic_cx(Key* a, int t, int j, int k, int base) {
  const int i = 2 * t - (t & (j - 1)), l = i + j;
  const bool up = ((base + i) & k) == 0;
  const Key x = a[i], y = a[l];
  if ((x > y) == up) {
    a[i] = y;
    a[l] = x;
  }
}

// one CTA per min(N, kSortBlock) keys in shared memory: every stage up to that size (k == 0), or the strides below
// kSortBlock of stage k
__global__ void __launch_bounds__(kSortBlock / 2) k_et_sort_block(Key* keys, int N, int k) {
  __shared__ Key sh[kSortBlock];
  const int n = min(N, kSortBlock), base = blockIdx.x * kSortBlock;
  for (int i = threadIdx.x; i < n; i += blockDim.x) sh[i] = keys[base + i];
  __syncthreads();
  auto steps = [&](int kk, int j0) {
    for (int j = j0; j > 0; j >>= 1) {
      for (int t = threadIdx.x; t < n / 2; t += blockDim.x) bitonic_cx(sh, t, j, kk, base);
      __syncthreads();
    }
  };
  if (k == 0) {
    for (int kk = 2; kk <= n; kk <<= 1) steps(kk, kk >> 1);
  } else {
    steps(k, kSortBlock >> 1);
  }
  for (int i = threadIdx.x; i < n; i += blockDim.x) keys[base + i] = sh[i];
}

__global__ void k_et_sort_step(Key* keys, int N, int k, int j) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < N / 2) bitonic_cx(keys, t, j, k, 0);
}

// start[v], end[v] of token v's run in the sorted keys (both zeroed before: an empty run)
__global__ void k_et_bounds(const Key* keys, int F, int* start, int* end) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= F) return;
  const Key v = keys[i] >> 32;
  if (i == 0 || (keys[i - 1] >> 32) != v) start[v] = i;
  if (i == F - 1 || (keys[i + 1] >> 32) != v) end[v] = i + 1;
}

// block: kSegRows sorted frames, thread: a channel.  d_add[f] = gscale g[f] (or NULL); part[i] = the sum in sorted order
// of escale d_add over the frames of i's run in this chunk, at the run's last frame i in the chunk
__global__ void k_et_partial(const Key* keys, int F, int H, const float* __restrict__ g, float gscale, float escale,
                             const Fs2TapeHdr* hdr, int B, int T, float* __restrict__ d_add, float* __restrict__ part) {
  const int c = threadIdx.x, i0 = blockIdx.x * kSegRows, i1 = min(F, i0 + kSegRows);
  const float bad = tape_other(hdr, B, T) ? __int_as_float(0x7fc00000) : 0.f;
  float s = 0.f;
  for (int i = i0; i < i1; ++i) {
    const Key key = keys[i];
    const size_t f = static_cast<size_t>(key & 0xffffffffull);
    const float a = gscale * g[f * H + c];
    if (d_add) d_add[f * H + c] = bad == 0.f ? a : bad;
    s += escale * a;
    if (i + 1 == i1 || (keys[i + 1] >> 32) != (key >> 32)) {
      part[static_cast<size_t>(i) * H + c] = s;
      s = 0.f;
    }
  }
}

// block v, thread a channel: dE[v] = the piece sums of token v's run in chunk order (0 without a run, and for row 0)
__global__ void k_et_rows(const int* start, const int* end, const float* __restrict__ part, int H,
                          const Fs2TapeHdr* hdr, int B, int T, float* __restrict__ dE) {
  const int v = blockIdx.x, c = threadIdx.x;
  float s = 0.f;
  if (v > 0) {
    const int e = end[v];
    for (int i = start[v]; i < e;) {
      const int stop = min(e, (i / kSegRows + 1) * kSegRows);
      s += part[static_cast<size_t>(stop - 1) * H + c];
      i = stop;
    }
  }
  dE[static_cast<size_t>(v) * H + c] = tape_other(hdr, B, T) ? __int_as_float(0x7fc00000) : s;
}

int sort_len(int F) {
  int n = 2;
  while (n < F) n <<= 1;
  return n;
}

}  // namespace
}  // namespace dsx

struct dsx_fs2enc_train {
  int device = 0;
  dsx_fs2enc_config cfg{};
  dsx_fs2dec_train* stack = nullptr;   // the FFTBlocks layers and final LayerNorm
};

namespace dsx {
namespace {

struct Sizes {
  size_t stack_tape, stack_ws, tape, ws;
};

int check_geom(const dsx_fs2enc_train* h, int B, int T, Sizes* z) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_TRY(dsx_fs2dec_train_tape_bytes(h->stack, B, T, &z->stack_tape));   // checks B and T
  DSX_TRY(dsx_fs2dec_train_workspace_bytes(h->stack, B, T, &z->stack_ws));
  const size_t F = static_cast<size_t>(B) * T, H = h->cfg.stack.hidden;
  z->tape = z->stack_tape + align256(8 * F);
  z->ws = z->stack_ws + 2 * align256(4 * F * H) + align256(8 * static_cast<size_t>(sort_len(static_cast<int>(F)))) +
          2 * align256(4 * static_cast<size_t>(h->cfg.vocab));
  return DSX_OK;
}

int check_params(const dsx_fs2enc_train* h, const dsx_fs2enc_params* p, const char* what) {
  DSX_CHECK(p, DSX_E_INVALID, "%s is NULL", what);
  DSX_CHECK(p->embed_w, DSX_E_INVALID, "embed_w of %s is NULL", what);
  return fs2t_check_params(&p->stack, h->cfg.stack.layers, 0, what);
}

}  // namespace
}  // namespace dsx

using namespace dsx;

extern "C" {

int dsx_fs2enc_train_create(int device, const dsx_fs2enc_config* cfg, dsx_fs2enc_train** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_CHECK(cfg, DSX_E_INVALID, "config is NULL");
  DSX_CHECK(cfg->vocab >= 1, DSX_E_INVALID, "unsupported vocab %d: at least 1 row of embed_tokens", cfg->vocab);
  DSX_CHECK(cfg->pos == 0 || cfg->pos == 1, DSX_E_INVALID, "unsupported pos %d: 0 (sinusoidal) or 1 (relative)",
            cfg->pos);
  dsx_fs2dec_train* stack = nullptr;
  DSX_TRY(dsx_fs2dec_train_create(device, &cfg->stack, &stack));   // validates the stack and selects the device
  dsx_fs2enc_train* h = new dsx_fs2enc_train();
  h->device = device;
  h->cfg = *cfg;
  h->stack = stack;
  *out = h;
  return DSX_OK;
}

void dsx_fs2enc_train_destroy(dsx_fs2enc_train* h) {
  if (!h) return;
  dsx_fs2dec_train_destroy(h->stack);   // synchronises the device
  delete h;
}

int dsx_fs2enc_train_tape_bytes(dsx_fs2enc_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  Sizes z;
  DSX_TRY(check_geom(h, B, T, &z));
  *out = z.tape;
  return DSX_OK;
}

int dsx_fs2enc_train_workspace_bytes(dsx_fs2enc_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  Sizes z;
  DSX_TRY(check_geom(h, B, T, &z));
  *out = z.ws;
  return DSX_OK;
}

int dsx_fs2enc_train_forward(dsx_fs2enc_train* h, const dsx_fs2enc_params* w, const int64_t* tokens, int B, int T,
                             const float* const* add, const dsx_strides* as, int rel_len, float p_drop, uint64_t seed,
                             void* tape, size_t tape_bytes, void* workspace, size_t workspace_bytes, float* out,
                             void* stream) {
  Sizes z;
  DSX_TRY(check_geom(h, B, T, &z));
  DSX_TRY(check_params(h, w, "the parameters"));
  DSX_CHECK(tokens && tape && workspace && out, DSX_E_INVALID, "tokens, tape, workspace and out must not be NULL");
  DSX_CHECK(p_drop >= 0.f && p_drop < 1.f, DSX_E_INVALID, "dropout p = %g is outside [0, 1)", static_cast<double>(p_drop));
  DSX_CHECK(h->cfg.pos == 0 || rel_len >= T, DSX_E_INVALID, "rel_len %d is shorter than T = %d", rel_len, T);
  DSX_CHECK(tape_bytes >= z.tape, DSX_E_INVALID, "tape of %zu bytes is below the %zu this (B, T) needs", tape_bytes,
            z.tape);
  DSX_CHECK(workspace_bytes >= z.ws, DSX_E_INVALID, "workspace of %zu bytes is below the %zu this (B, T) needs",
            workspace_bytes, z.ws);
  for (int k = 0; k < 3; ++k)
    DSX_CHECK(!add || !add[k] || as, DSX_E_INVALID, "addend %d has no strides", k);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t F = static_cast<size_t>(B) * T;
  Fs2TrainTape tp;
  DSX_TRY(fs2t_begin(h->stack, &w->stack, B, T, p_drop, seed, tape, s, &tp));
  int64_t* tok = reinterpret_cast<int64_t*>(static_cast<uint8_t*>(tape) + z.stack_tape);
  DSX_CUDA(cudaMemcpyAsync(tok, tokens, F * sizeof(int64_t), cudaMemcpyDeviceToDevice, s));
  const dsx_fs2dec* stack = fs2t_stack(h->stack);
  Fs2Bufs fb = fs2_carve(stack, workspace, B, T);
  fb.PAD = tp.pad;
  fb.POS = tp.pos;
  DSX_TRY(fs2enc_entry(stack, h->cfg.pos, w->embed_w, h->cfg.vocab, tok, B, T, add, as, rel_len, fb, tp.tr.a1[0],
                       tp.tr.drop(0), tp.tr.xin[0], s));
  return fs2_layers_run(stack, fb, B, T, out, nullptr, s, &tp.tr);
}

int dsx_fs2enc_train_backward(dsx_fs2enc_train* h, const dsx_fs2enc_params* w, const void* tape, const float* d_out,
                              const dsx_fs2enc_params* grads, float* d_add, int B, int T, void* workspace,
                              size_t workspace_bytes, void* stream) {
  Sizes z;
  DSX_TRY(check_geom(h, B, T, &z));
  DSX_TRY(check_params(h, w, "the parameters"));
  DSX_TRY(check_params(h, grads, "the gradients"));
  DSX_CHECK(tape && d_out && workspace, DSX_E_INVALID, "tape, d_out and workspace must not be NULL");
  DSX_CHECK(workspace_bytes >= z.ws, DSX_E_INVALID, "workspace of %zu bytes is below the %zu this (B, T) needs",
            workspace_bytes, z.ws);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int H = h->cfg.stack.hidden, V = h->cfg.vocab, F = B * T, N = sort_len(F);
  const Fs2TapeHdr* hdr = static_cast<const Fs2TapeHdr*>(tape);
  const int64_t* tok = reinterpret_cast<const int64_t*>(static_cast<const uint8_t*>(tape) + z.stack_tape);
  Bump bp{static_cast<uint8_t*>(workspace)};
  void* SWS = bp.take<uint8_t>(z.stack_ws);
  float* G = bp.take<float>(4 * static_cast<size_t>(F) * H);
  float* PART = bp.take<float>(4 * static_cast<size_t>(F) * H);
  Key* KEYS = bp.take<Key>(8 * static_cast<size_t>(N));
  int* START = bp.take<int>(4 * static_cast<size_t>(V));
  int* END = bp.take<int>(4 * static_cast<size_t>(V));

  // the layers, down to g at the entry
  DSX_TRY(fs2t_backward(h->stack, &w->stack, tape, d_out, &grads->stack, G, nullptr, B, T, SWS, s));

  // the frames in token order
  k_et_keys<<<(N + 255) / 256, 256, 0, s>>>(tok, F, N, V, KEYS);
  DSX_TRY(launch_check("k_et_keys"));
  k_et_sort_block<<<(N + kSortBlock - 1) / kSortBlock, std::min(N, kSortBlock) / 2, 0, s>>>(KEYS, N, 0);
  DSX_TRY(launch_check("k_et_sort_block"));
  for (int k = 2 * kSortBlock; k <= N; k <<= 1) {
    for (int j = k >> 1; j >= kSortBlock; j >>= 1) {
      k_et_sort_step<<<(N / 2 + 255) / 256, 256, 0, s>>>(KEYS, N, k, j);
      DSX_TRY(launch_check("k_et_sort_step"));
    }
    k_et_sort_block<<<N / kSortBlock, kSortBlock / 2, 0, s>>>(KEYS, N, k);
    DSX_TRY(launch_check("k_et_sort_block"));
  }
  DSX_CUDA(cudaMemsetAsync(START, 0, 4 * static_cast<size_t>(V), s));
  DSX_CUDA(cudaMemsetAsync(END, 0, 4 * static_cast<size_t>(V), s));
  k_et_bounds<<<(F + 255) / 256, 256, 0, s>>>(KEYS, F, START, END);
  DSX_TRY(launch_check("k_et_bounds"));

  // d_add and the embedding gradient: x = sqrt(H) E[tok] + addends, then + table[pos] (sinusoidal) or * sqrt(H) + pe
  // (rel), so d_add = g or sqrt(H) g and d E[v] = sqrt(H) sum of d_add over v's frames
  const float sh = static_cast<float>(sqrt(static_cast<double>(H)));
  k_et_partial<<<(F + kSegRows - 1) / kSegRows, H, 0, s>>>(KEYS, F, H, G, h->cfg.pos == 1 ? sh : 1.f, sh, hdr, B, T,
                                                           d_add, PART);
  DSX_TRY(launch_check("k_et_partial"));
  k_et_rows<<<V, H, 0, s>>>(START, END, PART, H, hdr, B, T, const_cast<float*>(grads->embed_w));
  return launch_check("k_et_rows");
}

}  // extern "C"
