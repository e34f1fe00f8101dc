// FFT denoiser training step on sm_90a: FFT.forward (usr/diff/candidate_decoder.py:50-100) in training mode, as
// GaussianDiffusion.p_losses calls it with diff_decoder_type 'fft', with what the backward needs saved to a caller-owned
// tape, and the exact backward to every parameter and to cond.  dim = residual_channels, H = hidden, M = 80 mel bins,
// F = B T frames.
//
// The FFTBlocks stack is a dsx_fs2dec_train handle (dsx_fs2train.cu), driven through its C entries on regions carved from
// this step's tape and workspace; its tape comes first, so the tape starts with its header (seed, p, B, T).  Around it:
//
// Forward (the eval entry and exit of dsx_fftdiff.cu, from dsx_fftentry.cuh, with this step's weights packed every call):
//   k_fft_fold, k_fft_split_w, k_pack_conv   W' = Wd[:, :dim] W_in and b' (double), the (hi, hi, lo) weights, packs
//   k_embed_table                            mlp(emb(t)) per utterance, saving sinusoid, mlp.0 output and Mish (tape)
//   k_fft_tproj                              TTAB[b] = Wd[:, dim + H:] . mlp(emb(t_b))
//   k_fft_split, k_fft_in                    cond and x_t as (hi, lo, hi) fp16 planes (tape); CONDPART, then
//                                            decoder_inp = W' x_t + b' + CONDPART + TTAB[b]
//   dsx_fs2dec_train_forward                 the stack with dropout -> out fp32 [F][H]
//   k_fftt_half, k_fft_out                   out as fp16 (tape), eps = get_mel_out(out) [B][1][M][T]
//
// Backward, with S1 a power of two from amax |d_eps| and S2 one from amax |d| (d = d decoder_inp):
//   k_fftt_eps16        S1 d_eps -> fp16 [F][M]
//   k_fftt_gemm         d_out = d_eps . W_mel (fp32 [F][H], the stack's d_out)
//   run_wgrad           dW_mel = d_eps^T out16 and db_mel
//   dsx_fs2dec_train_backward   every stack gradient and d = d decoder_inp (fp32 [F][H])
//   k_fftt_half         S2 d -> fp16 [F][H]
//   run_wgrad           [G_spec | G_cond] = d^T [x_t | cond] (hi planes) with db_d = sum_f d; G_cond is dWd[:, dim:dim+H]
//   k_fftt_colsum/usum  u_b = sum_t d[b, t] (fixed order)
//   k_fftt_dwd          dWd[:, :dim] = G_spec W_in^T + db_d b_in^T, dWd[:, dim+H:] = sum_b u_b temb_b^T
//   k_fftt_dwin         dW_in = Wd[:, :dim]^T G_spec, db_in = Wd[:, :dim]^T db_d (the fold's transpose)
//   k_fftt_dtemb        d temb_b = Wd[:, dim+H:]^T u_b, then run_mlp_grad (dsx_wgrad.cuh)
//   k_fftt_gemm         d_cond = d . Wd[:, dim:dim+H] (frames-major), when asked for
// input_projection's output is never stored: its gradients come from G_spec = d^T x_t through the fold's transpose.
// Every gradient written is a scaled fp32 sum multiplied by 1 / S, so 2^k d_eps gives exactly 2^k times the gradients;
// no atomics touch a result, so two backwards of one tape are bitwise equal.
#include <math.h>

#include <algorithm>

#include "dsx_fftentry.cuh"
#include "dsx_wgrad.cuh"

namespace dsx {
namespace {

constexpr int kMel = 80;
constexpr int kSumRows = 128;   // frames per partial of k_fftt_colsum

// o[i] = fp16(x[i] * S), S = scal[0] (scal null: 1)
__global__ void k_fftt_half(const float* __restrict__ x, size_t n, const float* scal, __half* __restrict__ o) {
  const float S = scal ? scal[0] : 1.f;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<size_t>(gridDim.x) * blockDim.x)
    o[i] = __float2half_rn(x[i] * S);
}

// d_eps [B][M][T] fp32 -> fp16 [B][T][M] scaled by S = scal[0]
__global__ void k_fftt_eps16(const float* __restrict__ e, const float* scal, int T, int M, __half* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float S = scal[0];
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (t < T && c < M) ? e[(static_cast<size_t>(b) * M + c) * T + t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < M) out[(static_cast<size_t>(b) * T + t) * M + c] = __float2half_rn(tile[threadIdx.x][i] * S);
  }
}

// out[f][col] = (A[f] . g column col) / S, fp32 [B][T][g.n]; one 64-row tile of utterance blockIdx.y, all n <= 256 columns
template <int NT>
__global__ void __launch_bounds__(128 * (NT > 128 ? 2 : 1)) k_fftt_gemm(const ConvGemm g, const __half* __restrict__ a,
                                                                        int T, const float* scal, float* __restrict__ out) {
  constexpr int WG = NT > 128 ? 2 : 1, NH = NT / WG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, b = blockIdx.y, m0 = blockIdx.x * kConvRows;
  float acc[NH / 2];
  conv_k_loop<NT, WG>(g, a, T, T, b, m0, 0, smem, acc);
  const float is = scal[1];
  const int n = g.n, c0 = wg * NH, r0 = acc_row(wtid, 0);
#pragma unroll
  for (int e = 0; e < NH / 2; e += 2) {
    const int col = c0 + acc_col(wtid, e), m = m0 + r0 + 8 * ((e >> 1) & 1);
    if (col >= n || m >= T) continue;
    *reinterpret_cast<float2*>(out + (static_cast<size_t>(b) * T + m) * n + col) = make_float2(acc[e] * is, acc[e + 1] * is);
  }
}

// part[b][chunk][h] = sum of d[b, t, h] over the chunk's kSumRows frames; block (chunk, b), thread h
__global__ void k_fftt_colsum(const float* __restrict__ d, int T, int H, float* __restrict__ part) {
  const int b = blockIdx.y, ch = blockIdx.x, h = threadIdx.x;
  const int t1 = min(T, (ch + 1) * kSumRows);
  float s = 0.f;
  for (int t = ch * kSumRows; t < t1; ++t) s += d[(static_cast<size_t>(b) * T + t) * H + h];
  part[(static_cast<size_t>(b) * gridDim.x + ch) * H + h] = s;
}

// u[b][h] = S * sum of the chunks' partials, in chunk order
__global__ void k_fftt_usum(const float* __restrict__ part, int B, int chunks, int H, const float* scal,
                            float* __restrict__ u) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * H) return;
  const int b = i / H, h = i - b * H;
  float s = 0.f;
  for (int ch = 0; ch < chunks; ++ch) s += part[(static_cast<size_t>(b) * chunks + ch) * H + h];
  u[i] = s * scal[0];
}

// block h: dWd[h][c] = (G_spec[h] . W_in[c] + db_d[h] b_in[c]) / S and dWd[h][dim + H + c] = (sum_b u[b][h] temb[b][c]) / S
__global__ void k_fftt_dwd(const float* __restrict__ gs, const float* __restrict__ dbd, const float* __restrict__ u,
                           const float* __restrict__ temb, int B, const float* __restrict__ win,
                           const float* __restrict__ bin, int dim, int H, int ldw, const float* scal,
                           float* __restrict__ dwd) {
  __shared__ float g[kMel];
  const int h = blockIdx.x;
  for (int m = threadIdx.x; m < kMel; m += blockDim.x) g[m] = gs[static_cast<size_t>(h) * kMel + m];
  __syncthreads();
  const float is = scal[1], db = dbd[h];
  for (int c = threadIdx.x; c < dim; c += blockDim.x) {
    float s = 0.f;
    for (int m = 0; m < kMel; ++m) s = fmaf(g[m], win[static_cast<size_t>(c) * kMel + m], s);
    s = fmaf(db, bin[c], s);
    dwd[static_cast<size_t>(h) * ldw + c] = s * is;
    float e = 0.f;
    for (int b = 0; b < B; ++b) e = fmaf(u[static_cast<size_t>(b) * H + h], temb[static_cast<size_t>(b) * dim + c], e);
    dwd[static_cast<size_t>(h) * ldw + dim + H + c] = e * is;
  }
}

// block c, thread m <= M: dW_in[c][m] = (sum_h Wd[h][c] G_spec[h][m]) / S, and (m == M) db_in[c] with db_d for G_spec
__global__ void k_fftt_dwin(const float* __restrict__ wd, int ldw, const float* __restrict__ gs,
                            const float* __restrict__ dbd, int H, const float* scal, float* __restrict__ dwin,
                            float* __restrict__ dbin) {
  const int c = blockIdx.x, m = threadIdx.x;
  if (m > kMel) return;
  float s = 0.f;
  for (int h = 0; h < H; ++h)
    s = fmaf(wd[static_cast<size_t>(h) * ldw + c], m == kMel ? dbd[h] : gs[static_cast<size_t>(h) * kMel + m], s);
  if (m == kMel) dbin[c] = s * scal[1];
  else dwin[static_cast<size_t>(c) * kMel + m] = s * scal[1];
}

// block b: de[b][k] = sum_h Wd[h][col0 + k] u[b][h] (scaled, as u)
__global__ void k_fftt_dtemb(const float* __restrict__ wd, int ldw, int col0, const float* __restrict__ u, int dim,
                             int H, float* __restrict__ de) {
  const int b = blockIdx.x;
  for (int k = threadIdx.x; k < dim; k += blockDim.x) {
    float s = 0.f;
    for (int h = 0; h < H; ++h) s = fmaf(wd[static_cast<size_t>(h) * ldw + col0 + k], u[static_cast<size_t>(b) * H + h], s);
    de[static_cast<size_t>(b) * dim + k] = s;
  }
}

int gemm_run(const ConvGemm& g, const __half* a, int B, int T, const float* scal, float* out, cudaStream_t s) {
  const dim3 grid((T + kConvRows - 1) / kConvRows, B, 1);
  return conv_dispatch<256>(g.nt, [&](auto c) {
    constexpr int NT = decltype(c)::value;
    k_fftt_gemm<NT><<<grid, 128 * (NT > 128 ? 2 : 1), conv_smem<NT>(), s>>>(g, a, T, scal, out);
    return launch_check("k_fftt_gemm");
  });
}

// W^T of columns [col0, col0 + n) of a row-major [K][ld] matrix, as g (g.cin = K, g.n = n): k_pack_conv's transposed
// form with one output per phase reads v[k * ld + col]
int pack_cols_t(const ConvGemm& g, const float* w, int ld, cudaStream_t s) {
  return conv_repack(g, PackArgs{w, nullptr, nullptr, g.cin, 1, 1, ld, 1, 1}, s);
}

int linear_alloc(DevAllocs& mem, ConvGemm& g, int cin, int n, int nt_max) {
  g.cin = cin;
  g.n = n;
  g.taps = 1;
  g.tap0 = 0;
  return conv_alloc(mem, g, nt_max);
}

}  // namespace
}  // namespace dsx

struct dsx_fft_train {
  int device = 0;
  dsx_fft_config cfg{};
  dsx_fs2dec_train* dec = nullptr;   // the FFTBlocks stack
  dsx::DevAllocs mem;
  dsx::ConvGemm in, cond, out;       // the forward's: entry (3M -> H), cond part (3H -> H), get_mel_out (H -> M)
  dsx::ConvGemm melt, condt;         // the backward's: W_mel^T (M -> H), Wd[:, dim:dim+H]^T (H -> H)
  float *wf = nullptr, *bf = nullptr, *w_in = nullptr, *w_cond = nullptr;   // fold scratch: W', b', (hi, hi, lo) weights
};

namespace dsx {
namespace {

struct Tape {
  Fs2TapeHdr* hdr;   // the stack tape's header
  void* dec;         // the stack's tape
  float* emb;        // [B][dim] mlp(emb(t))
  float* save;       // [B][9 dim] sinusoid, mlp.0 output, Mish of it
  __half* xs;        // [F][3M] x_t as (hi, lo, hi)
  __half* xc;        // [F][3H] cond as (hi, lo, hi)
  __half* out16;     // [F][H] the stack's output
};

struct Sizes {
  size_t dec_tape, dec_ws, tape, fwd_ws, bwd_ws, part;
};

int check_geom(const dsx_fft_train* h, int B, int T, Sizes* z) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_TRY(dsx_fs2dec_train_tape_bytes(h->dec, B, T, &z->dec_tape));   // checks B and T
  DSX_TRY(dsx_fs2dec_train_workspace_bytes(h->dec, B, T, &z->dec_ws));
  const size_t F = static_cast<size_t>(B) * T, H = h->cfg.dec.hidden, dim = h->cfg.residual_channels, M = kMel;
  z->tape = z->dec_tape + align256(4 * B * dim) + align256(36 * B * dim) + align256(6 * F * M) + align256(6 * F * H) +
            align256(2 * F * H);
  z->fwd_ws = 3 * align256(4 * F * H) + align256(F) + align256(4 * B * H) + z->dec_ws;
  // the two weight-gradient launches: dW_mel (M rows, 1 tile), [G_spec | G_cond]
  z->part = wgrad_part_floats(static_cast<int>(F), {{(kMel + 63) / 64, 1}, {static_cast<int>(H) / 64, 2}}, h->device);
  const size_t chunks = (T + kSumRows - 1) / kSumRows;
  z->bwd_ws = 256 + align256(2 * F * M) + 2 * align256(4 * F * H) + align256(2 * F * H) + align256(4 * z->part) +
              align256(4 * H * M) + align256(4 * H) + align256(4 * B * chunks * H) + align256(4 * B * H) +
              align256(4 * B * dim) + align256(16 * B * dim) + z->dec_ws;
  return DSX_OK;
}

Tape tape_carve(const dsx_fft_train* h, const Sizes& z, int B, int T, void* base) {
  const size_t F = static_cast<size_t>(B) * T, H = h->cfg.dec.hidden, dim = h->cfg.residual_channels, M = kMel;
  Bump bp{static_cast<uint8_t*>(base)};
  Tape t;
  t.dec = bp.take<uint8_t>(z.dec_tape);
  t.hdr = static_cast<Fs2TapeHdr*>(t.dec);
  t.emb = bp.take<float>(4 * B * dim);
  t.save = bp.take<float>(36 * B * dim);
  t.xs = bp.take<__half>(6 * F * M);
  t.xc = bp.take<__half>(6 * F * H);
  t.out16 = bp.take<__half>(2 * F * H);
  return t;
}

int check_own_params(const dsx_fft_params* p, const char* what) {
  DSX_CHECK(p, DSX_E_INVALID, "%s is NULL", what);
  DSX_CHECK(p->in_w && p->in_b && p->mlp0_w && p->mlp0_b && p->mlp2_w && p->mlp2_b && p->decode_inp_w &&
                p->decode_inp_b && p->mel_out_w && p->mel_out_b,
            DSX_E_INVALID, "an input_projection, mlp, get_decode_inp or get_mel_out pointer of %s is NULL", what);
  return DSX_OK;
}

unsigned blocks_for(size_t n) { return static_cast<unsigned>(std::min<size_t>((n + 255) / 256, 4096)); }

}  // namespace
}  // namespace dsx

using namespace dsx;

extern "C" {

int dsx_fft_train_create(int device, const dsx_fft_config* cfg, dsx_fft_train** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  *out = nullptr;
  DSX_CHECK(cfg, DSX_E_INVALID, "null config");
  DSX_CHECK(cfg->mel_bins == kMel, DSX_E_INVALID, "unsupported mel_bins %d: 80 (get_mel_out is Linear(hidden_size, 80))",
            cfg->mel_bins);
  DSX_CHECK(cfg->residual_channels >= 16 && cfg->residual_channels <= 1024 && cfg->residual_channels % 16 == 0,
            DSX_E_INVALID, "unsupported residual_channels %d: a multiple of 16 in [16, 1024]", cfg->residual_channels);
  dsx_fs2dec_train* dec = nullptr;
  DSX_TRY(dsx_fs2dec_train_create(device, &cfg->dec, &dec));   // validates the stack and selects the device
  dsx_fft_train* h = new dsx_fft_train();
  h->device = device;
  h->cfg = *cfg;
  h->dec = dec;
  const int rc = [&]() -> int {
    DSX_TRY(conv_opt_in<256>([](auto k) { return k_fft_in<decltype(k)::value>; }));
    DSX_TRY(conv_opt_in<256>([](auto k) { return k_fftt_gemm<decltype(k)::value>; }));
    DSX_CUDA(cudaFuncSetAttribute(k_fft_out, cudaFuncAttributeMaxDynamicSharedMemorySize, conv_smem<kOutNT>()));
    DSX_CUDA(cudaFuncSetAttribute(k_wgrad, cudaFuncAttributeMaxDynamicSharedMemorySize, kWgSmem));
    const int H = cfg->dec.hidden, M = kMel;
    DSX_TRY(h->mem.alloc(&h->wf, static_cast<size_t>(H) * M * sizeof(float)));
    DSX_TRY(h->mem.alloc(&h->bf, static_cast<size_t>(H) * sizeof(float)));
    DSX_TRY(h->mem.alloc(&h->w_in, static_cast<size_t>(H) * kSplit * M * sizeof(float)));
    DSX_TRY(h->mem.alloc(&h->w_cond, static_cast<size_t>(H) * kSplit * H * sizeof(float)));
    DSX_TRY(linear_alloc(h->mem, h->in, kSplit * M, H, 256));
    DSX_TRY(linear_alloc(h->mem, h->cond, kSplit * H, H, 256));
    DSX_TRY(linear_alloc(h->mem, h->out, H, M, kOutNT));
    DSX_TRY(linear_alloc(h->mem, h->melt, M, H, 256));
    DSX_TRY(linear_alloc(h->mem, h->condt, H, H, 256));
    DSX_CHECK(h->in.ntiles == 1 && h->cond.ntiles == 1 && h->out.ntiles == 1 && h->out.nt == kOutNT &&
                  h->melt.ntiles == 1 && h->condt.ntiles == 1,
              DSX_E_INVALID, "internal: unexpected FFT denoiser tiling");
    return DSX_OK;
  }();
  if (rc != DSX_OK) {
    dsx_fft_train_destroy(h);
    return rc;
  }
  *out = h;
  return DSX_OK;
}

void dsx_fft_train_destroy(dsx_fft_train* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  h->mem.free_all();
  dsx_fs2dec_train_destroy(h->dec);
  delete h;
}

int dsx_fft_train_tape_bytes(dsx_fft_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  Sizes z;
  DSX_TRY(check_geom(h, B, T, &z));
  *out = z.tape;
  return DSX_OK;
}

int dsx_fft_train_workspace_bytes(dsx_fft_train* h, int B, int T, size_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null handle or out");
  Sizes z;
  DSX_TRY(check_geom(h, B, T, &z));
  *out = std::max(z.fwd_ws, z.bwd_ws);
  return DSX_OK;
}

int dsx_fft_train_forward(dsx_fft_train* h, const dsx_fft_params* w, const float* spec, dsx_strides ss,
                          const int64_t* t, const float* cond, dsx_strides cs, int B, int T, float p_drop,
                          uint64_t seed, void* tape, size_t tape_bytes, void* workspace, size_t workspace_bytes,
                          float* eps, void* stream) {
  Sizes z;
  DSX_TRY(check_geom(h, B, T, &z));
  DSX_TRY(check_own_params(w, "the parameters"));
  DSX_CHECK(spec && t && cond && tape && workspace && eps, DSX_E_INVALID,
            "spec, t, cond, tape, workspace and eps must not be NULL");
  DSX_CHECK(tape_bytes >= z.tape, DSX_E_INVALID, "tape of %zu bytes is below the %zu this (B, T) needs", tape_bytes,
            z.tape);
  const size_t wneed = std::max(z.fwd_ws, z.bwd_ws);
  DSX_CHECK(workspace_bytes >= wneed, DSX_E_INVALID, "workspace of %zu bytes is below the %zu this (B, T) needs",
            workspace_bytes, wneed);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int H = h->cfg.dec.hidden, M = kMel, dim = h->cfg.residual_channels, ldw = dim + H + dim;
  const size_t F = static_cast<size_t>(B) * T;
  const Tape tp = tape_carve(h, z, B, T, tape);
  Bump bp{static_cast<uint8_t*>(workspace)};
  float* CP = bp.take<float>(4 * F * H);
  float* X = bp.take<float>(4 * F * H);
  float* OUT = bp.take<float>(4 * F * H);
  uint8_t* PAD = bp.take<uint8_t>(F);
  float* TTAB = bp.take<float>(4 * static_cast<size_t>(B) * H);
  void* DECWS = bp.take<uint8_t>(z.dec_ws);

  // this step's packs: the fold of input_projection into get_decode_inp, the entry, cond and exit GEMMs, and the
  // transposed packs of the backward
  k_fft_fold<<<H, 128, 0, s>>>(w->decode_inp_w, ldw, w->in_w, w->in_b, w->decode_inp_b, dim, M, h->wf, h->bf);
  DSX_TRY(launch_check("k_fft_fold"));
  k_fft_split_w<<<(H * M + 255) / 256, 256, 0, s>>>(h->wf, M, 0, M, H, h->w_in);
  DSX_TRY(launch_check("k_fft_split_w"));
  k_fft_split_w<<<(H * H + 255) / 256, 256, 0, s>>>(w->decode_inp_w, ldw, dim, H, H, h->w_cond);
  DSX_TRY(launch_check("k_fft_split_w"));
  DSX_TRY(conv_repack(h->in, PackArgs{h->w_in, nullptr, h->bf, kSplit * M, H, H, 1, 1, 0}, s));
  DSX_TRY(conv_repack(h->cond, PackArgs{h->w_cond, nullptr, nullptr, kSplit * H, H, H, 1, 1, 0}, s));
  DSX_TRY(conv_repack(h->out, PackArgs{w->mel_out_w, nullptr, w->mel_out_b, H, M, M, 1, 1, 0}, s));
  DSX_TRY(pack_cols_t(h->melt, w->mel_out_w, H, s));
  DSX_TRY(pack_cols_t(h->condt, w->decode_inp_w + dim, ldw, s));

  // the step embedding with its saves, and its part of get_decode_inp
  ModelDev e{};
  e.C = dim;
  e.mlp0_w = w->mlp0_w;
  e.mlp0_b = w->mlp0_b;
  e.mlp2_w = w->mlp2_w;
  e.mlp2_b = w->mlp2_b;
  DSX_TRY(launch_embed_saved(e, t, B, tp.emb, tp.save, s));
  k_fft_tproj<<<(B * H + 7) / 8, 256, 0, s>>>(tp.emb, w->decode_inp_w, ldw, dim + H, dim, H, B, TTAB);
  DSX_TRY(launch_check("k_fft_tproj"));

  // decoder_inp = W' x_t + b' + CONDPART + TTAB[b]
  k_fft_split<<<dim3((T + 31) / 32, (H + 31) / 32, B), dim3(32, 8), 0, s>>>(cond, cs, T, H, tp.xc);
  DSX_TRY(launch_check("k_fft_split"));
  FftInArgs a{};
  a.g = h->cond;
  a.a = tp.xc;
  a.T = T;
  a.out = CP;
  DSX_TRY(fft_in_run(a, B, s));
  k_fft_split<<<dim3((T + 31) / 32, (M + 31) / 32, B), dim3(32, 8), 0, s>>>(spec, ss, T, M, tp.xs);
  DSX_TRY(launch_check("k_fft_split"));
  a.g = h->in;
  a.a = tp.xs;
  a.out = X;
  a.cp = CP;
  a.ttab = TTAB;
  a.row0 = 0;
  a.row_per_b = 1;
  a.pad = PAD;
  DSX_TRY(fft_in_run(a, B, s));

  // the stack, then get_mel_out
  const dsx_strides xs{static_cast<int64_t>(T) * H, 1, H};
  DSX_TRY(dsx_fs2dec_train_forward(h->dec, &w->dec, X, xs, B, T, p_drop, seed, tp.dec, z.dec_tape, DECWS, z.dec_ws,
                                   OUT, stream));
  k_fftt_half<<<blocks_for(F * H), 256, 0, s>>>(OUT, F * H, nullptr, tp.out16);
  DSX_TRY(launch_check("k_fftt_half"));
  k_fft_out<<<dim3((T + kConvRows - 1) / kConvRows, B, 1), 128, conv_smem<kOutNT>(), s>>>(h->out, tp.out16, T, eps);
  return launch_check("k_fft_out");
}

int dsx_fft_train_backward(dsx_fft_train* h, const dsx_fft_params* w, const void* tape, const float* d_eps,
                           const dsx_fft_params* grads, float* d_cond, int B, int T, void* workspace,
                           size_t workspace_bytes, void* stream) {
  Sizes z;
  DSX_TRY(check_geom(h, B, T, &z));
  DSX_TRY(check_own_params(w, "the parameters"));
  DSX_TRY(check_own_params(grads, "the gradients"));
  DSX_CHECK(tape && d_eps && workspace, DSX_E_INVALID, "tape, d_eps and workspace must not be NULL");
  const size_t wneed = std::max(z.fwd_ws, z.bwd_ws);
  DSX_CHECK(workspace_bytes >= wneed, DSX_E_INVALID, "workspace of %zu bytes is below the %zu this (B, T) needs",
            workspace_bytes, wneed);
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int H = h->cfg.dec.hidden, M = kMel, dim = h->cfg.residual_channels, ldw = dim + H + dim;
  const int F = B * T, chunks = (T + kSumRows - 1) / kSumRows;
  const Tape tp = tape_carve(h, z, B, T, const_cast<void*>(tape));
  Bump bp{static_cast<uint8_t*>(workspace)};
  unsigned* amax = bp.take<unsigned>(256);   // [0], [1]: amax |d_eps|, amax |d|
  float* sc1 = reinterpret_cast<float*>(amax + 4);    // S1, 1 / S1
  float* sc2 = reinterpret_cast<float*>(amax + 8);    // S2, 1 / S2
  __half* E16 = bp.take<__half>(2 * static_cast<size_t>(F) * M);
  float* DOUT = bp.take<float>(4 * static_cast<size_t>(F) * H);
  float* DX = bp.take<float>(4 * static_cast<size_t>(F) * H);
  __half* D16 = bp.take<__half>(2 * static_cast<size_t>(F) * H);
  float* PART = bp.take<float>(4 * z.part);
  float* GS = bp.take<float>(4 * static_cast<size_t>(H) * M);
  float* DBD = bp.take<float>(4 * static_cast<size_t>(H));
  float* UPART = bp.take<float>(4 * static_cast<size_t>(B) * chunks * H);
  float* U = bp.take<float>(4 * static_cast<size_t>(B) * H);
  float* DE = bp.take<float>(4 * static_cast<size_t>(B) * dim);
  float* DH = bp.take<float>(16 * static_cast<size_t>(B) * dim);
  void* DECWS = bp.take<uint8_t>(z.dec_ws);
  auto gp = [](const float* p) { return const_cast<float*>(p); };

  // sum_f A[f][m] B_j[f][c] over the frames for ntiles B tiles into o, scaled by sc
  auto wgrad = [&](const __half* A, int lda, int am, WgradArgs t, int ntiles, const WgradDst& o,
                   const float* sc) -> int {
    t.a = A;
    t.lda = lda;
    t.am = am;
    t.F = F;
    t.T = T;
    return run_wgrad(t, ntiles, o, PART, sc, h->device, s);
  };

  // get_mel_out: d_out = d_eps . W_mel for the stack, dW_mel, db_mel; S1 is NaN when the tape is of another (B, T)
  DSX_TRY(run_scale(d_eps, static_cast<size_t>(F) * M, amax, sc1, tp.hdr, B, T, s));
  k_fftt_eps16<<<dim3((T + 31) / 32, (M + 31) / 32, B), dim3(32, 8), 0, s>>>(d_eps, sc1, T, M, E16);
  DSX_TRY(launch_check("k_fftt_eps16"));
  DSX_TRY(gemm_run(h->melt, E16, B, T, sc1, DOUT, s));
  {
    WgradArgs t{};
    t.b[0] = tp.out16;
    t.ldb[0] = H;
    t.bn[0] = H;
    WgradDst o{};
    o.dst[0] = gp(grads->mel_out_w);
    o.ms[0] = H;
    o.cs[0] = 1;
    o.db = gp(grads->mel_out_b);
    DSX_TRY(wgrad(E16, M, M, t, 1, o, sc1));
  }

  // the stack: every FFTBlocks gradient and d = d decoder_inp
  DSX_TRY(dsx_fs2dec_train_backward(h->dec, &w->dec, tp.dec, DOUT, &grads->dec, DX, B, T, DECWS, z.dec_ws, stream));

  // get_decode_inp and input_projection: [G_spec | G_cond] = d^T [x_t | cond] with db_d
  DSX_TRY(run_scale(DX, static_cast<size_t>(F) * H, amax + 1, sc2, tp.hdr, B, T, s));
  k_fftt_half<<<blocks_for(static_cast<size_t>(F) * H), 256, 0, s>>>(DX, static_cast<size_t>(F) * H, sc2, D16);
  DSX_TRY(launch_check("k_fftt_half"));
  {
    WgradArgs t{};
    t.b[0] = tp.xs;   // the hi planes of the split operands
    t.ldb[0] = kSplit * M;
    t.bn[0] = M;
    t.b[1] = tp.xc;
    t.ldb[1] = kSplit * H;
    t.bn[1] = H;
    WgradDst o{};   // G_spec and db_d unscaled (k_fftt_dwd and k_fftt_dwin scale them), G_cond and db scaled
    o.dst[0] = GS;
    o.ms[0] = M;
    o.cs[0] = 1;
    o.raw[0] = 1;
    o.dst[1] = gp(grads->decode_inp_w) + dim;
    o.ms[1] = ldw;
    o.cs[1] = 1;
    o.db = DBD;
    o.db_raw = 1;
    o.db2 = gp(grads->decode_inp_b);
    DSX_TRY(wgrad(D16, H, H, t, 2, o, sc2));
  }
  // the step part: u_b = sum_t d[b, t]
  k_fftt_colsum<<<dim3(chunks, B), H, 0, s>>>(DX, T, H, UPART);
  DSX_TRY(launch_check("k_fftt_colsum"));
  k_fftt_usum<<<(B * H + 255) / 256, 256, 0, s>>>(UPART, B, chunks, H, sc2, U);
  DSX_TRY(launch_check("k_fftt_usum"));
  k_fftt_dwd<<<H, 256, 0, s>>>(GS, DBD, U, tp.emb, B, w->in_w, w->in_b, dim, H, ldw, sc2, gp(grads->decode_inp_w));
  DSX_TRY(launch_check("k_fftt_dwd"));
  k_fftt_dwin<<<dim, 96, 0, s>>>(w->decode_inp_w, ldw, GS, DBD, H, sc2, gp(grads->in_w), gp(grads->in_b));
  DSX_TRY(launch_check("k_fftt_dwin"));
  k_fftt_dtemb<<<B, 256, 0, s>>>(w->decode_inp_w, ldw, dim + H, U, dim, H, DE);
  DSX_TRY(launch_check("k_fftt_dtemb"));
  DSX_TRY(run_mlp_grad(DE, B, dim, tp.save, w->mlp2_w, sc2, gp(grads->mlp2_w), gp(grads->mlp2_b), DH,
                       gp(grads->mlp0_w), gp(grads->mlp0_b), s));
  if (d_cond) DSX_TRY(gemm_run(h->condt, D16, B, T, sc2, d_cond, s));
  return DSX_OK;
}

}  // extern "C"
