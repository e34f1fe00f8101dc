// FFT denoiser of DiffSinger on sm_90a (usr/diff/candidate_decoder.py:35-100, DIFF_DECODERS['fft']) in eval mode:
//   eps = get_mel_out(FFTBlocks(get_decode_inp([input_projection(x_t), cond, mlp(emb(t))])))
// with dim = residual_channels, H = hidden_size, M = 80 mel bins.  get_decode_inp splits by its weight columns:
//   decoder_inp[b, t] = W' x_t[b, :, t] + b'  +  CONDPART[b, t]  +  TTAB[row(b)]
//   W' = Wd[:, 0:dim] . W_in, b' = Wd[:, 0:dim] . b_in + b_d   folded at load time in double (no activation between them)
//   CONDPART = Wd[:, dim:dim+H] . cond                          once per conditioner (dsx_set_cond / any call with cond)
//   TTAB[row] = Wd[:, dim+H:] . mlp(emb(t_row))                 once per step-table row, fp32
// The two GEMMs over the sampler's inputs (x_t: K = M, cond: K = H) run on the implicit-GEMM core of dsx_conv.cuh with
// hi+lo fp16 operands laid along K as A = (hi, lo, hi), B = (hi, hi, lo): three products in one fp32 accumulation, all
// but lo x lo, which is fp32-equivalent at 3x a K that is small.
//
// Per evaluation, 5 + 5 L launches (25 at L = 4), plus the sampler's update:
//   k_fft_split       x_t (any strides) -> fp16 (hi, lo, hi) [B][T][3M]
//   k_fft_in          X = acc + b' + CONDPART + TTAB[row(b)] (fp32) and the pad flags (all H channels exactly 0)
//   FFTBlocks stack   k_pos_scan, k_fs2_embed, 5 L layer kernels (dsx_fs2dec.cu); the last writes LN(x) * !pad as fp16
//   k_fft_out         get_mel_out + bias -> eps, contiguous fp32 [B][1][M][T]
#include <math.h>

#include <algorithm>

#include "dsx_conv.cuh"
#include "dsx_internal.h"
#include "dsx_ptx.cuh"

namespace dsx {

struct FftDenoiser {
  dsx_fft_config cfg{};
  dsx_fs2dec* dec = nullptr;   // the FFTBlocks stack (layers, final LayerNorm, pos_embed_alpha)
  DevAllocs mem;
  float* wd = nullptr;         // get_decode_inp.weight [H][dim + H + dim] fp32
  ModelDev emb{};              // C = dim and the mlp weights, for k_embed_table
  ConvGemm in, cond, out;      // entry (3M -> H), cond part (3H -> H), get_mel_out (H -> M)
  GrowBuffer ws;               // per evaluation: split operand, the stack's buffers, the exit operand
  GrowBuffer cp;               // CONDPART [B][T][H] fp32, kept between calls
  GrowBuffer tab;              // EMB [rows][dim], TTAB [rows][H]
  int rows = 0;                // rows tab holds
};

namespace {

constexpr int kSplit = 3;      // planes of a hi+lo operand along K
constexpr int kOutNT = 128;    // get_mel_out: M = 80 columns in one tile

// x logically [B][C][T] fp32 (strides xs) -> fp16 [B][T][3C] = (hi, lo, hi) of every value
__global__ void k_fft_split(const float* __restrict__ x, dsx_strides xs, int T, int C, __half* __restrict__ out) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const bool c_fast = xs.c == 1 && xs.t != 1;   // read along the unit-stride axis
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = c_fast ? t0 + i : t0 + threadIdx.x, c = c_fast ? c0 + threadIdx.x : c0 + i;
    const float v = (t < T && c < C) ? x[b * xs.b + c * xs.c + t * xs.t] : 0.f;
    if (c_fast) tile[threadIdx.x][i] = v; else tile[i][threadIdx.x] = v;   // tile[c][t]
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int t = t0 + i, c = c0 + threadIdx.x;
    if (t < T && c < C) {
      const float v = tile[threadIdx.x][i];
      const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
      __half* o = out + (static_cast<size_t>(b) * T + t) * kSplit * C + c;
      o[0] = hi;
      o[C] = lo;
      o[2 * C] = hi;
    }
  }
}

// w[n][col0 + k] (row stride ldw) -> out [N][3K] = (hi, hi, lo): fp32 values that fp16 holds exactly
__global__ void k_fft_split_w(const float* __restrict__ w, int ldw, int col0, int K, int N, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * K) return;
  const int n = i / K, k = i - n * K;
  const float v = w[static_cast<size_t>(n) * ldw + col0 + k];
  const float hi = __half2float(__float2half_rn(v)), lo = __half2float(__float2half_rn(v - hi));
  float* o = out + static_cast<size_t>(n) * kSplit * K + k;
  o[0] = hi;
  o[K] = hi;
  o[2 * K] = lo;
}

// W' [H][M] = Wd[:, 0:dim] . W_in and b' = Wd[:, 0:dim] . b_in + b_d, summed in double (block h, thread m; m == M: b')
__global__ void k_fft_fold(const float* __restrict__ wd, int ldw, const float* __restrict__ win,
                           const float* __restrict__ bin, const float* __restrict__ bd, int dim, int M,
                           float* __restrict__ wf, float* __restrict__ bf) {
  const int h = blockIdx.x, m = threadIdx.x;
  if (m > M) return;
  double acc = m == M ? static_cast<double>(bd[h]) : 0.0;
  for (int c = 0; c < dim; ++c) {
    const double a = wd[static_cast<size_t>(h) * ldw + c];
    acc += a * (m == M ? bin[c] : win[static_cast<size_t>(c) * M + m]);
  }
  if (m == M) bf[h] = static_cast<float>(acc);
  else wf[static_cast<size_t>(h) * M + m] = static_cast<float>(acc);
}

// TTAB[row][h] = Wd[h][col0:col0 + dim] . EMB[row] in fp32, one warp per (row, h)
__global__ void k_fft_tproj(const float* __restrict__ emb, const float* __restrict__ wd, int ldw, int col0, int dim,
                            int H, int rows, float* __restrict__ ttab) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= rows * H) return;
  const int row = warp / H, h = warp - row * H;
  const float* w = wd + static_cast<size_t>(h) * ldw + col0;
  const float* v = emb + static_cast<size_t>(row) * dim;
  float acc = 0.f;
  for (int k = lane; k < dim; k += 32) acc = fmaf(w[k], v[k], acc);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) ttab[warp] = acc;
}

struct FftInArgs {
  ConvGemm g;
  const __half* a;             // [B][T][g.cin] split operand
  int T;
  float* out;                  // [B][T][n] fp32
  const float* cp;             // non-null (entry): CONDPART [B][T][n]; null: out = the product alone (the cond part)
  const float* ttab;           // [rows][n]
  int row0, row_per_b;
  uint8_t* pad;                // [B][T]
};

// One 64-row tile of utterance blockIdx.y; one column tile holds all n <= 256 columns, so the pad flag of a row is
// decided here.
template <int NT>
__global__ void __launch_bounds__(128 * (NT > 128 ? 2 : 1)) k_fft_in(const FftInArgs p) {
  constexpr int WG = NT > 128 ? 2 : 1, NH = NT / WG;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ int nonzero[kConvRows];
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, b = blockIdx.y, m0 = blockIdx.x * kConvRows;
  if (tid < kConvRows) nonzero[tid] = 0;   // published by the K loop's barriers
  float acc[NH / 2];
  conv_k_loop<NT, WG>(p.g, p.a, p.T, p.T, b, m0, 0, smem, acc);

  const int n = p.g.n, c0 = wg * NH, r0 = acc_row(wtid, 0);
  const size_t rbase = static_cast<size_t>(b) * p.T;
  const float* tt = p.cp ? p.ttab + static_cast<size_t>(p.row0 + b * p.row_per_b) * n : nullptr;
  bool any[2] = {false, false};
#pragma unroll
  for (int e = 0; e < NH / 2; e += 2) {
    const int col = c0 + acc_col(wtid, e), r = (e >> 1) & 1, m = m0 + r0 + 8 * r;
    if (col >= n || m >= p.T) continue;
    const size_t idx = (rbase + m) * n + col;
    float v0 = acc[e], v1 = acc[e + 1];
    if (p.cp) {
      const float2 c = *reinterpret_cast<const float2*>(p.cp + idx);
      v0 = ((v0 + __ldg(p.g.b + col)) + c.x) + __ldg(tt + col);
      v1 = ((v1 + __ldg(p.g.b + col + 1)) + c.y) + __ldg(tt + col + 1);
      any[r] = any[r] || v0 != 0.f || v1 != 0.f;
    }
    *reinterpret_cast<float2*>(p.out + idx) = make_float2(v0, v1);
  }
  if (!p.cp) return;
  if (any[0]) nonzero[r0] = 1;
  if (any[1]) nonzero[r0 + 8] = 1;
  __syncthreads();
  if (tid < kConvRows && m0 + tid < p.T) p.pad[rbase + m0 + tid] = nonzero[tid] ? 0 : 1;
}

// eps[b][0][col][m] = A[b][m] . mel_out_w[col] + bias[col], contiguous [B][1][n][T]
__global__ void __launch_bounds__(128) k_fft_out(const ConvGemm g, const __half* __restrict__ a, int T,
                                                 float* __restrict__ eps) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int tid = threadIdx.x, b = blockIdx.y, m0 = blockIdx.x * kConvRows;
  float acc[kOutNT / 2];
  conv_k_loop<kOutNT, 1>(g, a, T, T, b, m0, 0, smem, acc);
  const int n = g.n, r0 = acc_row(tid, 0);
#pragma unroll
  for (int e = 0; e < kOutNT / 2; e += 2) {
    const int col = acc_col(tid, e), m = m0 + r0 + 8 * ((e >> 1) & 1);
    if (col >= n || m >= T) continue;
    float* o = eps + (static_cast<size_t>(b) * n + col) * T + m;
    o[0] = acc[e] + __ldg(g.b + col);
    o[T] = acc[e + 1] + __ldg(g.b + col + 1);
  }
}

int fft_in_run(const FftInArgs& p, int B, cudaStream_t s) {
  const dim3 grid((p.T + kConvRows - 1) / kConvRows, B, 1);
  return conv_dispatch<256>(p.g.nt, [&](auto c) {
    constexpr int NT = decltype(c)::value;
    k_fft_in<NT><<<grid, 128 * (NT > 128 ? 2 : 1), conv_smem<NT>(), s>>>(p);
    return launch_check("k_fft_in");
  });
}

// packs w [N][3K] (the output of k_fft_split_w) with bias b (or none) as a linear 3K -> N
int fft_pack(DevAllocs& mem, ConvGemm& g, const float* w, const float* b, int K, int N, int nt_max, cudaStream_t s) {
  g.cin = kSplit * K;
  g.n = N;
  g.taps = 1;
  g.tap0 = 0;
  return conv_pack(mem, g, nt_max, PackArgs{w, nullptr, b, kSplit * K, N, N, 1, 1, 0}, s);
}

int fft_copy(DevAllocs& mem, float** dst, const float* src, size_t n, const char* what, cudaStream_t s) {
  DSX_CHECK(src, DSX_E_INVALID, "missing %s", what);
  DSX_TRY(mem.alloc(dst, n * sizeof(float)));
  DSX_CUDA(cudaMemcpyAsync(*dst, src, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return DSX_OK;
}

int fft_build(FftDenoiser* f, int device, const dsx_fft_config* c, const dsx_fft_params* p, cudaStream_t s) {
  DSX_TRY(dsx_fs2dec_create(device, &c->dec, &f->dec));
  DSX_TRY(dsx_fs2dec_load(f->dec, &p->dec, s));
  DSX_TRY(conv_opt_in<256>([](auto k) { return k_fft_in<decltype(k)::value>; }));
  DSX_CUDA(cudaFuncSetAttribute(k_fft_out, cudaFuncAttributeMaxDynamicSharedMemorySize, conv_smem<kOutNT>()));
  const int dim = c->residual_channels, H = c->dec.hidden, M = c->mel_bins, ldw = dim + H + dim;
  DSX_CHECK(p->in_w && p->in_b && p->decode_inp_b && p->mel_out_w && p->mel_out_b, DSX_E_INVALID,
            "missing input_projection, get_decode_inp or get_mel_out arrays");
  ModelDev& e = f->emb;
  e.C = dim;
  float *mlp0_w, *mlp0_b, *mlp2_w, *mlp2_b;
  DSX_TRY(fft_copy(f->mem, &mlp0_w, p->mlp0_w, static_cast<size_t>(4) * dim * dim, "mlp.0.weight", s));
  DSX_TRY(fft_copy(f->mem, &mlp0_b, p->mlp0_b, static_cast<size_t>(4) * dim, "mlp.0.bias", s));
  DSX_TRY(fft_copy(f->mem, &mlp2_w, p->mlp2_w, static_cast<size_t>(4) * dim * dim, "mlp.2.weight", s));
  DSX_TRY(fft_copy(f->mem, &mlp2_b, p->mlp2_b, dim, "mlp.2.bias", s));
  e.mlp0_w = mlp0_w;
  e.mlp0_b = mlp0_b;
  e.mlp2_w = mlp2_w;
  e.mlp2_b = mlp2_b;
  DSX_TRY(fft_copy(f->mem, &f->wd, p->decode_inp_w, static_cast<size_t>(H) * ldw, "get_decode_inp.weight", s));

  // pack scratch, freed with the model: W' and b', then the (hi, hi, lo) weights of the entry and the cond part
  float *wf, *bf, *w_in, *w_cond;
  DSX_TRY(f->mem.alloc(&wf, static_cast<size_t>(H) * M * sizeof(float)));
  DSX_TRY(f->mem.alloc(&bf, static_cast<size_t>(H) * sizeof(float)));
  DSX_TRY(f->mem.alloc(&w_in, static_cast<size_t>(H) * kSplit * M * sizeof(float)));
  DSX_TRY(f->mem.alloc(&w_cond, static_cast<size_t>(H) * kSplit * H * sizeof(float)));
  k_fft_fold<<<H, 128, 0, s>>>(f->wd, ldw, p->in_w, p->in_b, p->decode_inp_b, dim, M, wf, bf);
  DSX_TRY(launch_check("k_fft_fold"));
  k_fft_split_w<<<(H * M + 255) / 256, 256, 0, s>>>(wf, M, 0, M, H, w_in);
  DSX_TRY(launch_check("k_fft_split_w"));
  k_fft_split_w<<<(H * H + 255) / 256, 256, 0, s>>>(f->wd, ldw, dim, H, H, w_cond);
  DSX_TRY(launch_check("k_fft_split_w"));
  DSX_TRY(fft_pack(f->mem, f->in, w_in, bf, M, H, 256, s));
  DSX_TRY(fft_pack(f->mem, f->cond, w_cond, nullptr, H, H, 256, s));
  f->out.cin = H;
  f->out.n = M;
  f->out.taps = 1;
  f->out.tap0 = 0;
  DSX_TRY(conv_pack(f->mem, f->out, kOutNT, PackArgs{p->mel_out_w, nullptr, p->mel_out_b, H, M, M, 1, 1, 0}, s));
  DSX_CHECK(f->in.ntiles == 1 && f->cond.ntiles == 1 && f->out.ntiles == 1 && f->out.nt == kOutNT, DSX_E_INVALID,
            "internal: unexpected FFT denoiser tiling");
  return DSX_OK;
}

}  // namespace

int fft_create(int device, const dsx_fft_config* c, const dsx_fft_params* p, cudaStream_t s, FftDenoiser** out) {
  *out = nullptr;
  DSX_CHECK(c && p, DSX_E_INVALID, "null config or params");
  DSX_CHECK(c->mel_bins == 80, DSX_E_INVALID, "unsupported mel_bins %d: 80 (get_mel_out is Linear(hidden_size, 80))",
            c->mel_bins);
  DSX_CHECK(c->residual_channels >= 16 && c->residual_channels <= 1024 && c->residual_channels % 16 == 0,
            DSX_E_INVALID, "unsupported residual_channels %d: a multiple of 16 in [16, 1024]", c->residual_channels);
  FftDenoiser* f = new FftDenoiser();
  f->cfg = *c;
  const int rc = fft_build(f, device, c, p, s);
  if (rc == DSX_OK) {
    cudaError_t e = cudaStreamSynchronize(s);   // the pack scratch is read by queued kernels
    if (e == cudaSuccess) {
      *out = f;
      return DSX_OK;
    }
    set_error("FFT denoiser load: %s", cudaGetErrorString(e));
    fft_destroy(f);
    return DSX_E_CUDA;
  }
  fft_destroy(f);
  return rc;
}

void fft_destroy(FftDenoiser* f) {
  if (!f) return;
  cudaDeviceSynchronize();
  dsx_fs2dec_destroy(f->dec);
  f->mem.free_all();
  f->ws.release();
  f->cp.release();
  f->tab.release();
  delete f;
}

int fft_workspace(dsx_handle* h, const Geom& g, int rows, cudaStream_t s) {
  FftDenoiser* f = h->fft;
  const int B = g.B, T = g.T, H = f->cfg.dec.hidden, M = f->cfg.mel_bins, dim = f->cfg.residual_channels;
  DSX_CHECK(B <= 65535, DSX_E_INVALID, "B = %d utterances per call is above the 65535 the launch grid holds", B);
  const long long Tp = (T + kConvRows - 1) / kConvRows * kConvRows;
  DSX_CHECK(static_cast<long long>(B) * Tp * 4 * H < (1ll << 31), DSX_E_INVALID, "B * T = %lld frames is too large",
            static_cast<long long>(B) * T);
  const size_t frames = static_cast<size_t>(B) * T;
  DSX_TRY(f->ws.reserve(align256(frames * kSplit * std::max(M, H) * 2) + fs2_workspace_bytes(f->dec, B, T) +
                            align256(frames * H * 2),
                        s));
  const void* cp_before = f->cp.ptr;
  DSX_TRY(f->cp.reserve(frames * H * 4, s));
  if (f->cp.ptr != cp_before) h->cond_ready = false;
  if (rows > f->rows) {
    DSX_TRY(f->tab.reserve(align256(static_cast<size_t>(rows) * dim * 4) + static_cast<size_t>(rows) * H * 4, s));
    f->rows = rows;
  }
  return DSX_OK;
}

int fft_set_cond(dsx_handle* h, const float* cond, dsx_strides cs, const Geom& g, cudaStream_t s) {
  FftDenoiser* f = h->fft;
  const int H = f->cfg.dec.hidden;
  __half* split = static_cast<__half*>(f->ws.ptr);
  k_fft_split<<<dim3((g.T + 31) / 32, (H + 31) / 32, g.B), dim3(32, 8), 0, s>>>(cond, cs, g.T, H, split);
  DSX_TRY(launch_check("k_fft_split"));
  FftInArgs a{};
  a.g = f->cond;
  a.a = split;
  a.T = g.T;
  a.out = static_cast<float*>(f->cp.ptr);
  DSX_TRY(fft_in_run(a, g.B, s));
  h->launches += 2;
  return DSX_OK;
}

int fft_embed_table(dsx_handle* h, const int64_t* t_dev, int rows, cudaStream_t s) {
  FftDenoiser* f = h->fft;
  const int dim = f->cfg.residual_channels, H = f->cfg.dec.hidden;
  float* emb = static_cast<float*>(f->tab.ptr);
  float* ttab = reinterpret_cast<float*>(static_cast<uint8_t*>(f->tab.ptr) + align256(static_cast<size_t>(f->rows) * dim * 4));
  DSX_TRY(launch_embed_mlp(h, f->emb, t_dev, rows, emb, s));
  const int warps = rows * H;
  k_fft_tproj<<<(warps + 7) / 8, 256, 0, s>>>(emb, f->wd, dim + H + dim, dim + H, dim, H, rows, ttab);
  return counted_launch(h, "k_fft_tproj");
}

int fft_eval(dsx_handle* h, const float* x, dsx_strides xs, const Geom& g, int row0, int row_per_b, float* eps,
             cudaStream_t s) {
  FftDenoiser* f = h->fft;
  const int B = g.B, T = g.T, H = f->cfg.dec.hidden, M = f->cfg.mel_bins, dim = f->cfg.residual_channels;
  const size_t frames = static_cast<size_t>(B) * T;
  uint8_t* base = static_cast<uint8_t*>(f->ws.ptr);
  __half* split = reinterpret_cast<__half*>(base);
  base += align256(frames * kSplit * std::max(M, H) * 2);
  const Fs2Bufs w = fs2_carve(f->dec, base, B, T);
  __half* a16 = reinterpret_cast<__half*>(base + fs2_workspace_bytes(f->dec, B, T));

  k_fft_split<<<dim3((T + 31) / 32, (M + 31) / 32, B), dim3(32, 8), 0, s>>>(x, xs, T, M, split);
  DSX_TRY(launch_check("k_fft_split"));
  FftInArgs a{};
  a.g = f->in;
  a.a = split;
  a.T = T;
  a.out = w.X;
  a.cp = static_cast<const float*>(f->cp.ptr);
  a.ttab = reinterpret_cast<const float*>(static_cast<const uint8_t*>(f->tab.ptr) +
                                          align256(static_cast<size_t>(f->rows) * dim * 4));
  a.row0 = row0;
  a.row_per_b = row_per_b;
  a.pad = w.PAD;
  DSX_TRY(fft_in_run(a, B, s));
  DSX_TRY(fs2_stack_run(f->dec, w, B, T, nullptr, a16, s));
  k_fft_out<<<dim3((T + kConvRows - 1) / kConvRows, B, 1), 128, conv_smem<kOutNT>(), s>>>(f->out, a16, T, eps);
  DSX_TRY(launch_check("k_fft_out"));
  h->launches += 5 + 5 * fs2_layers(f->dec);
  return DSX_OK;
}

}  // namespace dsx
