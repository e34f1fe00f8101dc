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

#include "dsx_fftentry.cuh"

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
