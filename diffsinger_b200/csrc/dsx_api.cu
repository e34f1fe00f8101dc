// C ABI of the dsx sampler (include/dsx.h): handle, weight loading, schedule, workspace, and the host
// side of the sampling loops.  The K-step loops run as a fixed sequence of kernel launches on the
// caller's stream -- no host synchronisation and no PyTorch op inside the loop
// (usr/diff/shallow_diffusion_tts.py:261-270 is a Python loop of ~300 ATen launches per step).
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>

#include "dsx_internal.h"

namespace dsx {

static thread_local char g_err[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

// Grow-only workspace: a call with a new (B, T) that fits re-uses the allocations (only the geometry changes), so
// utterance lengths that change from call to call cost no cudaFree / cudaMalloc.  New allocations are zeroed on the
// caller's stream: padding frames, SKIP and FLAGS depend on it.
int ensure_workspace(dsx_handle* h, const Geom& g, int rows, cudaStream_t s) {
  Workspace& w = h->ws;
  const ModelDev& m = h->m;
  const bool tc = h->precision != DSX_PREC_FP32_SIMT;
  const size_t nf = g.frames_padded();
  if (!h->fft) {   // the FFT denoiser keeps its own per-evaluation buffers (fft_workspace)
    DSX_TRY(w.X.reserve_zeroed(nf * m.C * 4, s));
    DSX_TRY(w.SKIP.reserve_zeroed(nf * m.C * 4, s));
    if (tc) {
      const void* cond_before[2] = {w.CONDH, w.CP};
      DSX_TRY(w.Y.reserve_zeroed(nf * m.C * 2 * 4, s));
      DSX_TRY(w.CONDH.reserve_zeroed(nf * m.H * 2 * 2, s));
      DSX_TRY(w.S16.reserve_zeroed(nf * m.C * 2 * 2, s));
      DSX_TRY(w.FLAGS.reserve_zeroed(nf / 64 * 2 * sizeof(unsigned), s));   // two per tile at the smallest tile height, 64 frames
      DSX_TRY(w.CP.reserve_zeroed(static_cast<size_t>(m.L) * nf * 2 * m.C * 4, s));
      if (cond_before[0] != w.CONDH || cond_before[1] != w.CP) h->cond_ready = false;
    } else {
      const void* cond_before = w.CONDF;
      DSX_TRY(w.G1.reserve_zeroed(nf * simt_g1_cols(m) * 4, s));
      DSX_TRY(w.Zf.reserve_zeroed(nf * m.C * 4, s));
      DSX_TRY(w.CONDF.reserve_zeroed(nf * m.H * 4, s));
      if (cond_before != w.CONDF) h->cond_ready = false;
    }
  }
  if (w.rows_cap < rows) {
    const int keep_rows = std::max(rows, w.rows_cap + w.rows_cap / 2);
    if (!h->fft) {
      DSX_TRY(w.DTAB.reserve_zeroed(static_cast<size_t>(keep_rows) * m.L * m.C * 4, s));
      DSX_TRY(w.EMB.reserve_zeroed(static_cast<size_t>(keep_rows) * m.C * 4, s));
    }
    DSX_TRY(w.TVALS.reserve_zeroed(static_cast<size_t>(keep_rows) * 8, s));
    w.rows_cap = keep_rows;
  }
  if (h->fft) DSX_TRY(fft_workspace(h, g, w.rows_cap, s));
  const size_t mel = static_cast<size_t>(g.B) * m.M * g.T;
  DSX_TRY(w.EPS.reserve_zeroed(5 * mel * 4, s));
  DSX_TRY(w.XTMP.reserve_zeroed(mel * 4, s));
  DSX_TRY(w.XSTATE.reserve_zeroed(mel * 4, s));
  w.g = g;
  return DSX_OK;
}

int check_status(dsx_handle* h, cudaStream_t s, const char* what) {
  DSX_CUDA(cudaMemcpyAsync(h->status_host, h->status_dev, sizeof(int), cudaMemcpyDeviceToHost, s));
  DSX_CUDA(cudaStreamSynchronize(s));
  if (*h->status_host != 0) {
    int code = *h->status_host;
    cudaMemsetAsync(h->status_dev, 0, sizeof(int), s);
    set_error("%s: in-kernel self-check tripped (code %d)", what, code);
    return DSX_E_KERNEL;
  }
  return DSX_OK;
}

// `run` between two CUDA events on s when `on` (DSX_OPT_PROFILE), summed by DSX_INFO_LAYER_KERNEL_NS
template <typename F>
static int profiled(dsx_handle* h, bool on, cudaStream_t s, F&& run) {
  if (!on) return run();
  while (h->prof_events.size() < h->prof_used + 2) {
    cudaEvent_t e;
    DSX_CUDA(cudaEventCreate(&e));
    h->prof_events.push_back(e);
  }
  const size_t i = h->prof_used;
  h->prof_used += 2;
  DSX_CUDA(cudaEventRecord(h->prof_events[i], s));
  DSX_TRY(run());
  DSX_CUDA(cudaEventRecord(h->prof_events[i + 1], s));
  return DSX_OK;
}

// the tensor-core DiffNet kernels (fused heads, updates and input projections); the SIMT DiffNet and the FFT denoiser
// evaluate to eps and run the fp32 update kernels
static bool tc_diffnet(const dsx_handle* h) { return !h->fft && h->precision != DSX_PREC_FP32_SIMT; }

// One evaluation of the loaded denoiser on x_in (strides ha.xs) at FiLM table row (row0, row_per_b), then what `ha`
// asks for: eps (TC_WRITE_EPS), the DDPM (TC_UPDATE) or PLMS (TC_PLMS) update of ha.x, and on the tensor-core path the
// input projection of the next evaluation (TC_INPROJ).  The tensor-core layers read x_in through the projection the
// previous head made; `project` makes it here instead (a loop's first evaluation, a forward).  Fewer than L layers
// (dsx_debug_set_layer_limit) run no head and nothing after it.
static int evaluate(dsx_handle* h, const Geom& g, const float* x_in, int row0, int row_per_b, int nl, bool project,
                    const HeadArgs& ha, cudaStream_t s) {
  const bool head = nl == h->m.L;
  if (tc_diffnet(h)) {
    if (project) {
      HeadArgs in;
      in.flags = TC_INPROJ;
      in.x = const_cast<float*>(x_in);   // read only with this flag
      in.xs = ha.xs;
      in.next_row0 = row0;
      in.row_per_b = row_per_b;
      DSX_TRY(launch_tc_step(h, g, 0, 0, row0, row_per_b, &in, s));
    }
    const bool fuse = head && tc_fuse_head(h);
    DSX_TRY(profiled(h, h->profile == 1, s, [&] { return launch_tc_step(h, g, 0, nl, row0, row_per_b, fuse ? &ha : nullptr, s); }));
    if (head && !fuse) DSX_TRY(profiled(h, h->profile == 2, s, [&] { return launch_tc_step(h, g, 0, 0, row0, row_per_b, &ha, s); }));
    return DSX_OK;
  }
  // SIMT and FFT: eps to where the flags keep it, else to slot 4 of the EPS ring, then the fp32 update kernel
  const size_t mel = static_cast<size_t>(g.B) * h->m.M * g.T;
  const PlmsFuse* p = ha.plms;
  float* eps = (ha.flags & TC_WRITE_EPS) ? ha.eps : (p && p->eps_store) ? p->eps_store : h->ws.EPS + 4 * mel;
  if (h->fft) {
    DSX_TRY(fft_eval(h, x_in, ha.xs, g, row0, row_per_b, eps, s));
  } else {
    DSX_TRY(launch_inproj(h, x_in, ha.xs, g, row0, row_per_b, s));
    DSX_TRY(profiled(h, h->profile == 1, s, [&]() -> int {
      for (int l = 0; l < nl; ++l) DSX_TRY(launch_simt_layer(h, l, g, row0, row_per_b, s));
      return DSX_OK;
    }));
    if (!head) return DSX_OK;
    DSX_TRY(launch_head(h, g, eps, s));
  }
  if (ha.flags & TC_UPDATE) return launch_ddpm_update(h, ha.x, eps, ha.noise, ha.seed, ha.offset, ha.c, mel, g.T, s);
  if (!(ha.flags & TC_PLMS)) return DSX_OK;
  float* x_out = p->x_out ? p->x_out : ha.x;
  if (p->eps_store) return launch_plms_update(h, x_out, ha.x, eps, p->h1, p->h2, p->h3, p->c, mel, s);
  // the warm-up's combine: this eps is the second of (eps_t + eps') / 2
  return launch_plms_update(h, x_out, ha.x, p->h1, eps, nullptr, nullptr, p->c, mel, s);
}

// Workspace for (B, T) and, when `cond` is given, the conditioner pack and its hoisted projection (the
// step-independent part of every residual layer).  cond == NULL re-uses what the last call with a conditioner left behind
// (dsx_set_cond or any entry point): callers that drive the sampling loop themselves, one p_sample / DiffNet.forward per
// call, pay the pack + projection once per utterance batch instead of once per step.
static int prepare(dsx_handle* h, const float* cond, dsx_strides cs, int B, int T, int rows, Geom& g, cudaStream_t s) {
  DSX_CHECK(h && h->loaded, DSX_E_STATE, "dsx_load_diffnet has not been called");
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CUDA(cudaSetDevice(h->device));
  g.set(B, T);
  DSX_TRY(ensure_workspace(h, g, rows, s));
  if (!cond) {
    DSX_CHECK(h->cond_ready && h->cond_geom.B == B && h->cond_geom.T == T, DSX_E_STATE,
              "cond == NULL needs a conditioner set for the same (B, T) by dsx_set_cond or an earlier call (have %s %dx%d, asked %dx%d)",
              h->cond_ready ? "one for" : "none;", h->cond_geom.B, h->cond_geom.T, B, T);
    return DSX_OK;
  }
  h->cond_ready = false;
  if (h->fft) {
    DSX_TRY(fft_set_cond(h, cond, cs, g, s));
  } else {
    DSX_TRY(launch_pack_cond(h, cond, cs, g, s));
    if (h->precision != DSX_PREC_FP32_SIMT) DSX_TRY(launch_tc_condproj(h, g, s));
  }
  h->cond_ready = true;
  h->cond_geom = g;
  return DSX_OK;
}

// step table of the loaded denoiser: rows of t_dev -> DiffNet's FiLM vectors or the FFT's get_decode_inp step part
static int embed_table(dsx_handle* h, const int64_t* t_dev, int rows, cudaStream_t s) {
  return h->fft ? fft_embed_table(h, t_dev, rows, s) : launch_embed_table(h, t_dev, rows, s);
}

static dsx_strides contiguous_mel(int M, int T) {
  dsx_strides xs;
  xs.b = static_cast<int64_t>(M) * T;
  xs.c = T;
  xs.t = 1;
  return xs;
}

static int sample_ddpm_impl(dsx_handle* h, float* x, const Geom& g, int t_start, int n_steps, const float* noise,
                            uint64_t seed, cudaStream_t s) {
  const size_t mel = static_cast<size_t>(g.B) * h->m.M * g.T;
  std::vector<int64_t> tv(n_steps);
  for (int j = 0; j < n_steps; ++j) tv[j] = t_start - 1 - j;
  DSX_CUDA(cudaMemcpyAsync(h->ws.TVALS, tv.data(), n_steps * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  DSX_CUDA(cudaStreamSynchronize(s));   // tv is a stack-owned staging buffer
  DSX_TRY(embed_table(h, h->ws.TVALS, n_steps, s));
  const dsx_strides xs = contiguous_mel(h->m.M, g.T);
  for (int j = 0; j < n_steps; ++j) {
    const int t = t_start - 1 - j;
    HeadArgs ha;
    ha.flags = TC_HEAD | TC_UPDATE | (j + 1 < n_steps ? TC_INPROJ : 0);
    ha.x = x;
    ha.xs = xs;
    ha.noise = noise ? noise + static_cast<size_t>(j) * mel : nullptr;
    ha.seed = seed;
    ha.offset = static_cast<uint64_t>(j);
    ha.c.A = h->sched[DSX_SCH_SQRT_RECIP_ALPHAS_CUMPROD][t];
    ha.c.Bc = h->sched[DSX_SCH_SQRT_RECIPM1_ALPHAS_CUMPROD][t];
    ha.c.c1 = h->sched[DSX_SCH_POSTERIOR_MEAN_COEF1][t];
    ha.c.c2 = h->sched[DSX_SCH_POSTERIOR_MEAN_COEF2][t];
    ha.c.sigma = (t == 0) ? 0.f : expf(0.5f * h->sched[DSX_SCH_POSTERIOR_LOG_VARIANCE_CLIPPED][t]);
    ha.next_row0 = j + 1;
    DSX_TRY(evaluate(h, g, x, j, 0, h->m.L, j == 0, ha, s));
  }
  return DSX_OK;
}

// PLMS weights (w0, w1, w2, w3, denom) of eps_t and the earlier eps, by dsx_plms_update mode: 0 / 1 the warm-up's
// first update and its combine, 2 / 3 / 4 with one / two / three earlier eps
static const float kPlmsWeights[5][5] = {
    {1.f, 0.f, 0.f, 0.f, 1.f}, {1.f, 1.f, 0.f, 0.f, 2.f}, {3.f, -1.f, 0.f, 0.f, 2.f},
    {23.f, -16.f, 5.f, 0.f, 12.f}, {55.f, -59.f, 37.f, -9.f, 24.f}};

// get_x_pred coefficients (usr/diff/shallow_diffusion_tts.py:174-185), fp32 op by op, and the weights of `mode`
static PlmsCoef plms_coefs(const dsx_handle* h, int t, int interval, int mode) {
  const std::vector<float>& ac = h->sched[DSX_SCH_ALPHAS_CUMPROD];
  const float a_t = ac[t];
  const float a_prev = (t < interval) ? 1.0f : ac[std::max(t - interval, 0)];
  const float a_t_sq = sqrtf(a_t), a_prev_sq = sqrtf(a_prev);
  PlmsCoef c;
  c.a_diff = a_prev - a_t;
  c.kx = 1.0f / (a_t_sq * (a_t_sq + a_prev_sq));
  c.ke = 1.0f / (a_t_sq * (sqrtf((1.0f - a_prev) * a_t) + sqrtf((1.0f - a_t) * a_prev)));
  const float* w = kPlmsWeights[mode];
  c.w0 = w[0]; c.w1 = w[1]; c.w2 = w[2]; c.w3 = w[3]; c.denom = w[4];
  return c;
}

static int sample_plms_impl(dsx_handle* h, float* x, const Geom& g, int t_start, int interval, cudaStream_t s) {
  const size_t mel = static_cast<size_t>(g.B) * h->m.M * g.T;
  std::vector<int> steps;
  for (int t = 0; t < t_start; t += interval) steps.push_back(t);
  std::reverse(steps.begin(), steps.end());
  const int n = static_cast<int>(steps.size());
  DSX_CHECK(n > 0, DSX_E_INVALID, "empty PLMS schedule");
  // table rows: 0..n-1 = the steps, row n = the extra warm-up evaluation at max(t0 - interval, 0)
  std::vector<int64_t> tv(n + 1);
  for (int j = 0; j < n; ++j) tv[j] = steps[j];
  tv[n] = std::max(steps[0] - interval, 0);
  DSX_CUDA(cudaMemcpyAsync(h->ws.TVALS, tv.data(), (n + 1) * sizeof(int64_t), cudaMemcpyHostToDevice, s));
  DSX_CUDA(cudaStreamSynchronize(s));
  DSX_TRY(embed_table(h, h->ws.TVALS, n + 1, s));
  const dsx_strides xs = contiguous_mel(h->m.M, g.T);
  // eps_t of step j goes to slot j % 4 of the EPS ring; the three before it are the multistep history
  auto ring = [&](int j) -> float* { return j >= 0 ? h->ws.EPS + static_cast<size_t>(j % 4) * mel : nullptr; };
  for (int j = 0; j < n; ++j) {
    PlmsFuse pf{};
    HeadArgs ha;
    ha.flags = TC_HEAD | TC_PLMS | (j + 1 < n ? TC_INPROJ : 0);
    ha.x = x;
    ha.xs = xs;
    ha.next_row0 = j + 1;
    ha.plms = &pf;
    if (j == 0) {
      // warm-up: x' = phi(x, eps_t, t) -> XTMP; eps' = net(x', max(t - interval, 0)); x = phi(x, (eps_t + eps') / 2, t)
      PlmsFuse first{};
      first.c = plms_coefs(h, steps[0], interval, 0);
      first.eps_store = ring(0);
      first.x_out = h->ws.XTMP;
      HeadArgs ha1 = ha;
      ha1.flags = TC_HEAD | TC_PLMS | TC_INPROJ;
      ha1.next_row0 = n;
      ha1.plms = &first;
      DSX_TRY(evaluate(h, g, x, 0, 0, h->m.L, true, ha1, s));
      pf.c = plms_coefs(h, steps[0], interval, 1);
      pf.h1 = ring(0);
      DSX_TRY(evaluate(h, g, h->ws.XTMP, n, 0, h->m.L, false, ha, s));
    } else {
      pf.c = plms_coefs(h, steps[j], interval, std::min(j, 3) + 1);
      pf.h1 = ring(j - 1);
      pf.h2 = ring(j - 2);
      pf.h3 = ring(j - 3);
      pf.eps_store = ring(j);
      DSX_TRY(evaluate(h, g, x, j, 0, h->m.L, false, ha, s));
    }
  }
  return DSX_OK;
}

}  // namespace dsx

using namespace dsx;

extern "C" {

int dsx_version(void) { return DSX_VERSION; }
const char* dsx_last_error(void) { return g_err; }

int dsx_create(int device, dsx_handle** out) {
  DSX_CHECK(out, DSX_E_INVALID, "out is NULL");
  cudaDeviceProp prop;
  DSX_TRY(select_device(device, &prop));
  dsx_handle* h = new dsx_handle();
  h->device = device;
  h->sm_count = prop.multiProcessorCount;
  // the tensor-core kernels are built for sm_90a (wgmma) only; other devices can still run the fp32 path
  h->tc_group = (prop.major == 9 && prop.minor == 0) ? 2 : 0;
  if (cudaMalloc(&h->status_dev, sizeof(int)) != cudaSuccess ||
      cudaMallocHost(&h->status_host, sizeof(int)) != cudaSuccess) {
    set_error("status word allocation failed");
    delete h;
    return DSX_E_CUDA;
  }
  cudaMemset(h->status_dev, 0, sizeof(int));
  *h->status_host = 0;
  *out = h;
  return DSX_OK;
}

static void free_model(dsx_handle* h) {
  h->mem.free_all();
  h->loaded = false;
}

void dsx_destroy(dsx_handle* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  free_model(h);
  h->ws.release();
  fft_destroy(h->fft);
  for (cudaEvent_t e : h->prof_events) cudaEventDestroy(e);
  for (GrowBuffer& b : h->stage) b.release();
  if (h->status_dev) cudaFree(h->status_dev);
  if (h->status_host) cudaFreeHost(h->status_host);
  if (h->trace_dev) cudaFree(h->trace_dev);
  delete h;
}

int dsx_load_diffnet(dsx_handle* h, const dsx_diffnet_params* p, int M, int C, int H, int L, int dilation_cycle,
                     int precision, void* stream) {
  DSX_CHECK(h && p, DSX_E_INVALID, "null handle or params");
  DSX_CHECK(M > 0 && C > 0 && H > 0 && L > 0 && dilation_cycle > 0, DSX_E_INVALID, "bad model dimensions");
  DSX_CHECK(C % 16 == 0 && H % 16 == 0 && M % 16 == 0, DSX_E_INVALID, "M, C, H must be multiples of 16 (got %d %d %d)", M, C, H);
  DSX_CHECK(precision == DSX_PREC_FP32_SIMT || precision == DSX_PREC_FP16 || precision == DSX_PREC_FP16X2 ||
                precision == DSX_PREC_FP16X3 || precision == DSX_PREC_FP16S,
            DSX_E_INVALID, "unknown precision %d", precision);
  DSX_CHECK(M <= kSimtMaxM && C <= kSimtMaxC, DSX_E_INVALID,
            "mel bins must be <= %d and residual channels <= %d (got M %d, C %d)", kSimtMaxM, kSimtMaxC, M, C);
  if (precision != DSX_PREC_FP32_SIMT) {
    DSX_CHECK(M == 80 && C == 256 && H == 256, DSX_E_INVALID,
              "tensor-core path needs mel bins == 80 and residual_channels == hidden_size == 256 (got M %d, C %d, H %d); "
              "use DSX_PREC_FP32_SIMT", M, C, H);
    DSX_CHECK(dilation_cycle <= 4, DSX_E_INVALID,
              "tensor-core path supports dilations up to 8 (dilation_cycle_length <= 4, got %d); use DSX_PREC_FP32_SIMT", dilation_cycle);
  }
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  free_model(h);
  h->ws.release();
  fft_destroy(h->fft);
  h->fft = nullptr;
  h->cond_ready = false;
  memset(&h->m, 0, sizeof(h->m));
  h->m.M = M; h->m.C = C; h->m.H = H; h->m.L = L; h->m.cycle = dilation_cycle;
  h->precision = precision;
  if (precision != DSX_PREC_FP32_SIMT)
    DSX_CHECK(h->tc_group != 0, DSX_E_INVALID, "tensor-core precisions need an sm_90 (H100) device");
  DSX_TRY(simt_pack_model(h, p, s));
  if (precision != DSX_PREC_FP32_SIMT) DSX_TRY(tc_pack_model(h, s));
  DSX_CUDA(cudaStreamSynchronize(s));
  h->loaded = true;
  return DSX_OK;
}

int dsx_load_fft(dsx_handle* h, const dsx_fft_config* cfg, const dsx_fft_params* p, void* stream) {
  DSX_CHECK(h && cfg && p, DSX_E_INVALID, "null handle, config or params");
  DSX_CUDA(cudaSetDevice(h->device));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  FftDenoiser* f = nullptr;
  DSX_TRY(fft_create(h->device, cfg, p, s, &f));   // validates and packs before the old denoiser is let go
  free_model(h);
  h->ws.release();
  fft_destroy(h->fft);
  h->fft = f;
  h->cond_ready = false;
  memset(&h->m, 0, sizeof(h->m));
  h->m.M = cfg->mel_bins;
  h->m.H = cfg->dec.hidden;
  h->precision = DSX_PREC_FP16;
  h->loaded = true;
  return DSX_OK;
}

int dsx_set_schedule(dsx_handle* h, const float* const* bufs, int T) {
  DSX_CHECK(h && bufs && T > 0, DSX_E_INVALID, "bad schedule arguments");
  for (int i = 0; i < DSX_SCH_COUNT; ++i) {
    DSX_CHECK(bufs[i], DSX_E_INVALID, "schedule buffer %d is NULL", i);
    h->sched[i].assign(bufs[i], bufs[i] + T);
  }
  h->sched_T = T;
  return DSX_OK;
}

int dsx_diffnet_forward(dsx_handle* h, const float* x, dsx_strides xs, const int64_t* t, const float* cond,
                        dsx_strides cs, float* eps, int B, int T, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_CHECK(x && t && eps, DSX_E_INVALID, "null tensor pointer");
  Geom g;
  DSX_TRY(prepare(h, cond, cs, B, T, B, g, s));
  DSX_TRY(embed_table(h, t, B, s));
  HeadArgs ha;
  ha.flags = TC_HEAD | TC_WRITE_EPS;
  ha.x = const_cast<float*>(x);          // read only with these flags
  ha.xs = xs;
  ha.eps = eps;
  const int nl = (h->layer_limit >= 0) ? std::min(h->layer_limit, h->m.L) : h->m.L;
  DSX_TRY(evaluate(h, g, x, 0, 1, nl, true, ha, s));
  return check_status(h, s, "dsx_diffnet_forward");
}

int dsx_set_cond(dsx_handle* h, const float* cond, dsx_strides cs, int B, int T, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_CHECK(cond, DSX_E_INVALID, "null tensor pointer");
  Geom g;
  DSX_TRY(prepare(h, cond, cs, B, T, 1, g, s));
  return check_status(h, s, "dsx_set_cond");
}

int dsx_plms_update(dsx_handle* h, float* x_out, const float* x_in, const float* const* eps, int mode, int t, int interval,
                    int B, int T, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_CHECK(h && h->loaded, DSX_E_STATE, "dsx_load_diffnet has not been called");
  DSX_CHECK(h->sched_T > 0, DSX_E_STATE, "dsx_set_schedule has not been called");
  DSX_CHECK(x_out && x_in && eps && eps[0], DSX_E_INVALID, "null tensor pointer");
  DSX_CHECK(mode >= 0 && mode <= 4 && interval > 0 && t >= 0 && t < h->sched_T && B > 0 && T > 0, DSX_E_INVALID,
            "bad dsx_plms_update arguments (mode %d, t %d, interval %d)", mode, t, interval);
  static const int n_eps[5] = {1, 2, 2, 3, 4};
  for (int i = 0; i < n_eps[mode]; ++i) DSX_CHECK(eps[i], DSX_E_INVALID, "mode %d needs %d eps tensors", mode, n_eps[mode]);
  DSX_CUDA(cudaSetDevice(h->device));
  const size_t mel = static_cast<size_t>(B) * h->m.M * T;
  return launch_plms_update(h, x_out, x_in, eps[0], n_eps[mode] > 1 ? eps[1] : nullptr, n_eps[mode] > 2 ? eps[2] : nullptr,
                            n_eps[mode] > 3 ? eps[3] : nullptr, plms_coefs(h, t, interval, mode), mel, s);
}

int dsx_sample_ddpm(dsx_handle* h, float* x_inout, const float* cond, dsx_strides cs, int B, int T, int t_start,
                    int n_steps, const float* noise, uint64_t seed, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_CHECK(x_inout, DSX_E_INVALID, "null tensor pointer");
  DSX_CHECK(h && h->sched_T > 0, DSX_E_STATE, "dsx_set_schedule has not been called");
  DSX_CHECK(n_steps > 0 && t_start <= h->sched_T && t_start - n_steps >= 0, DSX_E_INVALID,
            "steps t_start=%d n_steps=%d outside schedule of %d", t_start, n_steps, h->sched_T);
  Geom g;
  DSX_TRY(prepare(h, cond, cs, B, T, n_steps + 1, g, s));
  DSX_TRY(sample_ddpm_impl(h, x_inout, g, t_start, n_steps, noise, seed, s));
  return check_status(h, s, "dsx_sample_ddpm");
}

int dsx_sample_plms(dsx_handle* h, float* x_inout, const float* cond, dsx_strides cs, int B, int T, int t_start,
                    int interval, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_CHECK(x_inout, DSX_E_INVALID, "null tensor pointer");
  DSX_CHECK(h && h->sched_T > 0, DSX_E_STATE, "dsx_set_schedule has not been called");
  DSX_CHECK(interval > 0 && t_start > 0 && t_start <= h->sched_T, DSX_E_INVALID, "bad PLMS arguments");
  Geom g;
  const int rows = (t_start + interval - 1) / interval + 2;
  DSX_TRY(prepare(h, cond, cs, B, T, rows, g, s));
  DSX_TRY(sample_plms_impl(h, x_inout, g, t_start, interval, s));
  return check_status(h, s, "dsx_sample_plms");
}

int dsx_infer(dsx_handle* h, const float* cond, dsx_strides cs, const float* fs2_mel, const float* start_noise,
              const float* x_start, const float* step_noise, uint64_t seed, const int64_t* mel2ph,
              const float* spec_min, const float* spec_max, int B, int T, int K_step, int pndm_interval,
              float* mel_out, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_CHECK(cond && mel_out && spec_min && spec_max, DSX_E_INVALID, "null tensor pointer");
  DSX_CHECK(fs2_mel || x_start, DSX_E_INVALID, "need fs2_mel (shallow start) or x_start (gaussian start)");
  DSX_CHECK(h && h->sched_T > 0, DSX_E_STATE, "dsx_set_schedule has not been called");
  DSX_CHECK(K_step > 0 && K_step <= h->sched_T, DSX_E_INVALID, "K_step %d outside schedule of %d", K_step, h->sched_T);
  Geom g;
  const int rows = pndm_interval > 0 ? (K_step + pndm_interval - 1) / pndm_interval + 2 : K_step + 1;
  DSX_TRY(prepare(h, cond, cs, B, T, rows, g, s));
  const int M = h->m.M;
  const size_t mel = static_cast<size_t>(B) * M * T;
  float* x = h->ws.XSTATE;   // x_t, [B,1,M,T]
  int rc = DSX_OK;
  if (x_start) {
    cudaError_t e = cudaMemcpyAsync(x, x_start, mel * 4, cudaMemcpyDeviceToDevice, s);
    if (e != cudaSuccess) { set_error("copy of x_start failed: %s", cudaGetErrorString(e)); rc = DSX_E_CUDA; }
  } else {
    rc = launch_prologue(h, x, fs2_mel, start_noise, seed ^ 0x9E3779B97F4A7C15ull, spec_min, spec_max,
                         h->sched[DSX_SCH_SQRT_ALPHAS_CUMPROD][K_step - 1],
                         h->sched[DSX_SCH_SQRT_ONE_MINUS_ALPHAS_CUMPROD][K_step - 1], B, T, M, s);
  }
  if (rc == DSX_OK)
    rc = pndm_interval > 0 ? sample_plms_impl(h, x, g, K_step, pndm_interval, s)
                           : sample_ddpm_impl(h, x, g, K_step, K_step, step_noise, seed, s);
  if (rc == DSX_OK) rc = launch_epilogue(h, x, mel2ph, spec_min, spec_max, mel_out, B, T, M, s);
  if (rc == DSX_OK) rc = check_status(h, s, "dsx_infer");
  return rc;
}

int dsx_infer_host(dsx_handle* h, const float* cond_host, dsx_strides cs, const float* fs2_mel_host,
                   const float* x_start_host, uint64_t seed, const int64_t* mel2ph_host, const float* spec_min_host,
                   const float* spec_max_host, int B, int T, int K_step, int pndm_interval, float* mel_out_host,
                   void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_CHECK(h && h->loaded, DSX_E_STATE, "dsx_load_diffnet has not been called");
  DSX_CHECK(cond_host && mel_out_host && spec_min_host && spec_max_host, DSX_E_INVALID, "null host pointer");
  DSX_CUDA(cudaSetDevice(h->device));
  const int M = h->m.M, H = h->m.H;
  const size_t mel = static_cast<size_t>(B) * M * T;
  // the host cond tensor must be dense in some permutation of [B,H,T]; copy its full extent.  Device staging
  // buffers live in the handle (grow-only) so a call costs copies, not cudaMalloc / cudaFree.
  const size_t cond_elems = static_cast<size_t>(B) * H * T;
  DSX_CHECK(B > 0 && T > 0, DSX_E_INVALID, "B and T must be positive (got %d, %d)", B, T);
  DSX_CHECK(cs.b > 0 && cs.c > 0 && cs.t > 0 &&
                static_cast<size_t>((B - 1) * cs.b + (H - 1) * cs.c + (T - 1) * cs.t) + 1 == cond_elems,
            DSX_E_INVALID, "dsx_infer_host: cond_host must be a dense permutation of a contiguous [B,H,T] block (strides %lld %lld %lld)",
            static_cast<long long>(cs.b), static_cast<long long>(cs.c), static_cast<long long>(cs.t));
  int rc = DSX_OK;
  auto up = [&](int slot, const void* src, size_t bytes, bool copy = true) -> void* {
    if (rc != DSX_OK || (copy && !src)) return nullptr;
    GrowBuffer& b = h->stage[slot];
    rc = b.reserve(bytes, s);
    if (rc == DSX_OK && copy && cudaMemcpyAsync(b.ptr, src, bytes, cudaMemcpyHostToDevice, s) != cudaSuccess) {
      set_error("host->device copy failed");
      rc = DSX_E_CUDA;
    }
    return b.ptr;
  };
  float* d_cond = static_cast<float*>(up(0, cond_host, cond_elems * 4));
  float* d_fs2 = static_cast<float*>(up(1, fs2_mel_host, mel * 4));
  float* d_x = static_cast<float*>(up(2, x_start_host, mel * 4));
  float* d_min = static_cast<float*>(up(3, spec_min_host, M * 4));
  float* d_max = static_cast<float*>(up(4, spec_max_host, M * 4));
  int64_t* d_m2p = static_cast<int64_t*>(up(5, mel2ph_host, static_cast<size_t>(B) * T * 8));
  float* d_out = static_cast<float*>(up(6, nullptr, mel * 4, false));   // output buffer: no upload
  if (rc == DSX_OK)
    rc = dsx_infer(h, d_cond, cs, d_fs2, nullptr, d_x, nullptr, seed, d_m2p, d_min, d_max, B, T, K_step, pndm_interval,
                   d_out, stream);
  if (rc == DSX_OK && cudaMemcpyAsync(mel_out_host, d_out, mel * 4, cudaMemcpyDeviceToHost, s) != cudaSuccess) {
    set_error("device->host copy failed");
    rc = DSX_E_CUDA;
  }
  cudaStreamSynchronize(s);
  return rc;
}

int dsx_get_info(dsx_handle* h, int what, int64_t* out) {
  DSX_CHECK(h && out, DSX_E_INVALID, "null argument");
  switch (what) {
    case DSX_INFO_PRECISION: *out = h->precision; break;
    case DSX_INFO_KERNEL_LAUNCHES: *out = h->launches; break;
    case DSX_INFO_WORKSPACE_BYTES: *out = static_cast<int64_t>(h->ws.bytes()); break;
    case DSX_INFO_SM_COUNT: *out = h->sm_count; break;
    case DSX_INFO_TC_CTA_GROUP: *out = h->tc_group; break;
    case DSX_INFO_LAYER_KERNEL_LAUNCHES: *out = static_cast<int64_t>(h->prof_used / 2); break;
    case DSX_INFO_STACK_MODE: *out = h->stack_mode; break;
    case DSX_INFO_CLUSTER_OCCUPANCY: *out = h->step_occ[1] > 0 ? h->step_occ[1] : 0; break;
    case DSX_INFO_STACK_KERNEL_LAUNCHES: *out = h->stack_launches; break;
    case DSX_INFO_STACK_ROWS: *out = h->stack_rows_used; break;
    case DSX_INFO_LAYER_KERNEL_NS: {
      double total_ms = 0;
      for (size_t i = 0; i + 1 < h->prof_used; i += 2) {
        float ms = 0.f;
        DSX_CUDA(cudaEventSynchronize(h->prof_events[i + 1]));
        DSX_CUDA(cudaEventElapsedTime(&ms, h->prof_events[i], h->prof_events[i + 1]));
        total_ms += ms;
      }
      *out = static_cast<int64_t>(total_ms * 1e6);
      break;
    }
    default: set_error("unknown info %d", what); return DSX_E_INVALID;
  }
  return DSX_OK;
}

int dsx_set_option(dsx_handle* h, int what, int64_t value) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  switch (what) {
    case DSX_OPT_TC_CTA_GROUP:
      DSX_CHECK(value == 2, DSX_E_INVALID, "DSX_OPT_TC_CTA_GROUP only accepts 2 (kept for ABI compatibility)");
      DSX_CHECK(h->tc_group != 0, DSX_E_INVALID, "no tensor-core path on this device");
      break;
    case DSX_OPT_CP_PREFETCH: break;   // the step kernel's L2 prefetch is unconditional; results never depended on it
    case DSX_OPT_STACK_MODE: h->stack_mode = static_cast<int>(value); break;
    case DSX_OPT_STACK_KERNEL: h->stack_kernel = static_cast<int>(value); break;
    case DSX_OPT_GATE_APPROX: h->gate_approx = static_cast<int>(value); break;
    case DSX_OPT_FUSED_HEAD: h->fused_head = static_cast<int>(value); break;
    case DSX_OPT_STACK_ROWS:
      DSX_CHECK(value == 0 || value == 64 || value == 128, DSX_E_INVALID, "DSX_OPT_STACK_ROWS must be 0 (automatic), 64 or 128");
      h->stack_rows = static_cast<int>(value);
      break;
    case DSX_OPT_BATCH_OFFSET:
      DSX_CHECK(value >= 0 && value < (1ll << 30), DSX_E_INVALID, "DSX_OPT_BATCH_OFFSET out of range");
      h->batch_offset = static_cast<int>(value);
      break;
    case DSX_OPT_SR_SETS:
      DSX_CHECK(value >= 1 && value <= 1024, DSX_E_INVALID, "DSX_OPT_SR_SETS must be in [1, 1024]");
      h->sr_sets = static_cast<int>(value);
      break;
    case DSX_OPT_PROFILE:
      h->profile = static_cast<int>(value);
      h->prof_used = 0;
      break;
    default: set_error("unknown option %d", what); return DSX_E_INVALID;
  }
  return DSX_OK;
}

int dsx_debug_read(dsx_handle* h, int which, float* out, int B, int T, void* stream) {
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  DSX_CHECK(!(h && h->fft), DSX_E_STATE, "dsx_debug_read taps DiffNet buffers; the loaded denoiser is the FFT");
  DSX_CHECK(h && out && h->ws.X, DSX_E_STATE, "no workspace");
  DSX_CHECK(B == h->ws.g.B && T == h->ws.g.T, DSX_E_INVALID, "geometry mismatch");
  const float* src = which == 0 ? h->ws.X : h->ws.SKIP;
  const int C = h->m.C;
  DSX_CUDA(cudaMemcpy2DAsync(out, static_cast<size_t>(T) * C * 4, src, static_cast<size_t>(h->ws.g.Tp) * C * 4,
                             static_cast<size_t>(T) * C * 4, B, cudaMemcpyDeviceToDevice, s));
  return DSX_OK;
}

int dsx_debug_trace(dsx_handle* h, int enable, int64_t* out_host) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(!h->fft, DSX_E_STATE, "dsx_debug_trace records the DiffNet step kernel; the loaded denoiser is the FFT");
  DSX_CUDA(cudaSetDevice(h->device));
  const size_t bytes = static_cast<size_t>(2) * h->sm_count * DSX_TRACE_SLOTS * sizeof(int64_t);
  if (enable) {
    if (!h->trace_dev) DSX_CUDA(cudaMalloc(&h->trace_dev, bytes));
    DSX_CUDA(cudaMemset(h->trace_dev, 0, bytes));
    DSX_CUDA(cudaDeviceSynchronize());
    h->trace_on = true;
    return DSX_OK;
  }
  h->trace_on = false;
  if (out_host) {
    DSX_CHECK(h->trace_dev, DSX_E_STATE, "no trace recorded (enable it first)");
    DSX_CUDA(cudaDeviceSynchronize());
    DSX_CUDA(cudaMemcpy(out_host, h->trace_dev, bytes, cudaMemcpyDeviceToHost));
  }
  return DSX_OK;
}

int dsx_debug_set_layer_limit(dsx_handle* h, int n_layers) {
  DSX_CHECK(h, DSX_E_INVALID, "null handle");
  DSX_CHECK(!h->fft, DSX_E_STATE, "dsx_debug_set_layer_limit applies to DiffNet; the loaded denoiser is the FFT");
  h->layer_limit = n_layers;
  return DSX_OK;
}

}  // extern "C"
