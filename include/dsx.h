/*
 * dsx -- C ABI of the H100-native (sm_90a) DiffSinger reverse-diffusion sampler.
 *
 * The reference (MoonInTheRiver/DiffSinger) has no native boundary: the hot path is a Python
 * class surface.  This header is the boundary a binding would target;
 * each entry point names the reference interface it replaces (paths relative to the
 * reference tree).  Conventions:
 *   - plain pointers and sizes only; device pointers unless a parameter says "host";
 *   - every call returns 0 on success or a negative DSX_E_* code; dsx_last_error() gives a
 *     thread-local message; nothing throws across the ABI;
 *   - all GPU work is enqueued on the caller's stream (a cudaStream_t passed as void*);
 *     no internal threads; a handle belongs to one device and is not thread-safe;
 *   - the library owns only packed weights, step tables and workspace (freed by
 *     dsx_destroy); inputs are never modified except the documented in/out state.
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails
 *     with DSX_E_CUDA.
 */
#ifndef DSX_H_
#define DSX_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DSX_VERSION 100

enum {
  DSX_OK = 0,
  DSX_E_INVALID = -1,   /* bad argument / unsupported shape                      */
  DSX_E_CUDA = -2,      /* CUDA runtime / driver error (message has the string)  */
  DSX_E_STATE = -3,     /* call order: weights or schedule not loaded            */
  DSX_E_KERNEL = -4,    /* in-kernel watchdog or self-check tripped              */
  DSX_E_NOMEM = -5
};

/* Arithmetic of the contractions of each residual layer (usr/diff/net.py:66-78).  In the tensor-core modes the conditioner
 * projection -- it does not depend on the diffusion step -- is computed once per call with hi+lo operands and kept in
 * fp32; the modes differ in the dilated conv and the output projection. */
enum {
  DSX_PREC_FP32_SIMT = 0, /* fp32 CUDA-core path, any channel count                          */
  DSX_PREC_FP16 = 1,      /* wgmma f16, fp16 operands, fp32 accumulate (fast mode)           */
  DSX_PREC_FP16X2 = 2,    /* wgmma, weights as hi+lo fp16 pairs, running activations fp16: 2 MMA passes */
  DSX_PREC_FP16X3 = 3,    /* wgmma, hi+lo fp16 split of both operands, 3 MMAs (fp32-equivalent)*/
  DSX_PREC_FP16S = 4      /* wgmma, ONE MMA pass; the weights are rounded to fp16 stochastically into R sets
                             (DSX_OPT_SR_SETS, default 64) and evaluation j of a sampling loop uses set j % R, so the weight
                             rounding error is unbiased and decorrelated across diffusion steps instead of accumulating,
                             at half the MMA work of FP16X2 */
};

typedef struct dsx_handle dsx_handle;

/* Element strides of a logically [B, C, T] fp32 tensor (the reference hands the sampler
 * x[:,0] with strides (80T,1... or (80T,80,1,80)) and cond as a transposed view with strides
 * (256T,1,256); usr/diff/shallow_diffusion_tts.py:238,253-259). */
typedef struct {
  int64_t b, c, t;
} dsx_strides;

/* DiffNet parameters, fp32 device pointers, each tensor contiguous in the reference's own
 * state-dict layout (usr/diff/net.py:58-64, 91-104).  Per-layer arrays are HOST arrays of L
 * device pointers. */
typedef struct {
  const float* in_w;   /* input_projection.weight            [C, M, 1]  */
  const float* in_b;   /* input_projection.bias              [C]        */
  const float* mlp0_w; /* mlp.0.weight                       [4C, C]    */
  const float* mlp0_b; /* mlp.0.bias                         [4C]       */
  const float* mlp2_w; /* mlp.2.weight                       [C, 4C]    */
  const float* mlp2_b; /* mlp.2.bias                         [C]        */
  const float* const* dil_w;  /* residual_layers.l.dilated_conv.weight           [2C, C, 3] */
  const float* const* dil_b;  /* residual_layers.l.dilated_conv.bias             [2C]       */
  const float* const* dif_w;  /* residual_layers.l.diffusion_projection.weight   [C, C]     */
  const float* const* dif_b;  /* residual_layers.l.diffusion_projection.bias     [C]        */
  const float* const* cond_w; /* residual_layers.l.conditioner_projection.weight [2C, H, 1] */
  const float* const* cond_b; /* residual_layers.l.conditioner_projection.bias   [2C]       */
  const float* const* out_w;  /* residual_layers.l.output_projection.weight      [2C, C, 1] */
  const float* const* out_b;  /* residual_layers.l.output_projection.bias        [2C]       */
  const float* skip_w; /* skip_projection.weight             [C, C, 1]  */
  const float* skip_b; /* skip_projection.bias               [C]        */
  const float* fin_w;  /* output_projection.weight           [M, C, 1]  */
  const float* fin_b;  /* output_projection.bias             [M]        */
} dsx_diffnet_params;

/* Order of the schedule buffers for dsx_set_schedule == the registered buffers of
 * GaussianDiffusion.__init__ (usr/diff/shallow_diffusion_tts.py:101-123). */
enum {
  DSX_SCH_BETAS = 0,
  DSX_SCH_ALPHAS_CUMPROD,
  DSX_SCH_ALPHAS_CUMPROD_PREV,
  DSX_SCH_SQRT_ALPHAS_CUMPROD,
  DSX_SCH_SQRT_ONE_MINUS_ALPHAS_CUMPROD,
  DSX_SCH_LOG_ONE_MINUS_ALPHAS_CUMPROD,
  DSX_SCH_SQRT_RECIP_ALPHAS_CUMPROD,
  DSX_SCH_SQRT_RECIPM1_ALPHAS_CUMPROD,
  DSX_SCH_POSTERIOR_VARIANCE,
  DSX_SCH_POSTERIOR_LOG_VARIANCE_CLIPPED,
  DSX_SCH_POSTERIOR_MEAN_COEF1,
  DSX_SCH_POSTERIOR_MEAN_COEF2,
  DSX_SCH_COUNT
};

int dsx_version(void);
const char* dsx_last_error(void);

/* Handle: owns packed weights + workspace on `device`. */
int dsx_create(int device, dsx_handle** out);
void dsx_destroy(dsx_handle* h);

/* Replaces: DiffNet.__init__ / load_state_dict (usr/diff/net.py:82-105; checkpoint keys
 * model.denoise_fn.*, utils/__init__.py:178-203).  (Re)packs the weights for the selected
 * precision; call again after every load_state_dict / .to().  M mel bins, C residual
 * channels, H conditioner channels, L layers, dilation 2^(l % cycle).  M, C and H are multiples
 * of 16, M <= 768 and C <= 2448 (the fp32 kernels stage an input frame block and the step
 * embedding in the default 48 KB of shared memory; larger models are refused with DSX_E_INVALID
 * rather than opted in).  The tensor-core precisions take M = 80, C = H = 256 and cycle <= 4
 * only; DSX_PREC_FP32_SIMT takes any cycle. */
int dsx_load_diffnet(dsx_handle* h, const dsx_diffnet_params* p, int M, int C, int H, int L,
                     int dilation_cycle, int precision, void* stream);

/* Replaces: the schedule buffers registered in GaussianDiffusion.__init__
 * (usr/diff/shallow_diffusion_tts.py:90-123).  bufs: HOST array of DSX_SCH_COUNT HOST
 * pointers to fp32[T] -- the module's buffers verbatim, never recomputed from hparams. */
int dsx_set_schedule(dsx_handle* h, const float* const* bufs, int T);

/* Replaces: DiffNet.forward(spec, diffusion_step, cond) (usr/diff/net.py:107-130), or FFT.forward after dsx_load_fft:
 * one evaluation of the loaded denoiser, utterance b at diffusion step t[b].
 * x: [B,1,M,T] addressed through xs (b, c=mel bin, t); t: device int64[B];
 * cond: [B,H,T] through cs; eps out: contiguous [B,1,M,T]. */
int dsx_diffnet_forward(dsx_handle* h, const float* x, dsx_strides xs, const int64_t* t,
                        const float* cond, dsx_strides cs, float* eps, int B, int T, void* stream);

/* Conditioner of the following calls: packs cond [B,H,T] (any strides) and computes the step-independent
 * conditioner_projection of every residual layer (usr/diff/net.py:56,70) once.  Every entry point below that takes `cond`
 * does the same when the pointer is non-NULL and accepts cond == NULL to re-use the conditioner already set for the same
 * (B, T) -- for callers that drive the sampling loop themselves, one p_sample / p_sample_plms / DiffNet.forward per call
 * (usr/diff/shallow_diffusion_tts.py:159-204), so that the pack + projection are paid once per batch, not once per step. */
int dsx_set_cond(dsx_handle* h, const float* cond, dsx_strides cs, int B, int T, void* stream);

/* Replaces: the linear-multistep combination + get_x_pred of ONE p_sample_plms step
 * (usr/diff/shallow_diffusion_tts.py:174-199), fp32 in the reference's operation order, for callers that keep the eps
 * history themselves (self.noise_list).  eps: HOST array of device pointers, most recent first; all tensors contiguous
 * [B,1,M,T].  mode 0: x_out = phi(x_in, eps[0], t) (the warm-up prediction); 1: eps' = (eps[0] + eps[1]) / 2;
 * 2: (3 e0 - e1) / 2; 3: (23 e0 - 16 e1 + 5 e2) / 12; 4: (55 e0 - 59 e1 + 37 e2 - 9 e3) / 24; then x_out = phi(x_in, eps', t). */
int dsx_plms_update(dsx_handle* h, float* x_out, const float* x_in, const float* const* eps, int mode, int t,
                    int interval, int B, int T, void* stream);

/* Replaces: the DDPM loop `for i in reversed(range(0, t)): x = p_sample(x, i, cond)`
 * (usr/diff/shallow_diffusion_tts.py:159-166, 269-270): n_steps steps t_start-1 ... t_start-n_steps.
 * x_inout: contiguous [B,1,M,T], overwritten with the result.  noise: contiguous
 * [n_steps,B,1,M,T] consumed in execution order (noise[j] at t = t_start-1-j), or NULL
 * for the in-kernel Philox4x32-10 generator seeded by `seed`. */
int dsx_sample_ddpm(dsx_handle* h, float* x_inout, const float* cond, dsx_strides cs, int B, int T,
                    int t_start, int n_steps, const float* noise, uint64_t seed, void* stream);

/* Replaces: the PNDM loop `for i in reversed(range(0, t, interval)): x = p_sample_plms(...)`
 * (usr/diff/shallow_diffusion_tts.py:168-204, 261-267), history owned by the call. */
int dsx_sample_plms(dsx_handle* h, float* x_inout, const float* cond, dsx_strides cs, int B, int T,
                    int t_start, int interval, void* stream);

/* Replaces: the infer branch of GaussianDiffusion.forward after self.fs2
 * (usr/diff/shallow_diffusion_tts.py:248-275): norm_spec + q_sample(K_step-1) prologue (or a
 * gaussian start when fs2_mel == NULL and x_start != NULL), the sampling loop, and the
 * transpose + denorm_spec + (mel2ph > 0) mask epilogue.
 *   fs2_mel [B,T,M] contiguous (or NULL), start_noise [B,1,M,T] (or NULL -> Philox),
 *   x_start [B,1,M,T] (gaussian start; may be NULL), step_noise as in dsx_sample_ddpm,
 *   mel2ph device int64 [B,T] or NULL, spec_min/spec_max device fp32 [M],
 *   pndm_interval 0 = DDPM.  mel_out [B,T,M] contiguous. */
int dsx_infer(dsx_handle* h, const float* cond, dsx_strides cs, const float* fs2_mel,
              const float* start_noise, const float* x_start, const float* step_noise, uint64_t seed,
              const int64_t* mel2ph, const float* spec_min, const float* spec_max, int B, int T,
              int K_step, int pndm_interval, float* mel_out, void* stream);

/* Same as dsx_infer but every tensor pointer is a HOST pointer (pinned or pageable); the
 * copies to and from the device are issued on `stream` inside the call and the call returns
 * after mel_out_host is complete (it synchronises the stream). */
int dsx_infer_host(dsx_handle* h, const float* cond_host, dsx_strides cs, const float* fs2_mel_host,
                   const float* x_start_host, uint64_t seed, const int64_t* mel2ph_host,
                   const float* spec_min_host, const float* spec_max_host, int B, int T, int K_step,
                   int pndm_interval, float* mel_out_host, void* stream);

/* Introspection for tests / bench. */
int dsx_get_info(dsx_handle* h, int what, int64_t* out);
enum {
  DSX_INFO_PRECISION = 0,
  DSX_INFO_KERNEL_LAUNCHES = 1, /* kernels launched by this handle so far               */
  DSX_INFO_WORKSPACE_BYTES = 2,
  DSX_INFO_SM_COUNT = 3,
  DSX_INFO_TC_CTA_GROUP = 4,    /* 2 when the tensor-core (sm_90a) path is available on the device, else 0 */
  DSX_INFO_LAYER_KERNEL_NS = 5, /* DSX_OPT_PROFILE: summed device time of the residual-layer kernels since the
                                   option was set (CUDA events on the launching stream; synchronises)     */
  DSX_INFO_LAYER_KERNEL_LAUNCHES = 6, /* number of (start, stop) brackets = evaluations profiled */
  DSX_INFO_STACK_MODE = 7,
  DSX_INFO_CLUSTER_OCCUPANCY = 8, /* co-resident 128-frame CTAs of the step kernel on the device (0 before the first launch) */
  DSX_INFO_STACK_KERNEL_LAUNCHES = 9, /* one-launch-per-step launches (all layers + head, DSX_OPT_STACK_KERNEL) so far */
  DSX_INFO_STACK_ROWS = 10 /* frames per CTA of the last such launch: 128, or 64 for small batches */
};
/* Tuning knobs (tests exercise every variant): */
int dsx_set_option(dsx_handle* h, int what, int64_t value);
enum {
  DSX_OPT_TC_CTA_GROUP = 0, /* accepts 2 only; kept for ABI compatibility, no effect */
  DSX_OPT_CP_PREFETCH = 1,  /* accepted and ignored (kept for ABI compatibility): the step kernel always prefetches the
                               epilogue operands (conditioner projection, x, skip) into L2 */
  DSX_OPT_PROFILE = 2,      /* 1: bracket the residual-layer kernel(s) of every evaluation with CUDA events; 2: run the
                               tensor-core head of every evaluation (DDPM, PLMS, dsx_diffnet_forward) as a launch of its own
                               and bracket that instead; 0: off.  Setting it resets the sums */
  DSX_OPT_STACK_MODE = 3,   /* 1 (default): all residual layers of an evaluation in ONE persistent cooperative launch (a tile
                               starts a layer when its neighbour tiles have finished the one before); 0: one launch per
                               layer */
  DSX_OPT_STACK_KERNEL = 4, /* 1 (default): for FP16 / FP16X2 / FP16S the layers and the head of a step share ONE launch, with
                               64-frame CTAs for small batches and FP16S's stochastically rounded weight sets; 0: the layers use
                               the hi/lo weight planes at 128 frames per CTA (FP16S then runs the FP16X2 scheme) */
  DSX_OPT_SR_SETS = 5,      /* number of stochastically rounded weight sets of DSX_PREC_FP16S; set before dsx_load_diffnet */
  DSX_OPT_GATE_APPROX = 7,  /* gate sigmoid(g) * tanh(f) with tanh.approx.f32 (1) or with ex2 / rcp to ~2e-7 (0); -1 (default) =
                               1 except for FP16X3: its 2^-11 relative error is below the fp16 rounding of the gate output */
  DSX_OPT_FUSED_HEAD = 9,   /* 1 (default): the skip / output projections, the sampler update and the next input projection run
                               inside the layers' launch (one kernel per diffusion step); 0: a second launch */
  DSX_OPT_STACK_ROWS = 8,   /* frames per CTA of the one-launch-per-step form.  0 (default) = 64 whenever the batch then has a
                               resident CTA per 64-frame tile (small batches), else 128; 64 / 128 force it (results are bit-identical) */
  DSX_OPT_BATCH_OFFSET = 6  /* global index of this call's utterance 0: the in-kernel Philox noise of utterance b is drawn for
                               index (offset + b), so a batch sharded over ranks (one seed) reproduces the unsharded noise */
};

/* Debug taps for layer-by-layer parity (tests only): copies internal fp32 frames-major
 * buffers after a dsx_diffnet_forward.  which: 0 = residual stream after the last layer
 * executed, 1 = skip sum.  out: [B, T, C] contiguous. */
int dsx_debug_read(dsx_handle* h, int which, float* out, int B, int T, void* stream);
/* Phase timeline of the step kernel (k_hp_step).  enable = 1 clears the handle's trace buffer and makes every later
 * launch of the step kernel record into it; enable = 0 stops recording and, when out_host is not NULL, synchronises the
 * device and copies the buffer out.  Each launch overwrites the slots it reaches, so the buffer holds the last launch.
 * out_host: int64 [2 * DSX_INFO_SM_COUNT rows][DSX_TRACE_SLOTS], row = CTA (blockIdx.x), %globaltimer in ns, 0 = not
 * reached.  Thread 0 of each CTA stamps when it finishes a phase; a CTA that walks over several tiles of a layer
 * (more tiles than CTAs) overwrites the layer's slots, so they time its last tile only:
 *   slot 0                                launch entry
 *   slot 1 + 9 i + k, i = layer - l0      k = 0 / 2: GEMM1 chunk 0 / 1 end, 1 / 3: gate epilogue 0 / 1 end,
 *                                         4 / 6: GEMM2 residual / skip half end, 5 / 7: residual / skip epilogue end,
 *                                         8: end of the wait before the next layer (for the neighbour tiles and,
 *                                         between paired utterances, the partner tile) or before the head (0
 *                                         when nothing follows: the last layer of a launch without a head)
 *   slot 1 + 9 n + k, n = layers launched head: k = 0 H1 GEMM end, 1 H1 epilogue end, 2 H2 GEMM end, 3 mel update end,
 *                                         4 input projection GEMM end, 5 input projection epilogue end
 * Slots past DSX_TRACE_SLOTS are not recorded (at most 27 layers per launch). */
enum { DSX_TRACE_SLOTS = 256 };
int dsx_debug_trace(dsx_handle* h, int enable, int64_t* out_host);
/* Run only layers [0, n_layers) in the next dsx_diffnet_forward calls (<0: all). */
int dsx_debug_set_layer_limit(dsx_handle* h, int n_layers);

/* Hardware self-test of the encodings the tensor-core kernels rely on: the swizzled cp.async operand loads (row shifts,
 * zero fill outside [0, T)), the bulk copy of a pre-swizzled packed weight tile completing on an mbarrier, and the wgmma
 * shared-memory descriptors, on a small GEMM checked against a host product.
 * which = -1 or 0 runs it; returns 0 when it passes, otherwise DSX_E_KERNEL with the report in dsx_last_error().
 * report (may be NULL): host buffer receiving a text report. */
int dsx_selftest(int device, int which, char* report, int report_bytes);

/* ---- HiFi-GAN (NSF) vocoder: mel (+ f0) -> waveform --------------------------------------------------------------
 * Replaces: modules/hifigan/hifigan.py:104-171 (HifiGanGenerator with ResBlock1 / ResBlock2) and the NSF harmonic source
 * of modules/parallel_wavegan/models/source.py (SineGen, SourceModuleHnNSF), as vocoders/hifigan.py runs them.
 * Convolutions run on tensor cores with fp16 operands and fp32 accumulation; the residual stream, the multi-receptive-field
 * sum, the harmonic source and the output stay fp32.  A vocoder handle is independent of the sampler handles. */
typedef struct dsx_hifigan dsx_hifigan;

/* The generator's hyper-parameters (the `h` dict of HifiGanGenerator.__init__). */
typedef struct {
  int num_upsamples;                   /* len(upsample_rates): 1..4                                                     */
  int upsample_rates[4];               /* u_i >= 1                                                                      */
  int upsample_kernel_sizes[4];        /* k_i >= u_i, k_i % u_i == 0 and k_i - u_i even                                 */
  int upsample_initial_channel;        /* C0, divisible by 2^num_upsamples                                              */
  int resblock;                        /* 1 (ResBlock1: 3 dilated / plain conv pairs) or 2 (ResBlock2: 2 dilated convs) */
  int num_kernels;                     /* len(resblock_kernel_sizes): 1..3                                              */
  int resblock_kernel_sizes[3];        /* odd                                                                           */
  int resblock_dilation_sizes[3][3];   /* ResBlock2 uses the first two of each row                                      */
  int audio_sample_rate;               /* Hz, > 0                                                                       */
  int use_pitch_embed;                 /* 1: the NSF source and noise_convs exist (f0 may be passed to the forward)      */
} dsx_hifigan_config;

/* Parameters, fp32 device pointers, each tensor contiguous in the reference's state-dict layout.  A weight-normalised
 * conv passes weight_v as `*_w` and weight_g as `*_g`; a plain conv (after remove_weight_norm) passes `.weight` and
 * `*_g` = NULL.  Per-module arrays are HOST arrays of device pointers:
 *   ups_*:    num_upsamples entries (ups.i, ConvTranspose1d [C_in, C_out, k]);
 *   rb_*:     num_upsamples * num_kernels blocks in resblocks.* order, each block's convs in state-dict order --
 *             ResBlock1: convs1.0, convs1.1, convs1.2, convs2.0, convs2.1, convs2.2; ResBlock2: convs.0, convs.1;
 *   noise_*:  num_upsamples entries (noise_convs.i, plain Conv1d [C, 1, k]); NULL without use_pitch_embed. */
typedef struct {
  const float* conv_pre_w;
  const float* conv_pre_g;
  const float* conv_pre_b;
  const float* const* ups_w;
  const float* const* ups_g;
  const float* const* ups_b;
  const float* const* rb_w;
  const float* const* rb_g;
  const float* const* rb_b;
  const float* const* noise_w;
  const float* const* noise_b;
  const float* source_w;               /* m_source.l_linear.weight [1, 9] (use_pitch_embed) */
  const float* source_b;               /* m_source.l_linear.bias   [1]                      */
  const float* conv_post_w;
  const float* conv_post_g;
  const float* conv_post_b;
} dsx_hifigan_params;

/* Replaces: HifiGanGenerator(h).  Validates the configuration (DSX_E_INVALID). */
int dsx_hifigan_create(int device, const dsx_hifigan_config* cfg, dsx_hifigan** out);
void dsx_hifigan_destroy(dsx_hifigan* h);

/* Replaces: load_state_dict (+ remove_weight_norm).  Applies the weight norm g * v / ||v|| (norm over every dim but 0;
 * for ConvTranspose1d dim 0 is C_in) and packs fp16 tensor-core tiles.  Call again after every change of the weights. */
int dsx_hifigan_load(dsx_hifigan* h, const dsx_hifigan_params* p, void* stream);

/* Replaces: HifiGanGenerator.forward(mel, f0) as vocoders/hifigan.py:spec2wav calls it, one utterance at a time.
 *   mel      logically [B, 80, T], any element strides ms (dsx_infer's [B, T, 80] output feeds it untransposed);
 *   f0       [B, T] in Hz (0 = unvoiced), or NULL for the mel-only path (required NULL without use_pitch_embed);
 *   lengths  int32 [B] frames, or NULL for all T: utterance b is computed exactly as if it were alone at lengths[b]
 *            frames, and wav samples from lengths[b] * hop on are 0 (hop = product of the upsample rates);
 *   phase0   [B, 9] initial phases of the harmonics (harmonic 0 is always 0), or NULL: Philox4x32-10 uniforms of `seed`;
 *   src_noise [B, T * hop, 9] the source's additive gaussian noise, or NULL: Philox4x32-10 normals of `seed`;
 *   wav      [B, 1, T * hop] contiguous. */
int dsx_hifigan_forward(dsx_hifigan* h, const float* mel, dsx_strides ms, const float* f0, const int* lengths,
                        const float* phase0, const float* src_noise, uint64_t seed, int B, int T, float* wav,
                        void* stream);

/* ---- Parallel WaveGAN vocoder: noise + mel (+ coarse pitch) -> waveform ---------------------------------------------
 * Replaces: ParallelWaveGANGenerator (modules/parallel_wavegan/models/parallel_wavegan.py:21-191) with its
 * ConvInUpsampleNetwork (modules/parallel_wavegan/layers/upsample.py:16-183) and ResidualBlock
 * (modules/parallel_wavegan/layers/residual_block.py:15-129, eval mode), as vocoders/pwg.py runs them.  The residual
 * layers run on tensor cores with fp16 operands (the x taps, the upsampled conditioning, the gate output and the weights)
 * and fp32 accumulation; the conditioning network, the residual stream, the skip sum and the head stay fp32.  A PWG
 * handle is independent of the other handles. */
typedef struct dsx_pwg dsx_pwg;

/* The generator's hyper-parameters (ParallelWaveGANGenerator.__init__'s generator_params).  The kernels implement the
 * published widths only; anything else is DSX_E_INVALID ("unsupported ..."). */
typedef struct {
  int layers;               /* 1..64                                                        */
  int stacks;               /* layers % stacks == 0 and layers / stacks <= 16 (dilation 2^(l % (layers / stacks))) */
  int kernel_size;          /* 3                                                            */
  int residual_channels;    /* 64                                                           */
  int gate_channels;        /* 128                                                          */
  int skip_channels;        /* 64                                                           */
  int aux_channels;         /* 80                                                           */
  int aux_context_window;   /* w: 0..16 (conv_in has 2w + 1 taps)                           */
  int num_scales;           /* len(upsample_scales): 1..4                                   */
  int upsample_scales[4];   /* each 1..16; hop = their product <= 1024                      */
  int use_pitch_embed;      /* 1: pitch_embed and c_proj exist and the forward reads pitch   */
} dsx_pwg_config;

/* Parameters, fp32 device pointers, each tensor contiguous in the reference's state-dict layout.  A weight-normalised
 * conv passes weight_v as `*_w` and weight_g as `*_g`; a plain conv (after remove_weight_norm) passes `.weight` and
 * `*_g` = NULL.  Per-layer arrays are HOST arrays of device pointers:
 *   up_*:                     num_scales entries (upsample_net.upsample.up_layers.{2i + 1}, Conv2d [1, 1, 1, 2s + 1]);
 *   conv_*, aux_*, out_*, skip_*: `layers` entries (conv_layers.l.conv, .conv1x1_aux, .conv1x1_out, .conv1x1_skip).
 * A *_g array may be NULL as a whole.  pitch_embed and c_proj are NULL without use_pitch_embed. */
typedef struct {
  const float* first_w;        /* first_conv [64, 1, 1]                  */
  const float* first_g;
  const float* first_b;
  const float* conv_in_w;      /* upsample_net.conv_in [80, 80, 2w + 1]  */
  const float* conv_in_g;
  const float* const* up_w;
  const float* const* up_g;
  const float* const* conv_w;  /* [128, 64, 3]                           */
  const float* const* conv_g;
  const float* const* conv_b;
  const float* const* aux_w;   /* [128, 80, 1], no bias                  */
  const float* const* aux_g;
  const float* const* out_w;   /* [64, 64, 1]                            */
  const float* const* out_g;
  const float* const* out_b;
  const float* const* skip_w;  /* [64, 64, 1]                            */
  const float* const* skip_g;
  const float* const* skip_b;
  const float* last1_w;        /* last_conv_layers.1 [64, 64, 1]         */
  const float* last1_g;
  const float* last1_b;
  const float* last3_w;        /* last_conv_layers.3 [1, 64, 1]          */
  const float* last3_g;
  const float* last3_b;
  const float* pitch_embed;    /* pitch_embed.weight [300, 80]           */
  const float* c_proj_w;       /* c_proj.weight [80, 160]                */
  const float* c_proj_b;       /* c_proj.bias [80]                       */
} dsx_pwg_params;

/* Replaces: ParallelWaveGANGenerator(**generator_params) (parallel_wavegan.py:24-137).  Validates the configuration
 * (DSX_E_INVALID). */
int dsx_pwg_create(int device, const dsx_pwg_config* cfg, dsx_pwg** out);
void dsx_pwg_destroy(dsx_pwg* h);

/* Replaces: load_state_dict (+ remove_weight_norm, parallel_wavegan.py:174-189).  Applies the weight norm g * v / ||v||
 * (norm over every dim but 0) and packs the fp16 tensor-core tiles.  Call again after every change of the weights. */
int dsx_pwg_load(dsx_pwg* h, const dsx_pwg_params* p, void* stream);

/* Replaces: ParallelWaveGANGenerator.forward(x, c, pitch) (parallel_wavegan.py:139-172) as vocoders/pwg.py:82-103
 * (spec2wav) calls it.
 *   z      the noise [B, 1, T * hop], contiguous (hop = the product of upsample_scales);
 *   c      logically [B, 80, T + 2w], any element strides cs (spec2wav hands over a transposed view of the edge-padded
 *          mel);
 *   pitch  int64 [B, T + 2w], contiguous: the edge-padded coarse pitch.  Required with use_pitch_embed, where a value
 *          outside [0, 300) reads a zero embedding row; ignored (may be NULL) without, as the reference ignores it;
 *   wav    [B, 1, T * hop], contiguous.
 * B >= 1, T >= 1 and B * T * hop <= 2^25 samples, checked before any device access.  Each utterance of a batch gives the
 * same bits as that utterance alone (its convolutions are zero padded at its own edges), and repeated calls give the same
 * bits.  The workspace grows to the largest call: 928 bytes per output sample (fp32 x and skip sum, two fp16 copies of
 * x, the fp16 upsampled conditioning), plus 640 bytes per sample of the last upsampling stage's input (B * T * hop /
 * upsample_scales[num_scales - 1]), plus 320 bytes per padded frame with use_pitch_embed. */
int dsx_pwg_forward(dsx_pwg* h, const float* z, const float* c, dsx_strides cs, const int64_t* pitch, int B, int T,
                    float* wav, void* stream);

/* ---- Pitch extractor: mel -> f0 -------------------------------------------------------------------------------------
 * Replaces: PitchExtractor (modules/fastspeech/pe.py:119-149) with its Prenet (:7-41), ConvStacks (:81-116, GroupNorm),
 * PitchPredictor (modules/fastspeech/tts_modules.py:192-235, sinusoidal position embedding of
 * modules/commons/common_layers.py:88-143) and denorm_f0 (utils/pitch_utils.py:63-76), in eval mode, as
 * inference/svs/ds_e2e.py:26-45 runs it between the sampler and the vocoder.  Convolutions and linears run on tensor
 * cores with fp16 operands and fp32 accumulation; normalisations, the residual stream and the outputs are fp32.
 * A pitch-extractor handle is independent of the sampler and vocoder handles. */
typedef struct dsx_pe dsx_pe;

/* The hyper-parameters PitchExtractor reads (hparams + its constructor's conv_layers). */
typedef struct {
  int n_mel_bins;        /* 80                                                                          */
  int hidden;            /* hidden_size H: a multiple of 16 in [16, 256]                                */
  int predictor_hidden;  /* P (the reference's predictor_hidden, or H when that is <= 0): same range      */
  int predictor_kernel;  /* odd, <= 31                                                                  */
  int conv_layers;       /* mel_encoder GroupNorm conv blocks, 0..16 (0: no mel_encoder)                 */
  int causal;            /* ffn_padding: 0 'SAME', 1 'LEFT'                                             */
  int pitch_norm;        /* 0 'log' (f0 = 2^pred), 1 'standard' (f0 = pred * f0_std + f0_mean)           */
  float f0_mean, f0_std;
  int use_uv;            /* pitch_type == 'frame' and use_uv: f0 = 0 where pitch_pred[..., 1] > 0        */
} dsx_pe_config;

/* Parameters, fp32 device pointers, each tensor contiguous in the reference's state-dict layout.  Per-layer arrays are
 * HOST arrays of device pointers.  num_batches_tracked and embed_positions._float_tensor are not needed. */
typedef struct {
  const float* const* prenet_w;      /* mel_prenet.layers.i.0.weight [H, C_in, 5], i < 3, C_in = 80 then H           */
  const float* const* prenet_b;      /* mel_prenet.layers.i.0.bias [H]                                               */
  const float* const* bn_w;          /* mel_prenet.layers.i.2.weight [H] (BatchNorm1d)                               */
  const float* const* bn_b;          /* mel_prenet.layers.i.2.bias                                                   */
  const float* const* bn_mean;       /* mel_prenet.layers.i.2.running_mean                                           */
  const float* const* bn_var;        /* mel_prenet.layers.i.2.running_var                                            */
  const float* prenet_out_w;         /* mel_prenet.out_proj.weight [H, H]                                            */
  const float* prenet_out_b;
  const float* enc_in_w;             /* mel_encoder.in_proj.weight [H, H] (conv_layers > 0)                          */
  const float* enc_in_b;
  const float* const* enc_w;         /* mel_encoder.conv.i.conv.conv.weight [H, H, 5], i < conv_layers               */
  const float* const* enc_b;
  const float* const* gn_w;          /* mel_encoder.conv.i.norm.weight [H] (GroupNorm(H / 16, H))                    */
  const float* const* gn_b;
  const float* enc_out_w;            /* mel_encoder.out_proj.weight [H, H]                                           */
  const float* enc_out_b;
  const float* const* pred_w;        /* pitch_predictor.conv.i.1.weight [P, C_in, k], i < 5, C_in = H then P         */
  const float* const* pred_b;
  const float* const* ln_w;          /* pitch_predictor.conv.i.3.weight [P] (LayerNorm, eps 1e-12)                   */
  const float* const* ln_b;
  const float* linear_w;             /* pitch_predictor.linear.weight [2, P]                                         */
  const float* linear_b;             /* pitch_predictor.linear.bias [2]                                              */
  const float* pos_embed_alpha;      /* pitch_predictor.pos_embed_alpha [1]                                          */
} dsx_pe_params;

/* Replaces: PitchExtractor(n_mel_bins, conv_layers) under the global hparams.  Validates the configuration
 * (DSX_E_INVALID). */
int dsx_pe_create(int device, const dsx_pe_config* cfg, dsx_pe** out);
void dsx_pe_destroy(dsx_pe* h);

/* Replaces: load_state_dict (utils/__init__.py:load_ckpt of the pe_ckpt).  Packs fp16 tensor-core tiles and folds each
 * BatchNorm's running statistics and affine into a per-channel scale and shift.  Call again after every change of the
 * weights. */
int dsx_pe_load(dsx_pe* h, const dsx_pe_params* p, void* stream);

/* Replaces: PitchExtractor.forward(mel_input) (pe.py:135-149).
 *   mel         logically [B, T, 80], any element strides ms (b, c = bin, t): dsx_infer's mel_out as it is;
 *   pitch_pred  [B, T, 2] contiguous, or NULL;
 *   f0          [B, T] contiguous: f0_denorm_pred in Hz, 0 where uv says unvoiced and on padding frames, or NULL.
 * A frame is padding when all 80 bins are exactly 0 (pe.py:29, :143).  The batch is computed as given: GroupNorm
 * statistics and the position scan span all T frames of an utterance, padding included, exactly as in the reference, so
 * an utterance with a zero-padded tail is not the same as that utterance alone; utterances of equal T are independent. */
int dsx_pe_forward(dsx_pe* h, const float* mel, dsx_strides ms, int B, int T, float* pitch_pred, float* f0, void* stream);

/* ---- FastSpeech2 decoder: decoder_inp -> decoder output -------------------------------------------------------------
 * Replaces: FastspeechDecoder (modules/fastspeech/tts_modules.py:350-357), i.e. FFTBlocks.forward (:282-307) with the
 * sinusoidal position embedding (modules/commons/common_layers.py:88-143) and L EncSALayers (:542-588: LayerNorm,
 * bias-free MultiheadAttention with key padding mask, TransformerFFNLayer :486-522), in eval mode, as
 * FastSpeech2.forward runs it at inference (modules/fastspeech/fs2.py, FS_DECODERS['fft']).  GEMMs and the attention run
 * on tensor cores with fp16 operands and fp32 accumulation; the residual stream, LayerNorm statistics, the softmax state
 * and the output are fp32.  A decoder handle is independent of the other handles. */
typedef struct dsx_fs2dec dsx_fs2dec;

/* The hyper-parameters FastspeechDecoder reads (hidden_size, dec_layers, dec_ffn_kernel_size, num_heads, ffn_padding,
 * ffn_act). */
typedef struct {
  int hidden;            /* H: a multiple of 64 in [64, 256]                                    */
  int layers;            /* L: 1..64                                                            */
  int kernel;            /* ffn_1 kernel size k: odd for SAME, any k >= 1 for LEFT (k <= 255)   */
  int heads;             /* H / heads must be 64 or 128                                         */
  int padding;           /* ffn_padding: 0 'SAME' (k // 2 each side), 1 'LEFT' (k - 1 on the left) */
  int act;               /* ffn_act: 0 'gelu' (exact erf form), 1 'relu'                        */
} dsx_fs2dec_config;

/* Parameters, fp32 device pointers, each tensor contiguous in the reference's state-dict layout.  Per-layer arrays are
 * HOST arrays of L device pointers, entry i for layers.i.op.*.  embed_positions._float_tensor is not needed. */
typedef struct {
  const float* const* ln1_w;         /* layer_norm1.weight [H]                                                      */
  const float* const* ln1_b;         /* layer_norm1.bias [H]                                                        */
  const float* const* in_proj_w;     /* self_attn.in_proj_weight [3H, H] (no bias)                                  */
  const float* const* out_proj_w;    /* self_attn.out_proj.weight [H, H] (no bias)                                  */
  const float* const* ln2_w;         /* layer_norm2.weight [H]                                                      */
  const float* const* ln2_b;         /* layer_norm2.bias [H]                                                        */
  const float* const* ffn1_w;        /* ffn.ffn_1.weight (SAME) or ffn.ffn_1.1.weight (LEFT) [4H, H, k]             */
  const float* const* ffn1_b;        /* its bias [4H]                                                               */
  const float* const* ffn2_w;        /* ffn.ffn_2.weight [H, 4H]                                                    */
  const float* const* ffn2_b;        /* ffn.ffn_2.bias [H]                                                          */
  const float* ln_w;                 /* layer_norm.weight [H] (the final LayerNorm)                                 */
  const float* ln_b;                 /* layer_norm.bias [H]                                                         */
  const float* pos_embed_alpha;      /* pos_embed_alpha [1]                                                         */
} dsx_fs2dec_params;

/* Replaces: FastspeechDecoder(hidden_size, num_layers, kernel_size, num_heads) (tts_modules.py:351-356).  Validates the
 * configuration (DSX_E_INVALID, "unsupported ..."). */
int dsx_fs2dec_create(int device, const dsx_fs2dec_config* cfg, dsx_fs2dec** out);
void dsx_fs2dec_destroy(dsx_fs2dec* h);

/* Replaces: load_state_dict of the decoder's parameters (fs2.decoder.* of a FastSpeech2 checkpoint,
 * utils/__init__.py:178-203).  Packs fp16 tensor-core tiles.  Call again after every change of the weights. */
int dsx_fs2dec_load(dsx_fs2dec* h, const dsx_fs2dec_params* p, void* stream);

/* Replaces: FFTBlocks.forward(x) with padding_mask = attn_mask = None and return_hiddens = False (tts_modules.py:282-307).
 *   x    logically [B, T, H], any element strides xs (b, c = channel, t);
 *   out  [B, T, H] contiguous fp32.
 * A frame is padding when all H channels are exactly 0 (:288).  Nothing crosses utterances: each utterance of a batch,
 * padded tail included, gives the same bits as that utterance alone.  An utterance whose frames are all padding gives 0
 * (the reference's softmax over no key gives NaN there).  The workspace grows to the largest B * T seen. */
int dsx_fs2dec_forward(dsx_fs2dec* h, const float* x, dsx_strides xs, int B, int T, float* out, void* stream);

/* ---- FFT denoiser: the sampler handle's second denoiser ---------------------------------------------------------------
 * Replaces: FFT (usr/diff/candidate_decoder.py:35-100, DIFF_DECODERS['fft'] of usr/diffsinger_task.py:23-27), the
 * FastSpeech2 decoder stack run as the diffusion denoiser: eps = get_mel_out(FFTBlocks(get_decode_inp(
 * [input_projection(x_t), cond, mlp(emb(t))]))).  input_projection is folded into get_decode_inp at load time (in double),
 * so the entry GEMM has K = mel_bins; its operands, and those of the step-independent cond part, are hi+lo fp16 pairs
 * (fp32-equivalent).  The step part of get_decode_inp is an fp32 table per diffusion step.  The FFTBlocks stack is the
 * FastSpeech2 decoder's (fp16 operands, fp32 accumulation and residual stream); get_mel_out reads the final LayerNorm as an
 * fp16 operand and writes eps in fp32. */
typedef struct {
  dsx_fs2dec_config dec;   /* hidden_size, dec_layers, dec_ffn_kernel_size, num_heads, ffn_padding, ffn_act     */
  int residual_channels;   /* dim of input_projection and the step embedding: a multiple of 16 in [16, 1024]  */
  int mel_bins;            /* audio_num_mel_bins: 80 (get_mel_out is Linear(hidden_size, 80))                  */
} dsx_fft_config;

/* Parameters, fp32 device pointers in the reference's state-dict layout (dim = residual_channels, H = hidden). */
typedef struct {
  dsx_fs2dec_params dec;   /* the FFTBlocks stack: layers.*, layer_norm.*, pos_embed_alpha                     */
  const float* in_w;       /* input_projection.weight [dim, mel_bins, 1]                                      */
  const float* in_b;       /* input_projection.bias   [dim]                                                   */
  const float* mlp0_w;     /* mlp.0.weight [4 dim, dim]                                                       */
  const float* mlp0_b;     /* mlp.0.bias   [4 dim]                                                            */
  const float* mlp2_w;     /* mlp.2.weight [dim, 4 dim]                                                       */
  const float* mlp2_b;     /* mlp.2.bias   [dim]                                                              */
  const float* decode_inp_w; /* get_decode_inp.weight [H, dim + H + dim]: columns x | cond | step embedding   */
  const float* decode_inp_b; /* get_decode_inp.bias   [H]                                                     */
  const float* mel_out_w;  /* get_mel_out.weight [mel_bins, H]                                                */
  const float* mel_out_b;  /* get_mel_out.bias   [mel_bins]                                                   */
} dsx_fft_params;

/* Replaces: FFT(hidden_size, dec_layers, dec_ffn_kernel_size, num_heads) + load_state_dict as the denoise_fn of
 * GaussianDiffusion.  Validates like dsx_fs2dec_create plus residual_channels and mel_bins (DSX_E_INVALID,
 * "unsupported ..."); on failure the handle keeps what it held.  Replaces the handle's denoiser (DiffNet or FFT), as
 * dsx_load_diffnet replaces an FFT.  Afterwards dsx_diffnet_forward, dsx_set_cond, dsx_sample_ddpm, dsx_sample_plms,
 * dsx_plms_update, dsx_infer and dsx_infer_host run the FFT denoiser with unchanged meaning; DSX_INFO_PRECISION reports
 * DSX_PREC_FP16; the DiffNet-only options (STACK_*, FUSED_HEAD, SR_SETS, GATE_APPROX, PROFILE) are accepted and ignored;
 * dsx_debug_read, dsx_debug_trace and dsx_debug_set_layer_limit return DSX_E_STATE.  A padding frame (all H channels of
 * get_decode_inp's output exactly 0) gives eps = get_mel_out.bias. */
int dsx_load_fft(dsx_handle* h, const dsx_fft_config* cfg, const dsx_fft_params* p, void* stream);

/* ---- FastSpeech2 encoder: phoneme tokens -> encoder_out --------------------------------------------------------------
 * Replaces: FastspeechEncoder.forward(txt_tokens) (modules/fastspeech/tts_modules.py:310-347) and
 * FastspeechMIDIEncoder.forward(txt_tokens, midi_embedding, midi_dur_embedding, slur_embedding)
 * (modules/diffsinger_midi/fs2.py:11-36), in eval mode with use_pos_embed: the token embedding scaled by sqrt(H), the
 * MIDI addends, the position term, then FFTBlocks without pos_embed_alpha (tts_modules.py:282-307) whose padding mask is
 * txt_tokens == 0.  The layers are the FastSpeech2 decoder's (fp16 operands, fp32 accumulation, residual stream and
 * output).  An encoder handle is independent of the other handles. */
typedef struct dsx_fs2enc dsx_fs2enc;

typedef struct {
  dsx_fs2dec_config stack; /* hidden_size, enc_layers, enc_ffn_kernel_size, num_heads, ffn_padding, ffn_act: as the
                              decoder's                                                                         */
  int vocab;               /* rows of embed_tokens (len(dictionary)), >= 1                                      */
  int pos;                 /* 0: SinusoidalPositionalEmbedding over the tokens (common_layers.py:88-143), added;
                              1: RelPositionalEncoding (modules/commons/espnet_positional_embedding.py:91-113,
                              rel_pos: true): x = x * sqrt(H) + pe[t]                                           */
} dsx_fs2enc_config;

typedef struct {
  dsx_fs2dec_params stack; /* layers.*, layer_norm.*; pos_embed_alpha is not used (NULL)                        */
  const float* embed_w;    /* embed_tokens.weight [vocab, H]                                                    */
} dsx_fs2enc_params;

/* Replaces: FastspeechEncoder / FastspeechMIDIEncoder(embed_tokens, hidden_size, num_layers, kernel_size, num_heads).
 * Validates like dsx_fs2dec_create plus vocab and pos (DSX_E_INVALID, "unsupported ..."). */
int dsx_fs2enc_create(int device, const dsx_fs2enc_config* cfg, dsx_fs2enc** out);
void dsx_fs2enc_destroy(dsx_fs2enc* h);
/* Replaces: load_state_dict of encoder.* (embed_tokens is the shared encoder_embed_tokens).  Call again after every
 * change of the weights. */
int dsx_fs2enc_load(dsx_fs2enc* h, const dsx_fs2enc_params* p, void* stream);

/* Replaces: the encoder's forward.
 *   tokens   int64 [B, T] contiguous; 0 is padding.  A token outside [0, vocab) reads as a zero embedding row (the caller
 *            is expected to reject it first, as nn.Embedding does);
 *   add[i]   NULL or fp32 logically [B, T, H] with element strides as[i] (b, c = channel, t): midi_embedding,
 *            midi_dur_embedding, slur_embedding, added in that order after the scaled token embedding;
 *   rel_len  pos 1: the length P of the RelPositionalEncoding table (5000, or the largest T the module has seen when
 *            larger); row t of it holds position P - 1 - t.  Requires T <= P.  Ignored for pos 0;
 *   out      encoder_out [B, T, H] contiguous fp32; padding rows are 0.
 * Each utterance gives the same bits as that utterance alone at the same T; one whose tokens are all padding gives 0. */
int dsx_fs2enc_forward(dsx_fs2enc* h, const int64_t* tokens, int B, int T, const float* const* add, const dsx_strides* as,
                       int rel_len, float* out, void* stream);

/* ---- Duration predictor ----------------------------------------------------------------------------------------------
 * Replaces: DurationPredictor.forward / .inference (modules/fastspeech/tts_modules.py:59-151) with dur_loss 'mse', in eval
 * mode: n_layers x [ConstantPad1d + Conv1d, ReLU, LayerNorm over channels (eps 1e-12), * !mask], Linear(n_chans, 1),
 * * !mask, and out2dur.  The convolutions run on the pitch extractor's tensor-core conv kernel (fp16 operands, fp32
 * accumulation); LayerNorm, the linear head and out2dur are fp32 in the last convolution's epilogue. */
typedef struct dsx_durpred dsx_durpred;

typedef struct {
  int idim;              /* input channels: a multiple of 16 in [16, 256]                                       */
  int chans;             /* n_chans (predictor_hidden, or hidden_size when that is <= 0): same range            */
  int layers;            /* n_layers (dur_predictor_layers): 1..16                                              */
  int kernel;            /* kernel_size (dur_predictor_kernel): 1..31, odd for SAME                             */
  int padding;           /* 0 'SAME' ((k - 1) / 2 each side), 1 'LEFT' (k - 1 on the left)                      */
  float offset;          /* out2dur's offset (1.0)                                                              */
} dsx_durpred_config;

typedef struct {
  const float* const* conv_w;        /* conv.i.1.weight [chans, C_in, k], HOST array of n_layers device pointers  */
  const float* const* conv_b;        /* conv.i.1.bias [chans]                                                     */
  const float* const* ln_w;          /* conv.i.3.weight [chans]                                                   */
  const float* const* ln_b;          /* conv.i.3.bias [chans]                                                     */
  const float* linear_w;             /* linear.weight [1, chans]                                                  */
  const float* linear_b;             /* linear.bias [1]                                                           */
} dsx_durpred_params;

int dsx_durpred_create(int device, const dsx_durpred_config* cfg, dsx_durpred** out);
void dsx_durpred_destroy(dsx_durpred* h);
int dsx_durpred_load(dsx_durpred* h, const dsx_durpred_params* p, void* stream);

/* Replaces: DurationPredictor.forward(xs, x_masks) (-> xs) and .inference(xs, x_masks) (-> dur, xs).
 *   x     fp32 logically [B, T, idim], element strides xs_ (b, c = channel, t);
 *   mask  uint8 [B, T] contiguous, 1 = padding (the reference's src_padding);
 *   xs    [B, T] contiguous fp32: the log-domain prediction, 0 on padding rows;
 *   dur   [B, T] contiguous int64 or NULL: clamp(round_half_even(exp(xs) - offset), 0), 0 on padding rows. */
int dsx_durpred_forward(dsx_durpred* h, const float* x, dsx_strides xs_, const uint8_t* mask, int B, int T, float* xs,
                        int64_t* dur, void* stream);

/* ---- Duration predictor training step -------------------------------------------------------------------------------
 * Replaces: DurationPredictor._forward(xs, x_masks) (modules/fastspeech/tts_modules.py:106-120, dur_loss 'mse') in
 * training mode, and its autograd backward: the gradient of every parameter and of xs.  Layer i is ConstantPad1d + Conv1d,
 * ReLU, LayerNorm over channels (eps 1e-12), Dropout(p) (site i), * !mask; then Linear(chans, 1), * !mask.  Masks come
 * from Philox4x32-10 keyed by (seed, site, token, channel), as in the other training steps: the same seed and p give the
 * same masks, with torch's distribution (keep 1 - p, kept values scaled by 1 / (1 - p)) but not its stream.  The
 * convolutions run on dsx_durpred_forward's kernel with fp16 operands and fp32 accumulation; LayerNorm, the head and every
 * gradient are fp32.  At p = 0 the training forward's xs equals dsx_durpred_forward's bit for bit.  The backward scales its
 * fp16 gradient operands by a power of two S chosen on the device (S amax |d_xs * !mask| in [2^5, 2^6)) and divides it
 * out exactly, so 2^k d_xs gives exactly 2^k times every gradient and d_xs = 0 exact zeros.  Gradients are bitwise
 * reproducible (fixed-order reductions, no atomics).  No call allocates or synchronises the host: the tape and the
 * workspace are the caller's.  A handle is independent of the other handles. */
typedef struct dsx_durpred_train dsx_durpred_train;

/* Accepts what dsx_durpred_create accepts (DSX_E_INVALID, "unsupported ...").  offset is not used. */
int dsx_durpred_train_create(int device, const dsx_durpred_config* cfg, dsx_durpred_train** out);
void dsx_durpred_train_destroy(dsx_durpred_train* h);

/* Bytes of the tape of one forward over B utterances of T tokens (F = B T, P = chans, L = layers, each region rounded up
 * to 256 bytes, a256):
 *   a256(24) + a256(F) + a256(2 F idim) + L a256(4 F P) + (L - 1) a256(2 F P) + a256(4 F P)
 * the header (seed, p, B, T), a copy of the mask, each layer's fp16 input, each layer's LayerNorm input and the head's
 * input.  The masks are not stored: the backward draws them again from the seed and p the tape records. */
int dsx_durpred_train_tape_bytes(dsx_durpred_train* h, int B, int T, size_t* out);

/* Bytes of the scratch workspace a backward over (B, T) needs; it holds nothing between calls. */
int dsx_durpred_train_workspace_bytes(dsx_durpred_train* h, int B, int T, size_t* out);

/* One training forward: xs [B, T] contiguous fp32 (0 on padding tokens) of x (fp32, logically [B, T, idim], element
 * strides xs_: b, c = channel, t) and mask (uint8 [B, T] contiguous, 1 = padding), with dropout p_drop in [0, 1) drawn
 * from `seed`, and what the backward needs written to `tape` (at least dsx_durpred_train_tape_bytes).  The weights (fp32
 * device pointers, dsx_durpred_load's struct) are packed to fp16 inside the call, on the stream, into the handle, so
 * calls on one handle must not overlap on different streams.  The forward uses no workspace: workspace may be NULL and
 * workspace_bytes 0.  Several forwards may precede their backwards, each with its own tape. */
int dsx_durpred_train_forward(dsx_durpred_train* h, const dsx_durpred_params* w, const float* x, dsx_strides xs_,
                              const uint8_t* mask, int B, int T, float p_drop, uint64_t seed, void* tape,
                              size_t tape_bytes, void* workspace, size_t workspace_bytes, float* xs, void* stream);

/* The backward of the forward that wrote `tape`, with that forward's B and T and weights w: d_xs [B, T] contiguous.
 * Writes (does not accumulate) the fp32 gradient of every parameter through `grads` (same layout as w), and d_x
 * [B, T, idim] contiguous unless NULL: autograd's gradient of x, which is nonzero on a padding token within the
 * convolution's reach of a real one (the reference does not mask its input).  The tape is only read.  A (B, T) other than
 * the tape's makes every gradient NaN (checked on the device).  The call packs w's transposed convolutions into the
 * handle: calls on one handle must not overlap on different streams.  A scaled fp16 gradient operand beyond fp16's range
 * saturates at +-65504 rather than becoming inf. */
int dsx_durpred_train_backward(dsx_durpred_train* h, const dsx_durpred_params* w, const void* tape, const float* d_xs,
                               const dsx_durpred_params* grads, float* d_x, int B, int T, void* workspace,
                               size_t workspace_bytes, void* stream);

/* Test entry: the n_layers keep masks (1 kept, 0 dropped) that dsx_durpred_train_forward(seed, p_drop) draws, in site
 * (layer) order; out is a HOST array of n_layers device pointers to uint8 [B, T, chans]. */
int dsx_durpred_train_masks(dsx_durpred_train* h, uint64_t seed, float p_drop, int B, int T, uint8_t* const* out,
                            void* stream);

/* ---- Pitch and energy predictors -------------------------------------------------------------------------------------
 * Replaces: PitchPredictor.forward and EnergyPredictor.forward (modules/fastspeech/tts_modules.py:192-240), as
 * FastSpeech2.add_pitch / add_energy call them (modules/fastspeech/fs2.py:176-231): xs + pos_embed_alpha * table[pos]
 * with pos = make_positions(xs[..., 0], 0) (utils/__init__.py:145-157) and the sinusoidal table of
 * SinusoidalPositionalEmbedding(idim, 0) (modules/commons/common_layers.py:88-135, evaluated in fp32 without a size
 * limit, so T past its init_size needs no regrowth), then n_layers x [ConstantPad1d + Conv1d, ReLU, LayerNorm over
 * channels (eps 1e-12), Dropout], then Linear(chans, odim).  Nothing is masked: a padding frame gets what the reference
 * gives it.  The convolutions run on the duration predictor's tensor-core kernel (fp16 operands, fp32 accumulation);
 * the position term, LayerNorm and the head are fp32. */
typedef struct dsx_pitchpred dsx_pitchpred;

typedef struct {
  int idim;              /* input channels (hidden_size, or 128 behind the CWT Linear): a multiple of 16 in [16, 256] */
  int chans;             /* n_chans (predictor_hidden, or hidden_size when that is <= 0): same range                */
  int layers;            /* n_layers (predictor_layers): 1..16                                                      */
  int kernel;            /* kernel_size (predictor_kernel): 1..31, odd for SAME                                     */
  int padding;           /* 0 'SAME' ((k - 1) / 2 each side), 1 'LEFT' (k - 1 on the left)                          */
  int odim;              /* outputs of the head: 1..16 (2 for f0 and uv, 1 for energy or ph, 11 for CWT)            */
} dsx_pitchpred_config;

typedef struct {
  const float* const* conv_w;        /* conv.i.1.weight [chans, C_in, k], HOST array of n_layers device pointers  */
  const float* const* conv_b;        /* conv.i.1.bias [chans]                                                     */
  const float* const* ln_w;          /* conv.i.3.weight [chans]                                                   */
  const float* const* ln_b;          /* conv.i.3.bias [chans]                                                     */
  const float* linear_w;             /* linear.weight [odim, chans]                                               */
  const float* linear_b;             /* linear.bias [odim]                                                        */
  const float* pos_embed_alpha;      /* pos_embed_alpha [1]                                                       */
} dsx_pitchpred_params;

/* DSX_E_INVALID ("unsupported ...") for a configuration outside the ranges above. */
int dsx_pitchpred_create(int device, const dsx_pitchpred_config* cfg, dsx_pitchpred** out);
void dsx_pitchpred_destroy(dsx_pitchpred* h);
int dsx_pitchpred_load(dsx_pitchpred* h, const dsx_pitchpred_params* p, void* stream);

/* Replaces: PitchPredictor.forward(xs) in eval mode (tts_modules.py:222-235).
 *   x    fp32 [B, T, idim] contiguous;
 *   out  [B, T, odim] contiguous fp32.
 * The training forward's kernels with p = 0 and no tape: at p = 0 dsx_pitchpred_train_forward gives the same bits. */
int dsx_pitchpred_forward(dsx_pitchpred* h, const float* x, int B, int T, float* out, void* stream);

/* ---- Pitch and energy predictor training step ------------------------------------------------------------------------
 * Replaces: PitchPredictor.forward(xs) (tts_modules.py:222-235) in training mode, and its autograd backward: the gradient
 * of every parameter, pos_embed_alpha included, and of xs.  The forward is dsx_pitchpred_forward's with Dropout(p) at
 * site i after layer i's LayerNorm, the masks from Philox4x32-10 keyed by (seed, site, frame, channel) as in the other
 * training steps (torch's distribution, not its stream).  No gradient flows through the positions, which are integers:
 * d_x is the gradient at the first convolution's input, and d_pos_embed_alpha = sum over frames and channels of that
 * gradient times table[pos], summed in a fixed order.  The backward is the duration predictor step's with no mask and a
 * head of odim outputs: the fp16 gradient operands are scaled by a power of two S chosen on the device (S amax |d_out|
 * over all odim columns in [2^5, 2^6)) and divided out exactly, so 2^k d_out gives exactly 2^k times every gradient and
 * d_out = 0 exact zeros.  Gradients are written, not accumulated, and bitwise reproducible (fixed-order reductions, no
 * atomics).  No call allocates or synchronises the host: the tape and the workspace are the caller's.  Calls on one
 * handle must not overlap on different streams (the weights are packed into it). */
typedef struct dsx_pitchpred_train dsx_pitchpred_train;

/* Accepts what dsx_pitchpred_create accepts (DSX_E_INVALID, "unsupported ..."). */
int dsx_pitchpred_train_create(int device, const dsx_pitchpred_config* cfg, dsx_pitchpred_train** out);
void dsx_pitchpred_train_destroy(dsx_pitchpred_train* h);

/* Bytes of the tape of one forward over B utterances of T frames (F = B T, P = chans, L = layers, each region rounded up
 * to 256 bytes, a256):
 *   a256(24) + a256(4 F) + a256(2 F idim) + L a256(4 F P) + (L - 1) a256(2 F P) + a256(4 F P)
 * the header (seed, p, B, T), the int32 positions, each layer's fp16 input (layer 0's is x plus the position term), each
 * layer's LayerNorm input and the head's input.  The masks are not stored: the backward draws them again from the seed
 * and p the tape records. */
int dsx_pitchpred_train_tape_bytes(dsx_pitchpred_train* h, int B, int T, size_t* out);

/* Bytes of the scratch workspace a backward over (B, T) needs; it holds nothing between calls. */
int dsx_pitchpred_train_workspace_bytes(dsx_pitchpred_train* h, int B, int T, size_t* out);

/* One training forward: out [B, T, odim] contiguous fp32 of x (fp32 [B, T, idim] contiguous), with dropout p_drop in
 * [0, 1) drawn from `seed`, and what the backward needs written to `tape` (at least dsx_pitchpred_train_tape_bytes).
 * The forward uses no workspace: workspace may be NULL and workspace_bytes 0.  Several forwards may precede their
 * backwards, each with its own tape. */
int dsx_pitchpred_train_forward(dsx_pitchpred_train* h, const dsx_pitchpred_params* w, const float* x, int B, int T,
                                float p_drop, uint64_t seed, void* tape, size_t tape_bytes, void* workspace,
                                size_t workspace_bytes, float* out, void* stream);

/* The backward of the forward that wrote `tape`, with that forward's B and T and weights w: d_out [B, T, odim]
 * contiguous.  Writes the fp32 gradient of every parameter through `grads` (same layout as w), and d_x [B, T, idim]
 * contiguous unless NULL.  The tape is only read.  A (B, T) other than the tape's makes every gradient NaN (checked on
 * the device).  A scaled fp16 gradient operand beyond fp16's range saturates at +-65504 rather than becoming inf. */
int dsx_pitchpred_train_backward(dsx_pitchpred_train* h, const dsx_pitchpred_params* w, const void* tape,
                                 const float* d_out, const dsx_pitchpred_params* grads, float* d_x, int B, int T,
                                 void* workspace, size_t workspace_bytes, void* stream);

/* Test entry: the n_layers keep masks (1 kept, 0 dropped) that dsx_pitchpred_train_forward(seed, p_drop) draws, in site
 * (layer) order; out is a HOST array of n_layers device pointers to uint8 [B, T, chans]. */
int dsx_pitchpred_train_masks(dsx_pitchpred_train* h, uint64_t seed, float p_drop, int B, int T, uint8_t* const* out,
                              void* stream);

/* ---- Length regulator ------------------------------------------------------------------------------------------------
 * Replaces: LengthRegulator.forward(dur, dur_padding, alpha) (modules/fastspeech/tts_modules.py:159-189) in two calls,
 * because T_mel depends on the data, without its [B, T_txt, T_mel] temporaries.  Both run on the current device.
 *
 * dsx_length_totals: d = round_half_even(float(dur) * alpha) * !pad (pad: uint8 [B, T] or NULL), cum [B, T] int64 its
 * inclusive prefix sum per utterance, totals [B + 1] int64: totals[b] = cum[b, T - 1], totals[B] = 1 when any d < 0
 * (else 0).  One small copy of totals to the host gives T_mel = max totals[b] and the error flag.
 * dsx_length_regulate: mel2ph [B, T_mel] int64: for frame f < totals[b], the 1-based index of the token whose
 * [cum - d, cum) holds f; 0 from totals[b] on.  Bit-identical to the reference for non-negative d. */
int dsx_length_totals(const int64_t* dur, const uint8_t* pad, int B, int T, float alpha, int64_t* cum, int64_t* totals,
                      void* stream);
int dsx_length_regulate(const int64_t* cum, const int64_t* totals, int B, int T, int T_mel, int64_t* mel2ph,
                        void* stream);

/* ---- DiffNet training step: forward with a saved tape, and backward --------------------------------------------------
 * Replaces: DiffNet.forward (usr/diff/net.py:107-130) under autograd, as GaussianDiffusion.p_losses
 * (usr/diff/shallow_diffusion_tts.py:213-231) calls it in training, and its backward: the gradient of every DiffNet
 * parameter and of cond (not of spec).  q_sample, the loss and the optimizer stay with the caller.  GEMMs run on tensor
 * cores with fp16 operands and fp32 accumulation; the residual stream, the skip sum, eps and every gradient are fp32.
 * The backward scales its fp16 gradient operands by a power of two S chosen on the device from amax |d_eps| (S amax in
 * [2^5, 2^6), leaving about 2^10 of fp16 range above the largest scaled operand) and divides it out exactly, so the gradients for 2^k d_eps are exactly 2^k times those for d_eps, and
 * d_eps = 0 gives exact zeros.  Gradients are bitwise reproducible (fixed-order reductions, no atomics).  No call
 * synchronises the host or allocates: the tape and the scratch workspace are the caller's.  A training handle is independent of the other handles. */
typedef struct dsx_train dsx_train;

typedef struct {
  int M;                   /* in_dims: 80                                     */
  int C;                   /* residual_channels: 256                          */
  int H;                   /* hidden_size (cond channels): 256                */
  int L;                   /* residual_layers: 1..1024                        */
  int dilation_cycle;      /* dilation_cycle_length: 1..24, dilation 2^(l % cycle) */
} dsx_train_config;

/* Validates the configuration (DSX_E_INVALID). */
int dsx_train_create(int device, const dsx_train_config* cfg, dsx_train** out);
void dsx_train_destroy(dsx_train* h);

/* Bytes of the tape of one forward over B utterances of T frames (F = B T), each region rounded up to 256 bytes
 * (a256): a256(160 F) + a256(512 F) x 4 + a256(1024 B) + a256(9216 B) + L x (a256(512 F) x 2 + a256(1024 F)). */
int dsx_train_tape_bytes(dsx_train* h, int B, int T, size_t* out);

/* Bytes of the scratch workspace a forward or a backward over (B, T) needs.  The caller owns it (so a framework's
 * allocator sees and reuses it); it holds nothing between calls, and calls that may overlap need separate workspaces. */
int dsx_train_workspace_bytes(dsx_train* h, int B, int T, size_t* out);

/* One forward: eps [B,1,M,T] (contiguous) of spec [B,1,M,T] (through ss: b, c = mel bin, t), t device int64 [B], cond
 * [B,H,T] (through cs), with the activations the backward needs written to `tape` (caller-owned device memory of at
 * least dsx_train_tape_bytes) and `workspace` (at least dsx_train_workspace_bytes) as scratch.  B <= 65535,
 * B T <= 2^24 and L B T < 2^26 (DSX_E_INVALID otherwise).  The weights
 * (dsx_load_diffnet's pointer struct) are packed to fp16 inside the call, on the stream; the backward uses the packs of
 * the latest forward on the handle, so the weights must not change between a forward and the backward of its tape.
 * Several forwards may precede their backwards, each with its own tape. */
int dsx_train_forward(dsx_train* h, const dsx_diffnet_params* w, const float* spec, dsx_strides ss, const int64_t* t,
                      const float* cond, dsx_strides cs, int B, int T, void* tape, size_t tape_bytes, void* workspace,
                      size_t workspace_bytes, float* eps, void* stream);

/* The backward of the forward that wrote `tape` (same B, T): d_eps [B,1,M,T] contiguous.  Writes (does not accumulate)
 * the fp32 gradient of every parameter through `grads` (same layout as w), and d_cond [B,H,T] contiguous unless NULL.
 * The tape is only read; `workspace` (at least dsx_train_workspace_bytes) is scratch. */
int dsx_train_backward(dsx_train* h, const dsx_diffnet_params* w, const void* tape, const float* d_eps,
                       const dsx_diffnet_params* grads, float* d_cond, int B, int T, void* workspace,
                       size_t workspace_bytes, void* stream);

/* ---- FastSpeech2 decoder training step ------------------------------------------------------------------------------
 * Replaces: FFTBlocks.forward(x) of FastspeechDecoder in training mode (tts_modules.py:282-307, EncSALayer of
 * common_layers.py:542-588) and its autograd backward.  Dropout p at the reference's 1 + 3 L sites, in this order: site
 * 0 after x + alpha * positions (before * !pad); per layer i, site 1 + 3 i after out_proj, 2 + 3 i after the FFN
 * activation ([B, T, 4H]) and 3 + 3 i after ffn_2; attention probabilities have none (attention_dropout = 0).  Masks come
 * from Philox4x32-10 keyed by (seed, site, frame, channel): the same seed and p give the same masks, with torch's
 * distribution (keep 1 - p, kept values scaled by 1 / (1 - p)) but not its stream.  fp16 operands, fp32 accumulation,
 * LayerNorm statistics, softmax state and residual streams; the backward's fp16 operands are scaled by a power of two S
 * chosen on the device (S amax |d_out| in [2^5, 2^6)), divided out exactly, so 2^k d_out gives exactly 2^k times the
 * gradients.  Gradients are bitwise reproducible (fixed-order reductions, no atomics).  No call allocates or synchronises
 * the host: the tape and the workspace are the caller's.  A handle is independent of the other handles. */
typedef struct dsx_fs2dec_train dsx_fs2dec_train;

/* Accepts what dsx_fs2dec_create accepts (DSX_E_INVALID, "unsupported ..."). */
int dsx_fs2dec_train_create(int device, const dsx_fs2dec_config* cfg, dsx_fs2dec_train** out);
void dsx_fs2dec_train_destroy(dsx_fs2dec_train* h);

/* Bytes of the tape of one forward over B utterances of T frames (F = B T, H = hidden, L = layers, each region rounded
 * up to 256 bytes, a256):
 *   a256(24) + a256(F) + a256(4 F) + (2 L + 1) a256(4 F H) + L (6 a256(2 F H) + a256(4 F heads) + 2 a256(8 F H)).
 * The masks are not stored: the backward draws them again from the seed and p the tape records. */
int dsx_fs2dec_train_tape_bytes(dsx_fs2dec_train* h, int B, int T, size_t* out);

/* Bytes of the scratch workspace a forward or a backward over (B, T) needs; it holds nothing between calls. */
int dsx_fs2dec_train_workspace_bytes(dsx_fs2dec_train* h, int B, int T, size_t* out);

/* One training forward: out [B, T, H] contiguous fp32 of x (logically [B, T, H], any strides xs: b, c = channel, t), with
 * dropout p_drop in [0, 1) drawn from `seed`, and what the backward needs written to `tape` (at least
 * dsx_fs2dec_train_tape_bytes).  The weights (fp32 device pointers, pos_embed_alpha required) are packed to fp16 inside
 * the call, on the stream; the backward uses the packs of the latest forward on the handle, so the weights must not
 * change between a forward and the backward of its tape.  Several forwards may precede their backwards, each with its
 * own tape. */
int dsx_fs2dec_train_forward(dsx_fs2dec_train* h, const dsx_fs2dec_params* w, const float* x, dsx_strides xs, int B,
                             int T, float p_drop, uint64_t seed, void* tape, size_t tape_bytes, void* workspace,
                             size_t workspace_bytes, float* out, void* stream);

/* The backward of the forward that wrote `tape`, with that forward's B and T: d_out [B, T, H] contiguous.  Writes (does
 * not accumulate) the fp32 gradient of every parameter through `grads` (same layout as w, pos_embed_alpha included), and
 * d_x [B, T, H] contiguous (the gradient of decoder_inp; 0 on padding frames) unless NULL.  The tape is only read.  A
 * (B, T) other than the tape's makes every gradient NaN (checked on the device).  The backward reads the handle's packs
 * of the latest forward: a forward of other weights, on any stream, must not run before or during it. */
int dsx_fs2dec_train_backward(dsx_fs2dec_train* h, const dsx_fs2dec_params* w, const void* tape, const float* d_out,
                              const dsx_fs2dec_params* grads, float* d_x, int B, int T, void* workspace,
                              size_t workspace_bytes, void* stream);

/* Test entry: the 1 + 3 L keep masks (1 kept, 0 dropped) that dsx_fs2dec_train_forward(seed, p_drop) draws, in site
 * order; out is a HOST array of 1 + 3 L device pointers to uint8 [B, T, H] (sites 2 + 3 i: [B, T, 4H]).  It lets tests
 * rebuild the same forward in fp32 autograd. */
int dsx_fs2dec_train_masks(dsx_fs2dec_train* h, uint64_t seed, float p_drop, int B, int T, uint8_t* const* out,
                           void* stream);

/* ---- FastSpeech2 encoder training step ------------------------------------------------------------------------------
 * Replaces: FastspeechEncoder.forward(txt_tokens) (modules/fastspeech/tts_modules.py:310-347) and
 * FastspeechMIDIEncoder.forward(txt_tokens, midi_embedding, midi_dur_embedding, slur_embedding)
 * (modules/diffsinger_midi/fs2.py:11-36) in training mode, and their autograd backward: the gradient of every encoder
 * parameter, embed_tokens.weight included, and of the MIDI addends.  The forward is dsx_fs2enc_forward's with dropout:
 *   x = sqrt(H) E[tok] (+ midi_embedding + midi_dur_embedding + slur_embedding, left to right)
 *       + positions (pos 0)  |  x * sqrt(H) + pe[t] (pos 1, RelPositionalEncoding, whose own dropout has p = 0)
 *   x = dropout(x) (site 0), then FFTBlocks without pos_embed_alpha, padding mask txt_tokens == 0.
 * Dropout is the decoder training step's: the same 1 + 3 L sites (site 0 above; per layer i, 1 + 3 i after out_proj,
 * 2 + 3 i after the FFN activation, 3 + 3 i after ffn_2), the same (seed, site, frame, channel) keying and the same p, so
 * dsx_fs2dec_train_masks on a dsx_fs2dec_train handle of cfg.stack returns exactly the masks of a forward with that seed
 * and p.  The layers are the decoder step's (fp16 operands, fp32 accumulation, LayerNorm statistics, softmax state and
 * residual stream).  The backward's fp16 operands are scaled by a power of two chosen on the device (from amax |d_out|)
 * and divided out exactly, and the embedding gradient is that fp32 result times sqrt(H), so 2^k d_out gives exactly 2^k
 * times every gradient and d_out = 0 exact zeros.  Gradients are bitwise reproducible: the embedding gradient sums each
 * row's frames in a fixed order (a sort of the frames by token, then per-row sums; no atomics), at a cost that grows
 * with B T and with vocab, not with their product.  No call allocates or synchronises the host: the tape and the
 * workspace are the caller's.  A handle is independent of the other handles. */
typedef struct dsx_fs2enc_train dsx_fs2enc_train;

/* Accepts what dsx_fs2enc_create accepts (DSX_E_INVALID, "unsupported ..."). */
int dsx_fs2enc_train_create(int device, const dsx_fs2enc_config* cfg, dsx_fs2enc_train** out);
void dsx_fs2enc_train_destroy(dsx_fs2enc_train* h);

/* Bytes of the tape of one forward over B utterances of T tokens (F = B T, each region rounded up to 256 bytes, a256):
 *   D + a256(8 F)
 * with D = dsx_fs2dec_train_tape_bytes of cfg.stack, whose tape comes first; the second region is a copy of the tokens,
 * so the backward reads nothing the caller may have changed since the forward. */
int dsx_fs2enc_train_tape_bytes(dsx_fs2enc_train* h, int B, int T, size_t* out);

/* Bytes of the scratch workspace a forward or a backward over (B, T) needs; it holds nothing between calls. */
int dsx_fs2enc_train_workspace_bytes(dsx_fs2enc_train* h, int B, int T, size_t* out);

/* One training forward: out [B, T, H] contiguous fp32 from tokens, add, as and rel_len as dsx_fs2enc_forward takes them,
 * with dropout p_drop in [0, 1) drawn from `seed`, and what the backward needs written to `tape` (at least
 * dsx_fs2enc_train_tape_bytes).  The weights (fp32 device pointers; pos_embed_alpha not used) are packed to fp16 inside
 * the call, on the stream; the backward uses the packs of the latest forward on the handle, so the weights must not
 * change between a forward and the backward of its tape.  Several forwards may precede their backwards, each with its
 * own tape. */
int dsx_fs2enc_train_forward(dsx_fs2enc_train* h, const dsx_fs2enc_params* w, const int64_t* tokens, int B, int T,
                             const float* const* add, const dsx_strides* as, int rel_len, float p_drop, uint64_t seed,
                             void* tape, size_t tape_bytes, void* workspace, size_t workspace_bytes, float* out,
                             void* stream);

/* The backward of the forward that wrote `tape`, with that forward's B and T: d_out [B, T, H] contiguous.  Writes (does
 * not accumulate) the fp32 gradient of every stack parameter through grads->stack (pos_embed_alpha not written) and
 * grads->embed_w [vocab, H], every row: rows no token of the tape uses, and row 0 (padding_idx), are 0.  d_add, unless
 * NULL, is [B, T, H] contiguous: the gradient of the sum of the addends, so of each addend (0 on padding tokens).  The
 * tape is only read.  A (B, T) other than the tape's makes every gradient NaN (checked on the device).  The backward
 * reads the handle's packs of the latest forward: a forward of other weights, on any stream, must not run before or
 * during it. */
int dsx_fs2enc_train_backward(dsx_fs2enc_train* h, const dsx_fs2enc_params* w, const void* tape, const float* d_out,
                              const dsx_fs2enc_params* grads, float* d_add, int B, int T, void* workspace,
                              size_t workspace_bytes, void* stream);

/* ---- FFT denoiser training step -------------------------------------------------------------------------------------
 * Replaces: FFT.forward(spec, diffusion_step, cond) (usr/diff/candidate_decoder.py:50-100) in training mode, as
 * GaussianDiffusion.p_losses calls it with diff_decoder_type 'fft', and its autograd backward: the gradient of every
 * parameter and of cond (not of spec).  The entry and exit are dsx_load_fft's (input_projection folded into
 * get_decode_inp in double, hi+lo fp16 operands for x_t and cond, the step embedding in fp32); the FFTBlocks stack is the
 * decoder training step's, with its dropout: the same 1 + 3 L sites, the same (seed, site, frame, channel) keying and the
 * same p, so dsx_fs2dec_train_masks on a dsx_fs2dec_train handle of the same dsx_fs2dec_config returns exactly the masks
 * of a forward with that seed and p.  The backward's fp16 operands are scaled by powers of two chosen on the device
 * (from amax |d_eps|, then from amax |d decoder_inp|) and divided out exactly, so 2^k d_eps gives exactly 2^k times the
 * gradients and d_eps = 0 exact zeros.  Gradients are bitwise reproducible (fixed-order reductions, no atomics).  No call
 * allocates or synchronises the host: the tape and the workspace are the caller's.  A handle is independent of the other
 * handles. */
typedef struct dsx_fft_train dsx_fft_train;

/* Accepts what dsx_load_fft accepts (DSX_E_INVALID, "unsupported ..."). */
int dsx_fft_train_create(int device, const dsx_fft_config* cfg, dsx_fft_train** out);
void dsx_fft_train_destroy(dsx_fft_train* h);

/* Bytes of the tape of one forward over B utterances of T frames (F = B T, H = hidden, dim = residual_channels, each
 * region rounded up to 256 bytes, a256):
 *   D + a256(4 B dim) + a256(36 B dim) + a256(480 F) + a256(6 F H) + a256(2 F H)
 * with D = dsx_fs2dec_train_tape_bytes of the stack's configuration, whose tape comes first. */
int dsx_fft_train_tape_bytes(dsx_fft_train* h, int B, int T, size_t* out);

/* Bytes of the scratch workspace a forward or a backward over (B, T) needs; it holds nothing between calls. */
int dsx_fft_train_workspace_bytes(dsx_fft_train* h, int B, int T, size_t* out);

/* One training forward: eps [B,1,80,T] contiguous fp32 of spec [B,1,80,T] (through ss: b, c = mel bin, t), t device
 * int64 [B] and cond [B,H,T] (through cs), with dropout p_drop in [0, 1) drawn from `seed` and what the backward needs
 * written to `tape` (at least dsx_fft_train_tape_bytes).  The weights (fp32 device pointers, dsx_load_fft's struct,
 * pos_embed_alpha required) are packed inside the call, on the stream; the backward uses the packs of the latest forward
 * on the handle, so the weights must not change between a forward and the backward of its tape.  Several forwards may
 * precede their backwards, each with its own tape. */
int dsx_fft_train_forward(dsx_fft_train* h, const dsx_fft_params* w, const float* spec, dsx_strides ss,
                          const int64_t* t, const float* cond, dsx_strides cs, int B, int T, float p_drop,
                          uint64_t seed, void* tape, size_t tape_bytes, void* workspace, size_t workspace_bytes,
                          float* eps, void* stream);

/* The backward of the forward that wrote `tape`, with that forward's B and T: d_eps [B,1,80,T] contiguous.  Writes (does
 * not accumulate) the fp32 gradient of every parameter through `grads` (same layout as w, pos_embed_alpha included), and
 * d_cond unless NULL, frames-major [B, T, H] contiguous (the [B, H, T] gradient of cond, transposed).  The tape is only
 * read.  A (B, T) other than the tape's makes every gradient NaN (checked on the device).  The backward reads the handle's
 * packs of the latest forward: a forward of other weights, on any stream, must not run before or during it. */
int dsx_fft_train_backward(dsx_fft_train* h, const dsx_fft_params* w, const void* tape, const float* d_eps,
                           const dsx_fft_params* grads, float* d_cond, int B, int T, void* workspace,
                           size_t workspace_bytes, void* stream);

/* ---- SSIM mel loss ---------------------------------------------------------------------------------------------------
 * Replaces: ssim(img1, img2, window_size=11) (modules/commons/ssim.py:319-391) -- _ssim's five 11 x 11 conv2d and the
 * elementwise formula (:331-346) -- and its autograd backward, for one channel, as FastSpeech2Task.ssim_loss and
 * cwt_loss (tasks/tts/fs2.py:166-175, 271-277) call it.  Stateless, on the current device, like dsx_length_*.
 *
 * x, y, map, d_map, d_x, d_y: contiguous fp32 [B, H, W] (the [B, 1, H, W] images without the channel).  The window is
 * the outer product of the reference's float32 gaussian(11, 1.5), applied as two 11-tap passes with zero padding 5 in H
 * and W; C1 = 0.01^2, C2 = 0.03^2.  fp32 on CUDA cores throughout (no TF32).  B >= 1, H >= 1 and 1 <= W <= 256, else
 * DSX_E_INVALID.  One launch each; no workspace, atomics or handle.  Each image gives the same bits alone as in a
 * batch, and repeated calls give the same bits.
 *
 * dsx_ssim_forward: map = the SSIM map (_ssim's ssim_map; size_average=False returns it as ssim_map.mean(1)).
 * dsx_ssim_backward: d_x and d_y = the gradients of sum(d_map * map) with respect to x and y; either may be NULL (not
 * computed; both NULL launches nothing).  It recomputes the forward's moments instead of reading saved ones. */
int dsx_ssim_forward(const float* x, const float* y, int B, int H, int W, float* map, void* stream);
int dsx_ssim_backward(const float* x, const float* y, const float* d_map, int B, int H, int W, float* d_x, float* d_y,
                      void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DSX_H_ */
