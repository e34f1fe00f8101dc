"""ctypes binding of the dsx C ABI (include/dsx.h).  There is no Python or CPU fallback: if the
shared library is missing or does not load, importing this module raises."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("DSX_LIB", os.path.join(_HERE, "lib", "libdsx.so"))

PREC_FP32_SIMT, PREC_FP16, PREC_FP16X2, PREC_FP16X3, PREC_FP16S = 0, 1, 2, 3, 4
PRECISIONS = {"fp32": PREC_FP32_SIMT, "fp32_simt": PREC_FP32_SIMT, "fp16": PREC_FP16, "fp16x2": PREC_FP16X2,
              "fp16x3": PREC_FP16X3, "fp16s": PREC_FP16S}
(INFO_PRECISION, INFO_KERNEL_LAUNCHES, INFO_WORKSPACE_BYTES, INFO_SM_COUNT, INFO_TC_CTA_GROUP, INFO_LAYER_KERNEL_NS,
 INFO_LAYER_KERNEL_LAUNCHES, INFO_STACK_MODE, INFO_CLUSTER_OCCUPANCY, INFO_STACK_KERNEL_LAUNCHES, INFO_STACK_ROWS) = range(11)
TRACE_SLOTS = 256        # DSX_TRACE_SLOTS: int64 stamps per CTA row of dsx_debug_trace
OPT_TC_CTA_GROUP, OPT_CP_PREFETCH, OPT_PROFILE, OPT_STACK_MODE, OPT_STACK_KERNEL, OPT_SR_SETS, OPT_BATCH_OFFSET, OPT_GATE_APPROX, OPT_STACK_ROWS, OPT_FUSED_HEAD = 0, 1, 2, 3, 4, 5, 6, 7, 8, 9
SCHEDULE_BUFFERS = (
    "betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod",
    "sqrt_one_minus_alphas_cumprod", "log_one_minus_alphas_cumprod", "sqrt_recip_alphas_cumprod",
    "sqrt_recipm1_alphas_cumprod", "posterior_variance", "posterior_log_variance_clipped",
    "posterior_mean_coef1", "posterior_mean_coef2",
)
# every symbol include/dsx.h declares
SYMBOLS = (
    "dsx_version", "dsx_last_error", "dsx_create", "dsx_destroy", "dsx_load_diffnet", "dsx_set_schedule",
    "dsx_diffnet_forward", "dsx_sample_ddpm", "dsx_sample_plms", "dsx_infer", "dsx_infer_host", "dsx_get_info",
    "dsx_set_option", "dsx_set_cond", "dsx_plms_update", "dsx_debug_read", "dsx_debug_trace", "dsx_debug_set_layer_limit", "dsx_selftest",
    "dsx_hifigan_create", "dsx_hifigan_destroy", "dsx_hifigan_load", "dsx_hifigan_forward",
    "dsx_pe_create", "dsx_pe_destroy", "dsx_pe_load", "dsx_pe_forward",
    "dsx_fs2dec_create", "dsx_fs2dec_destroy", "dsx_fs2dec_load", "dsx_fs2dec_forward", "dsx_load_fft",
    "dsx_fs2enc_create", "dsx_fs2enc_destroy", "dsx_fs2enc_load", "dsx_fs2enc_forward",
    "dsx_durpred_create", "dsx_durpred_destroy", "dsx_durpred_load", "dsx_durpred_forward",
    "dsx_length_totals", "dsx_length_regulate",
    "dsx_train_create", "dsx_train_destroy", "dsx_train_tape_bytes", "dsx_train_workspace_bytes", "dsx_train_forward", "dsx_train_backward",
    "dsx_fs2dec_train_create", "dsx_fs2dec_train_destroy", "dsx_fs2dec_train_tape_bytes",
    "dsx_fs2dec_train_workspace_bytes", "dsx_fs2dec_train_forward", "dsx_fs2dec_train_backward", "dsx_fs2dec_train_masks",
    "dsx_fft_train_create", "dsx_fft_train_destroy", "dsx_fft_train_tape_bytes", "dsx_fft_train_workspace_bytes",
    "dsx_fft_train_forward", "dsx_fft_train_backward",
    "dsx_fs2enc_train_create", "dsx_fs2enc_train_destroy", "dsx_fs2enc_train_tape_bytes",
    "dsx_fs2enc_train_workspace_bytes", "dsx_fs2enc_train_forward", "dsx_fs2enc_train_backward",
    "dsx_durpred_train_create", "dsx_durpred_train_destroy", "dsx_durpred_train_tape_bytes",
    "dsx_durpred_train_workspace_bytes", "dsx_durpred_train_forward", "dsx_durpred_train_backward",
    "dsx_durpred_train_masks",
    "dsx_pitchpred_create", "dsx_pitchpred_destroy", "dsx_pitchpred_load", "dsx_pitchpred_forward",
    "dsx_pitchpred_train_create", "dsx_pitchpred_train_destroy", "dsx_pitchpred_train_tape_bytes",
    "dsx_pitchpred_train_workspace_bytes", "dsx_pitchpred_train_forward", "dsx_pitchpred_train_backward",
    "dsx_pitchpred_train_masks",
    "dsx_pwg_create", "dsx_pwg_destroy", "dsx_pwg_load", "dsx_pwg_forward",
    "dsx_ssim_forward", "dsx_ssim_backward",
)
_VOID = ("dsx_last_error", "dsx_destroy", "dsx_hifigan_destroy", "dsx_pe_destroy", "dsx_fs2dec_destroy",
         "dsx_fs2enc_destroy", "dsx_durpred_destroy", "dsx_train_destroy", "dsx_fs2dec_train_destroy",
         "dsx_fft_train_destroy", "dsx_fs2enc_train_destroy", "dsx_durpred_train_destroy", "dsx_pitchpred_destroy",
         "dsx_pitchpred_train_destroy", "dsx_pwg_destroy")


class DsxError(RuntimeError):
    pass


class Strides(ctypes.Structure):
    _fields_ = [("b", ctypes.c_int64), ("c", ctypes.c_int64), ("t", ctypes.c_int64)]


_fp = ctypes.c_void_p
_fpp = ctypes.POINTER(ctypes.c_void_p)


class DiffNetParams(ctypes.Structure):
    _fields_ = [("in_w", _fp), ("in_b", _fp), ("mlp0_w", _fp), ("mlp0_b", _fp), ("mlp2_w", _fp), ("mlp2_b", _fp),
                ("dil_w", _fpp), ("dil_b", _fpp), ("dif_w", _fpp), ("dif_b", _fpp), ("cond_w", _fpp),
                ("cond_b", _fpp), ("out_w", _fpp), ("out_b", _fpp), ("skip_w", _fp), ("skip_b", _fp),
                ("fin_w", _fp), ("fin_b", _fp)]


class HifiganConfig(ctypes.Structure):
    _fields_ = [("num_upsamples", ctypes.c_int), ("upsample_rates", ctypes.c_int * 4),
                ("upsample_kernel_sizes", ctypes.c_int * 4), ("upsample_initial_channel", ctypes.c_int),
                ("resblock", ctypes.c_int), ("num_kernels", ctypes.c_int), ("resblock_kernel_sizes", ctypes.c_int * 3),
                ("resblock_dilation_sizes", (ctypes.c_int * 3) * 3), ("audio_sample_rate", ctypes.c_int),
                ("use_pitch_embed", ctypes.c_int)]


class HifiganParams(ctypes.Structure):
    _fields_ = [("conv_pre_w", _fp), ("conv_pre_g", _fp), ("conv_pre_b", _fp), ("ups_w", _fpp), ("ups_g", _fpp),
                ("ups_b", _fpp), ("rb_w", _fpp), ("rb_g", _fpp), ("rb_b", _fpp), ("noise_w", _fpp), ("noise_b", _fpp),
                ("source_w", _fp), ("source_b", _fp), ("conv_post_w", _fp), ("conv_post_g", _fp), ("conv_post_b", _fp)]


class PwgConfig(ctypes.Structure):
    _fields_ = [("layers", ctypes.c_int), ("stacks", ctypes.c_int), ("kernel_size", ctypes.c_int),
                ("residual_channels", ctypes.c_int), ("gate_channels", ctypes.c_int), ("skip_channels", ctypes.c_int),
                ("aux_channels", ctypes.c_int), ("aux_context_window", ctypes.c_int), ("num_scales", ctypes.c_int),
                ("upsample_scales", ctypes.c_int * 4), ("use_pitch_embed", ctypes.c_int)]


class PwgParams(ctypes.Structure):
    _fields_ = [("first_w", _fp), ("first_g", _fp), ("first_b", _fp), ("conv_in_w", _fp), ("conv_in_g", _fp),
                ("up_w", _fpp), ("up_g", _fpp), ("conv_w", _fpp), ("conv_g", _fpp), ("conv_b", _fpp), ("aux_w", _fpp),
                ("aux_g", _fpp), ("out_w", _fpp), ("out_g", _fpp), ("out_b", _fpp), ("skip_w", _fpp), ("skip_g", _fpp),
                ("skip_b", _fpp), ("last1_w", _fp), ("last1_g", _fp), ("last1_b", _fp), ("last3_w", _fp),
                ("last3_g", _fp), ("last3_b", _fp), ("pitch_embed", _fp), ("c_proj_w", _fp), ("c_proj_b", _fp)]


class PeConfig(ctypes.Structure):
    _fields_ = [("n_mel_bins", ctypes.c_int), ("hidden", ctypes.c_int), ("predictor_hidden", ctypes.c_int),
                ("predictor_kernel", ctypes.c_int), ("conv_layers", ctypes.c_int), ("causal", ctypes.c_int),
                ("pitch_norm", ctypes.c_int), ("f0_mean", ctypes.c_float), ("f0_std", ctypes.c_float),
                ("use_uv", ctypes.c_int)]


class PeParams(ctypes.Structure):
    _fields_ = [("prenet_w", _fpp), ("prenet_b", _fpp), ("bn_w", _fpp), ("bn_b", _fpp), ("bn_mean", _fpp),
                ("bn_var", _fpp), ("prenet_out_w", _fp), ("prenet_out_b", _fp), ("enc_in_w", _fp), ("enc_in_b", _fp),
                ("enc_w", _fpp), ("enc_b", _fpp), ("gn_w", _fpp), ("gn_b", _fpp), ("enc_out_w", _fp), ("enc_out_b", _fp),
                ("pred_w", _fpp), ("pred_b", _fpp), ("ln_w", _fpp), ("ln_b", _fpp), ("linear_w", _fp), ("linear_b", _fp),
                ("pos_embed_alpha", _fp)]


class Fs2DecConfig(ctypes.Structure):
    _fields_ = [("hidden", ctypes.c_int), ("layers", ctypes.c_int), ("kernel", ctypes.c_int), ("heads", ctypes.c_int),
                ("padding", ctypes.c_int), ("act", ctypes.c_int)]


class Fs2DecParams(ctypes.Structure):
    _fields_ = [("ln1_w", _fpp), ("ln1_b", _fpp), ("in_proj_w", _fpp), ("out_proj_w", _fpp), ("ln2_w", _fpp),
                ("ln2_b", _fpp), ("ffn1_w", _fpp), ("ffn1_b", _fpp), ("ffn2_w", _fpp), ("ffn2_b", _fpp), ("ln_w", _fp),
                ("ln_b", _fp), ("pos_embed_alpha", _fp)]


class FftConfig(ctypes.Structure):
    _fields_ = [("dec", Fs2DecConfig), ("residual_channels", ctypes.c_int), ("mel_bins", ctypes.c_int)]


class FftParams(ctypes.Structure):
    _fields_ = [("dec", Fs2DecParams), ("in_w", _fp), ("in_b", _fp), ("mlp0_w", _fp), ("mlp0_b", _fp), ("mlp2_w", _fp),
                ("mlp2_b", _fp), ("decode_inp_w", _fp), ("decode_inp_b", _fp), ("mel_out_w", _fp), ("mel_out_b", _fp)]


class Fs2EncConfig(ctypes.Structure):
    _fields_ = [("stack", Fs2DecConfig), ("vocab", ctypes.c_int), ("pos", ctypes.c_int)]


class Fs2EncParams(ctypes.Structure):
    _fields_ = [("stack", Fs2DecParams), ("embed_w", _fp)]


class DurPredConfig(ctypes.Structure):
    _fields_ = [("idim", ctypes.c_int), ("chans", ctypes.c_int), ("layers", ctypes.c_int), ("kernel", ctypes.c_int),
                ("padding", ctypes.c_int), ("offset", ctypes.c_float)]


class DurPredParams(ctypes.Structure):
    _fields_ = [("conv_w", _fpp), ("conv_b", _fpp), ("ln_w", _fpp), ("ln_b", _fpp), ("linear_w", _fp),
                ("linear_b", _fp)]


class PitchPredConfig(ctypes.Structure):
    _fields_ = [("idim", ctypes.c_int), ("chans", ctypes.c_int), ("layers", ctypes.c_int), ("kernel", ctypes.c_int),
                ("padding", ctypes.c_int), ("odim", ctypes.c_int)]


class PitchPredParams(ctypes.Structure):
    _fields_ = [("conv_w", _fpp), ("conv_b", _fpp), ("ln_w", _fpp), ("ln_b", _fpp), ("linear_w", _fp),
                ("linear_b", _fp), ("pos_embed_alpha", _fp)]


class TrainConfig(ctypes.Structure):
    _fields_ = [("M", ctypes.c_int), ("C", ctypes.c_int), ("H", ctypes.c_int), ("L", ctypes.c_int),
                ("dilation_cycle", ctypes.c_int)]


if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"dsx CUDA library not found at {LIB_PATH}; build it with `python diffsinger_b200/build.py` "
        "(nvcc, sm_90a).  There is no CPU fallback.")
lib = ctypes.CDLL(LIB_PATH)

_i, _i64, _u64, _vp = ctypes.c_int, ctypes.c_int64, ctypes.c_uint64, ctypes.c_void_p
lib.dsx_version.restype = _i
lib.dsx_last_error.restype = ctypes.c_char_p
lib.dsx_create.argtypes = [_i, ctypes.POINTER(_vp)]
lib.dsx_destroy.argtypes = [_vp]
lib.dsx_destroy.restype = None
lib.dsx_load_diffnet.argtypes = [_vp, ctypes.POINTER(DiffNetParams), _i, _i, _i, _i, _i, _i, _vp]
lib.dsx_set_schedule.argtypes = [_vp, ctypes.POINTER(_vp), _i]
lib.dsx_diffnet_forward.argtypes = [_vp, _vp, Strides, _vp, _vp, Strides, _vp, _i, _i, _vp]
lib.dsx_sample_ddpm.argtypes = [_vp, _vp, _vp, Strides, _i, _i, _i, _i, _vp, _u64, _vp]
lib.dsx_sample_plms.argtypes = [_vp, _vp, _vp, Strides, _i, _i, _i, _i, _vp]
lib.dsx_infer.argtypes = [_vp, _vp, Strides, _vp, _vp, _vp, _vp, _u64, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]
lib.dsx_infer_host.argtypes = [_vp, _vp, Strides, _vp, _vp, _u64, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]
lib.dsx_set_cond.argtypes = [_vp, _vp, Strides, _i, _i, _vp]
lib.dsx_plms_update.argtypes = [_vp, _vp, _vp, ctypes.POINTER(_vp), _i, _i, _i, _i, _i, _vp]
lib.dsx_get_info.argtypes = [_vp, _i, ctypes.POINTER(_i64)]
lib.dsx_set_option.argtypes = [_vp, _i, _i64]
lib.dsx_debug_read.argtypes = [_vp, _i, _vp, _i, _i, _vp]
lib.dsx_debug_set_layer_limit.argtypes = [_vp, _i]
lib.dsx_debug_trace.argtypes = [_vp, _i, _vp]
lib.dsx_selftest.argtypes = [_i, _i, ctypes.c_char_p, _i]
lib.dsx_hifigan_create.argtypes = [_i, ctypes.POINTER(HifiganConfig), ctypes.POINTER(_vp)]
lib.dsx_hifigan_destroy.argtypes = [_vp]
lib.dsx_hifigan_destroy.restype = None
lib.dsx_hifigan_load.argtypes = [_vp, ctypes.POINTER(HifiganParams), _vp]
lib.dsx_hifigan_forward.argtypes = [_vp, _vp, Strides, _vp, _vp, _vp, _vp, _u64, _i, _i, _vp, _vp]
lib.dsx_pe_create.argtypes = [_i, ctypes.POINTER(PeConfig), ctypes.POINTER(_vp)]
lib.dsx_pe_destroy.argtypes = [_vp]
lib.dsx_pe_destroy.restype = None
lib.dsx_pe_load.argtypes = [_vp, ctypes.POINTER(PeParams), _vp]
lib.dsx_pe_forward.argtypes = [_vp, _vp, Strides, _i, _i, _vp, _vp, _vp]
lib.dsx_fs2dec_create.argtypes = [_i, ctypes.POINTER(Fs2DecConfig), ctypes.POINTER(_vp)]
lib.dsx_fs2dec_destroy.argtypes = [_vp]
lib.dsx_fs2dec_destroy.restype = None
lib.dsx_fs2dec_load.argtypes = [_vp, ctypes.POINTER(Fs2DecParams), _vp]
lib.dsx_fs2dec_forward.argtypes = [_vp, _vp, Strides, _i, _i, _vp, _vp]
lib.dsx_load_fft.argtypes = [_vp, ctypes.POINTER(FftConfig), ctypes.POINTER(FftParams), _vp]
lib.dsx_fs2enc_create.argtypes = [_i, ctypes.POINTER(Fs2EncConfig), ctypes.POINTER(_vp)]
lib.dsx_fs2enc_destroy.argtypes = [_vp]
lib.dsx_fs2enc_destroy.restype = None
lib.dsx_fs2enc_load.argtypes = [_vp, ctypes.POINTER(Fs2EncParams), _vp]
lib.dsx_fs2enc_forward.argtypes = [_vp, _vp, _i, _i, ctypes.POINTER(_vp), ctypes.POINTER(Strides), _i, _vp, _vp]
lib.dsx_durpred_create.argtypes = [_i, ctypes.POINTER(DurPredConfig), ctypes.POINTER(_vp)]
lib.dsx_durpred_destroy.argtypes = [_vp]
lib.dsx_durpred_destroy.restype = None
lib.dsx_durpred_load.argtypes = [_vp, ctypes.POINTER(DurPredParams), _vp]
lib.dsx_durpred_forward.argtypes = [_vp, _vp, Strides, _vp, _i, _i, _vp, _vp, _vp]
lib.dsx_length_totals.argtypes = [_vp, _vp, _i, _i, ctypes.c_float, _vp, _vp, _vp]
lib.dsx_length_regulate.argtypes = [_vp, _vp, _i, _i, _i, _vp, _vp]
lib.dsx_train_create.argtypes = [_i, ctypes.POINTER(TrainConfig), ctypes.POINTER(_vp)]
lib.dsx_train_destroy.argtypes = [_vp]
lib.dsx_train_destroy.restype = None
lib.dsx_train_tape_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_train_workspace_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_train_forward.argtypes = [_vp, ctypes.POINTER(DiffNetParams), _vp, Strides, _vp, _vp, Strides, _i, _i, _vp,
                                  ctypes.c_size_t, _vp, ctypes.c_size_t, _vp, _vp]
lib.dsx_train_backward.argtypes = [_vp, ctypes.POINTER(DiffNetParams), _vp, _vp, ctypes.POINTER(DiffNetParams), _vp,
                                   _i, _i, _vp, ctypes.c_size_t, _vp]
lib.dsx_fs2dec_train_create.argtypes = [_i, ctypes.POINTER(Fs2DecConfig), ctypes.POINTER(_vp)]
lib.dsx_fs2dec_train_destroy.argtypes = [_vp]
lib.dsx_fs2dec_train_destroy.restype = None
lib.dsx_fs2dec_train_tape_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_fs2dec_train_workspace_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_fs2dec_train_forward.argtypes = [_vp, ctypes.POINTER(Fs2DecParams), _vp, Strides, _i, _i, ctypes.c_float, _u64,
                                         _vp, ctypes.c_size_t, _vp, ctypes.c_size_t, _vp, _vp]
lib.dsx_fs2dec_train_backward.argtypes = [_vp, ctypes.POINTER(Fs2DecParams), _vp, _vp, ctypes.POINTER(Fs2DecParams), _vp,
                                          _i, _i, _vp, ctypes.c_size_t, _vp]
lib.dsx_fs2dec_train_masks.argtypes = [_vp, _u64, ctypes.c_float, _i, _i, ctypes.POINTER(_vp), _vp]
lib.dsx_fft_train_create.argtypes = [_i, ctypes.POINTER(FftConfig), ctypes.POINTER(_vp)]
lib.dsx_fft_train_destroy.argtypes = [_vp]
lib.dsx_fft_train_destroy.restype = None
lib.dsx_fft_train_tape_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_fft_train_workspace_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_fft_train_forward.argtypes = [_vp, ctypes.POINTER(FftParams), _vp, Strides, _vp, _vp, Strides, _i, _i,
                                      ctypes.c_float, _u64, _vp, ctypes.c_size_t, _vp, ctypes.c_size_t, _vp, _vp]
lib.dsx_fft_train_backward.argtypes = [_vp, ctypes.POINTER(FftParams), _vp, _vp, ctypes.POINTER(FftParams), _vp, _i,
                                       _i, _vp, ctypes.c_size_t, _vp]
lib.dsx_fs2enc_train_create.argtypes = [_i, ctypes.POINTER(Fs2EncConfig), ctypes.POINTER(_vp)]
lib.dsx_fs2enc_train_destroy.argtypes = [_vp]
lib.dsx_fs2enc_train_destroy.restype = None
lib.dsx_fs2enc_train_tape_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_fs2enc_train_workspace_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_fs2enc_train_forward.argtypes = [_vp, ctypes.POINTER(Fs2EncParams), _vp, _i, _i, ctypes.POINTER(_vp),
                                         ctypes.POINTER(Strides), _i, ctypes.c_float, _u64, _vp, ctypes.c_size_t, _vp,
                                         ctypes.c_size_t, _vp, _vp]
lib.dsx_fs2enc_train_backward.argtypes = [_vp, ctypes.POINTER(Fs2EncParams), _vp, _vp, ctypes.POINTER(Fs2EncParams), _vp,
                                          _i, _i, _vp, ctypes.c_size_t, _vp]
lib.dsx_durpred_train_create.argtypes = [_i, ctypes.POINTER(DurPredConfig), ctypes.POINTER(_vp)]
lib.dsx_durpred_train_destroy.argtypes = [_vp]
lib.dsx_durpred_train_destroy.restype = None
lib.dsx_durpred_train_tape_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_durpred_train_workspace_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_durpred_train_forward.argtypes = [_vp, ctypes.POINTER(DurPredParams), _vp, Strides, _vp, _i, _i, ctypes.c_float,
                                          _u64, _vp, ctypes.c_size_t, _vp, ctypes.c_size_t, _vp, _vp]
lib.dsx_durpred_train_backward.argtypes = [_vp, ctypes.POINTER(DurPredParams), _vp, _vp, ctypes.POINTER(DurPredParams),
                                           _vp, _i, _i, _vp, ctypes.c_size_t, _vp]
lib.dsx_durpred_train_masks.argtypes = [_vp, _u64, ctypes.c_float, _i, _i, ctypes.POINTER(_vp), _vp]
lib.dsx_pitchpred_create.argtypes = [_i, ctypes.POINTER(PitchPredConfig), ctypes.POINTER(_vp)]
lib.dsx_pitchpred_destroy.argtypes = [_vp]
lib.dsx_pitchpred_destroy.restype = None
lib.dsx_pitchpred_load.argtypes = [_vp, ctypes.POINTER(PitchPredParams), _vp]
lib.dsx_pitchpred_forward.argtypes = [_vp, _vp, _i, _i, _vp, _vp]
lib.dsx_pitchpred_train_create.argtypes = [_i, ctypes.POINTER(PitchPredConfig), ctypes.POINTER(_vp)]
lib.dsx_pitchpred_train_destroy.argtypes = [_vp]
lib.dsx_pitchpred_train_destroy.restype = None
lib.dsx_pitchpred_train_tape_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_pitchpred_train_workspace_bytes.argtypes = [_vp, _i, _i, ctypes.POINTER(ctypes.c_size_t)]
lib.dsx_pitchpred_train_forward.argtypes = [_vp, ctypes.POINTER(PitchPredParams), _vp, _i, _i, ctypes.c_float, _u64, _vp,
                                            ctypes.c_size_t, _vp, ctypes.c_size_t, _vp, _vp]
lib.dsx_pitchpred_train_backward.argtypes = [_vp, ctypes.POINTER(PitchPredParams), _vp, _vp,
                                             ctypes.POINTER(PitchPredParams), _vp, _i, _i, _vp, ctypes.c_size_t, _vp]
lib.dsx_pitchpred_train_masks.argtypes = [_vp, _u64, ctypes.c_float, _i, _i, ctypes.POINTER(_vp), _vp]
lib.dsx_pwg_create.argtypes = [_i, ctypes.POINTER(PwgConfig), ctypes.POINTER(_vp)]
lib.dsx_pwg_destroy.argtypes = [_vp]
lib.dsx_pwg_destroy.restype = None
lib.dsx_pwg_load.argtypes = [_vp, ctypes.POINTER(PwgParams), _vp]
lib.dsx_pwg_forward.argtypes = [_vp, _vp, _vp, Strides, _vp, _i, _i, _vp, _vp]
lib.dsx_ssim_forward.argtypes = [_vp, _vp, _i, _i, _i, _vp, _vp]
lib.dsx_ssim_backward.argtypes = [_vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]
for _n in SYMBOLS:
    if _n not in _VOID:
        getattr(lib, _n).restype = _i


def check(rc, what=""):
    if rc != 0:
        raise DsxError(f"{what or 'dsx call'} failed ({rc}): {lib.dsx_last_error().decode(errors='replace')}")
