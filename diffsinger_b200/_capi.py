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
)


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
for _n in SYMBOLS:
    if getattr(lib, _n).restype is ctypes.c_int or _n not in ("dsx_last_error", "dsx_destroy"):
        if _n not in ("dsx_last_error", "dsx_destroy"):
            getattr(lib, _n).restype = _i


def check(rc, what=""):
    if rc != 0:
        raise DsxError(f"{what or 'dsx call'} failed ({rc}): {lib.dsx_last_error().decode(errors='replace')}")
