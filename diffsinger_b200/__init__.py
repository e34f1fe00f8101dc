"""diffsinger_b200 -- H100-native (sm_90a) reverse-diffusion sampler for DiffSinger / DiffSpeech.

The compute lives in ``lib/libdsx.so`` (hand-written CUDA behind the C ABI of ``include/dsx.h``);
this package is the thin host side that mirrors the reference's ``DiffNet`` / ``GaussianDiffusion``
class surface.  Importing it requires the built library -- there is no Python or CPU fallback.
"""
from ._capi import DsxError, LIB_PATH, PRECISIONS  # noqa: F401  (raises ImportError when libdsx.so is missing)
from .sampler import DsxSampler, selftest  # noqa: F401
from .modules import DiffNet, GaussianDiffusion, Mish, SinusoidalPosEmb  # noqa: F401

__all__ = ["DiffNet", "GaussianDiffusion", "DsxSampler", "DsxError", "selftest"]
