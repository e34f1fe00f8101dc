"""diffsinger_b200 -- H100-native (sm_90a) reverse-diffusion sampler for DiffSinger / DiffSpeech.

The compute lives in ``lib/libdsx.so`` (hand-written CUDA behind the C ABI of ``include/dsx.h``);
this package is the thin host side that mirrors the reference's ``DiffNet`` / ``GaussianDiffusion``
class surface, ``HifiGanGenerator`` mirrors the reference's HiFi-GAN (NSF) vocoder, ``ParallelWaveGANGenerator`` its Parallel WaveGAN vocoder, ``PitchExtractor`` its mel-to-f0 pitch extractor, ``FastspeechDecoder`` the FastSpeech2 decoder, ``FastspeechEncoder`` / ``FastspeechMIDIEncoder`` / ``DurationPredictor`` / ``LengthRegulator`` its encoder and duration path, ``PitchPredictor`` / ``EnergyPredictor`` its pitch and energy predictors, ``FFT`` the FFT diffusion denoiser, and ``ssim`` the SSIM mel loss.  Importing it requires the built library -- there is no Python or CPU fallback.
"""
from ._capi import DsxError, LIB_PATH, PRECISIONS  # noqa: F401  (raises ImportError when libdsx.so is missing)
from .sampler import DsxSampler, selftest  # noqa: F401
from .modules import DiffNet, GaussianDiffusion, Mish, SinusoidalPosEmb  # noqa: F401
from .vocoder import HifiGanGenerator  # noqa: F401
from .pwg import ParallelWaveGANGenerator  # noqa: F401
from .pitch import PitchExtractor  # noqa: F401
from .fs2dec import FastspeechDecoder  # noqa: F401
from .fftdiff import FFT  # noqa: F401
from .fs2enc import DurationPredictor, FastspeechEncoder, FastspeechMIDIEncoder, LengthRegulator  # noqa: F401
from .pitchpred import EnergyPredictor, PitchPredictor  # noqa: F401
from .ssim import ssim  # noqa: F401

__all__ = ["DiffNet", "GaussianDiffusion", "DsxSampler", "DsxError", "HifiGanGenerator", "ParallelWaveGANGenerator", "PitchExtractor", "FastspeechDecoder",
           "FFT", "FastspeechEncoder", "FastspeechMIDIEncoder", "DurationPredictor", "LengthRegulator", "PitchPredictor", "EnergyPredictor", "ssim", "selftest"]
