"""FFT diffusion denoiser whose evaluations run the sm_90a kernels of libdsx.so (dsx_load_fft in include/dsx.h).

``FFT(hidden_size=None, num_layers=None, kernel_size=None, num_heads=None, *, hparams=None, train=None)`` keeps the
constructor, submodule names and the state dict of the reference's ``FFT`` (usr/diff/candidate_decoder.py:35-100, the
``DIFF_DECODERS['fft']`` entry of usr/diffsinger_task.py), so it loads with ``strict=True``.  Besides the constructor's
arguments it reads ``residual_channels``, ``audio_num_mel_bins``, ``ffn_padding``, ``ffn_act`` and ``dropout`` from
hparams.  Its eval ``forward(spec, diffusion_step, cond)`` is one evaluation in the sampler handle of ``.dsx``
(a ``DsxSampler``), which also runs whole sampling loops with it.  There is no eager or CPU path: a CPU tensor raises
``DsxError``.  A module in training mode raises ``DsxError`` too, unless the ``dsx_train`` opt-in (hparams key or
``train=`` keyword) is set: then a training-mode forward under autograd runs the sm_90a training step of
``diffsinger_b200.ffttrain`` (dropout p = hparams['dropout'], gradients for every parameter and for cond).

``DsxSampler`` recognises an FFT denoiser by its ``get_decode_inp.weight`` parameter, whether it is this class or the
reference's own ``FFT``, and takes the configuration from the module (``load_fft``).  So sampling needs no rebinding:
``dropin.install()``'s sampler subclasses route ``forward(infer=True)`` through ``DsxInferMixin`` with either class.  For
training, ``dropin.install()`` rebinds ``DIFF_DECODERS['fft']`` to build this class when hparams set ``dsx_train``.
"""
import ctypes

import torch
import torch.nn as nn

from . import _capi
from ._capi import DsxError, check, lib
from .fs2dec import FastspeechDecoder, _fs2dec_config, fs2dec_params
from .modules import Conv1d, Mish, SinusoidalPosEmb, _get_hparams
from .sampler import DsxSampler, _stream

MEL_BINS = 80   # get_mel_out is Linear(hidden_size, 80) in the reference


def _fft_config(dec_cfg, residual_channels, mel_bins):
    """-> FftConfig, or DsxError for what the kernels do not run."""
    dim, M = int(residual_channels), int(mel_bins)
    problems = []
    if not (16 <= dim <= 1024 and dim % 16 == 0):
        problems.append(f"residual_channels = {dim} (a multiple of 16 in [16, 1024])")
    if M != MEL_BINS:
        problems.append(f"audio_num_mel_bins = {M} ({MEL_BINS}: get_mel_out has {MEL_BINS} outputs)")
    if problems:
        raise DsxError("unsupported FFT denoiser configuration: " + "; ".join(problems))
    cfg = _capi.FftConfig()
    cfg.dec, cfg.residual_channels, cfg.mel_bins = dec_cfg, dim, M
    return cfg


def module_config(net, sd):
    """FftConfig of an FFT module (this class or the reference's) from its submodules and parameter shapes."""
    op = net.layers[0].op
    padding = 'LEFT' if isinstance(op.ffn.ffn_1, nn.Sequential) else 'SAME'
    H = sd["get_decode_inp.weight"].shape[0]
    dec = _fs2dec_config(H, len(net.layers), op.ffn.kernel_size, op.self_attn.num_heads, padding, op.ffn.act)
    dim, M = sd["input_projection.weight"].shape[:2]
    return _fft_config(dec, dim, M), padding


def load_fft(h, net, sd, device):
    """Packs the FFT module `net` (state dict `sd`) into sampler handle h -> its FftConfig."""
    cfg, padding = module_config(net, sd)
    keep = []

    def t(name):
        x = sd[name].detach().to(device=device, dtype=torch.float32).contiguous()
        keep.append(x)
        return x.data_ptr()

    def arr(names):
        a = (ctypes.c_void_p * len(names))(*[t(n) for n in names])
        keep.append(a)
        return ctypes.cast(a, ctypes.POINTER(ctypes.c_void_p))

    p = _capi.FftParams(
        dec=fs2dec_params(cfg.dec.layers, padding, t, arr),
        in_w=t("input_projection.weight"), in_b=t("input_projection.bias"),
        mlp0_w=t("mlp.0.weight"), mlp0_b=t("mlp.0.bias"), mlp2_w=t("mlp.2.weight"), mlp2_b=t("mlp.2.bias"),
        decode_inp_w=t("get_decode_inp.weight"), decode_inp_b=t("get_decode_inp.bias"),
        mel_out_w=t("get_mel_out.weight"), mel_out_b=t("get_mel_out.bias"))
    with torch.cuda.device(device):
        check(lib.dsx_load_fft(h, ctypes.byref(cfg), ctypes.byref(p), _stream(device)), "dsx_load_fft")
    return cfg


class FFT(FastspeechDecoder):
    def __init__(self, hidden_size=None, num_layers=None, kernel_size=None, num_heads=None, *, hparams=None, train=None):
        super().__init__(hidden_size, num_layers, kernel_size, num_heads, hparams=hparams, train=train)
        hp = _get_hparams(hparams)
        self._fft_cfg = _fft_config(self._cfg, hp['residual_channels'], hp['audio_num_mel_bins'])
        dim, M = self._fft_cfg.residual_channels, self._fft_cfg.mel_bins
        self.input_projection = Conv1d(M, dim, 1)             # candidate_decoder.py:38-48
        self.diffusion_embedding = SinusoidalPosEmb(dim)
        self.mlp = nn.Sequential(nn.Linear(dim, dim * 4), Mish(), nn.Linear(dim * 4, dim))
        self.get_mel_out = nn.Linear(self.hidden_size, MEL_BINS, bias=True)
        self.get_decode_inp = nn.Linear(self.hidden_size + dim + dim, self.hidden_size)
        self._sampler = None

    @property
    def dsx(self):
        if self._sampler is None:
            object.__setattr__(self, "_sampler", DsxSampler(self))
        return self._sampler

    def __getstate__(self):
        # the sampler holds a ctypes handle: copies build their own
        state = self.__dict__.copy()
        state["_sampler"] = None
        state["_dsx_trainer"] = None
        return state

    def _dsx_train_step(self):
        if self._dsx_trainer is None:
            from .ffttrain import FftTrainStep
            object.__setattr__(self, "_dsx_trainer", FftTrainStep(self._fft_cfg))
        return self._dsx_trainer

    def forward(self, spec, diffusion_step, cond, padding_mask=None, attn_mask=None, return_hiddens=False):
        """spec [B, 1, 80, T], diffusion_step [B], cond [B, hidden_size, T] -> eps [B, 1, 80, T] fp32
        (candidate_decoder.py:50-100), utterance b at step diffusion_step[b]."""
        if padding_mask is not None or attn_mask is not None or return_hiddens:
            raise DsxError("the dsx FFT denoiser takes spec, diffusion_step and cond only: padding_mask, attn_mask and "
                           "return_hiddens are not supported")
        if self.training and self._dsx_train and torch.is_grad_enabled():
            from .ffttrain import fft_train_forward
            return fft_train_forward(self, spec, diffusion_step, cond)
        if self.training:
            raise DsxError("the dsx FFT denoiser runs in eval mode only (call .eval()); training stays with the "
                           "reference's modules")
        return self.dsx.diffnet_forward(spec, diffusion_step, cond)
