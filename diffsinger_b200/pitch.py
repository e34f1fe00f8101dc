"""Pitch extractor whose forward runs the sm_90a kernels of libdsx.so (dsx_pe_* in include/dsx.h).

``PitchExtractor(n_mel_bins=80, conv_layers=2, hparams=None)`` keeps the reference's constructor, submodule names,
parameter and buffer shapes (modules/fastspeech/pe.py:7-149, modules/fastspeech/tts_modules.py:192-235), so the
reference's ``pe_ckpt`` loads strictly with ``utils.load_ckpt(pe, pe_ckpt, 'model', strict=True)``.  The modules only
hold the parameters: ``forward`` packs them into the library (once per storage and version, so again after
``load_state_dict`` or ``.to()``) and runs the whole extractor there, mel to denormalised f0.  There is no eager or CPU
path and no training path: a CPU tensor or a module in training mode raises ``DsxError``.
"""
import torch
import torch.nn as nn

from . import _capi
from ._capi import DsxError, check, lib
from .modules import _get_hparams
from .sampler import PackedModule, _need_cuda, _ptr, _stream, _strides_bct


class Prenet(nn.Module):
    """pe.py:7-21: 3 x [Conv1d(k=5, pad=2), ReLU, BatchNorm1d] and out_proj."""

    def __init__(self, in_dim=80, out_dim=256, kernel=5, n_layers=3):
        super().__init__()
        self.layers = nn.ModuleList([nn.Sequential(
            nn.Conv1d(in_dim if l == 0 else out_dim, out_dim, kernel_size=kernel, padding=kernel // 2),
            nn.ReLU(), nn.BatchNorm1d(out_dim)) for l in range(n_layers)])
        self.out_proj = nn.Linear(out_dim, out_dim)


class ConvNorm(nn.Module):
    """modules/commons/common_layers.py:41-59 (the submodule is named ``conv``)."""

    def __init__(self, in_channels, out_channels, kernel_size):
        super().__init__()
        self.conv = nn.Conv1d(in_channels, out_channels, kernel_size, padding=(kernel_size - 1) // 2)


class ConvBlock(nn.Module):
    """pe.py:44-60 with norm='gn'."""

    def __init__(self, n_chans, kernel_size):
        super().__init__()
        self.conv = ConvNorm(n_chans, n_chans, kernel_size)
        self.norm = nn.GroupNorm(n_chans // 16, n_chans)
        self.dropout = nn.Dropout(0)
        self.relu = nn.ReLU()


class ConvStacks(nn.Module):
    """pe.py:81-96: in_proj, n_layers GroupNorm conv blocks with residual, out_proj."""

    def __init__(self, n_chans, n_layers, kernel_size=5):
        super().__init__()
        self.in_proj = nn.Linear(n_chans, n_chans)
        self.conv = nn.ModuleList([ConvBlock(n_chans, kernel_size) for _ in range(n_layers)])
        self.out_proj = nn.Linear(n_chans, n_chans)


class SinusoidalPositionalEmbedding(nn.Module):
    """common_layers.py:88-103: only the ``_float_tensor`` buffer is state; the table is computed in the kernel."""

    def __init__(self, embedding_dim, padding_idx=0):
        super().__init__()
        self.embedding_dim, self.padding_idx = embedding_dim, padding_idx
        self.register_buffer('_float_tensor', torch.FloatTensor(1))


class LayerNorm(nn.LayerNorm):
    """tts_modules.py:37-56: LayerNorm over the channel dim with eps 1e-12."""

    def __init__(self, nout, dim=-1):
        super().__init__(nout, eps=1e-12)
        self.dim = dim


class PitchPredictor(nn.Module):
    """tts_modules.py:192-220: position embedding, 5 x [ConstantPad1d, Conv1d, ReLU, LayerNorm, Dropout], linear."""

    def __init__(self, idim, n_layers=5, n_chans=384, odim=2, kernel_size=5, dropout_rate=0.1, padding='SAME'):
        super().__init__()
        self.kernel_size, self.padding = kernel_size, padding
        pad = ((kernel_size - 1) // 2, (kernel_size - 1) // 2) if padding == 'SAME' else (kernel_size - 1, 0)
        self.conv = nn.ModuleList([nn.Sequential(
            nn.ConstantPad1d(pad, 0), nn.Conv1d(idim if i == 0 else n_chans, n_chans, kernel_size),
            nn.ReLU(), LayerNorm(n_chans, dim=1), nn.Dropout(dropout_rate)) for i in range(n_layers)])
        self.linear = nn.Linear(n_chans, odim)
        self.embed_positions = SinusoidalPositionalEmbedding(idim, 0)
        self.pos_embed_alpha = nn.Parameter(torch.Tensor([1]))


def _pe_config(hp, n_mel_bins, conv_layers):
    """hparams -> PeConfig, or DsxError for what the kernels do not run."""
    H = int(hp['hidden_size'])
    P = int(hp['predictor_hidden']) if int(hp['predictor_hidden']) > 0 else H
    k = int(hp['predictor_kernel'])
    norm = hp['pitch_norm']
    problems = []
    if n_mel_bins != 80:
        problems.append(f"n_mel_bins = {n_mel_bins} (80 only)")
    for name, v in (("hidden_size", H), ("predictor_hidden", P)):
        if not (16 <= v <= 256 and v % 16 == 0):
            problems.append(f"{name} = {v} (a multiple of 16 in [16, 256])")
    if not (1 <= k <= 31 and k % 2 == 1):
        problems.append(f"predictor_kernel = {k} (odd, <= 31)")
    if not (0 <= conv_layers <= 16):
        problems.append(f"conv_layers = {conv_layers} (0..16)")
    if norm not in ('log', 'standard'):
        problems.append(f"pitch_norm = {norm!r} ('log' or 'standard')")
    if problems:
        raise DsxError("unsupported pitch extractor configuration: " + "; ".join(problems))
    cfg = _capi.PeConfig()
    cfg.n_mel_bins, cfg.hidden, cfg.predictor_hidden, cfg.predictor_kernel = n_mel_bins, H, P, k
    cfg.conv_layers = conv_layers
    cfg.causal = 0 if hp['ffn_padding'] == 'SAME' else 1          # anything else pads (k - 1, 0): tts_modules.py:210
    cfg.pitch_norm = 0 if norm == 'log' else 1
    cfg.f0_mean = float(hp.get('f0_mean', 0.0) or 0.0) if cfg.pitch_norm else 0.0
    cfg.f0_std = float(hp.get('f0_std', 1.0) or 1.0) if cfg.pitch_norm else 1.0
    cfg.use_uv = 1 if (hp['pitch_type'] == 'frame' and hp['use_uv']) else 0   # pe.py:144
    return cfg


class PitchExtractor(PackedModule):
    def __init__(self, n_mel_bins=80, conv_layers=2, hparams=None):
        super().__init__()
        hp = _get_hparams(hparams)
        self._cfg = _pe_config(hp, n_mel_bins, conv_layers)
        self.hidden_size = self._cfg.hidden
        self.predictor_hidden = self._cfg.predictor_hidden
        self.conv_layers = conv_layers
        self.mel_prenet = Prenet(n_mel_bins, self.hidden_size)
        if conv_layers > 0:
            self.mel_encoder = ConvStacks(self.hidden_size, conv_layers)
        self.pitch_predictor = PitchPredictor(self.hidden_size, n_chans=self.predictor_hidden, n_layers=5,
                                              dropout_rate=0.1, odim=2, padding=hp['ffn_padding'],
                                              kernel_size=self._cfg.predictor_kernel)

    # -- library handle ---------------------------------------------------------------------------
    _lib_create, _lib_load, _lib_destroy = lib.dsx_pe_create, lib.dsx_pe_load, lib.dsx_pe_destroy

    def _config(self):
        return self._cfg

    def _params(self, sd, t, arr):
        pre =[f"mel_prenet.layers.{i}" for i in range(3)]
        enc = [f"mel_encoder.conv.{i}" for i in range(self.conv_layers)]
        pred = [f"pitch_predictor.conv.{i}" for i in range(5)]
        p = _capi.PeParams(
            prenet_w=arr([n + ".0.weight" for n in pre]), prenet_b=arr([n + ".0.bias" for n in pre]),
            bn_w=arr([n + ".2.weight" for n in pre]), bn_b=arr([n + ".2.bias" for n in pre]),
            bn_mean=arr([n + ".2.running_mean" for n in pre]), bn_var=arr([n + ".2.running_var" for n in pre]),
            prenet_out_w=t("mel_prenet.out_proj.weight"), prenet_out_b=t("mel_prenet.out_proj.bias"),
            pred_w=arr([n + ".1.weight" for n in pred]), pred_b=arr([n + ".1.bias" for n in pred]),
            ln_w=arr([n + ".3.weight" for n in pred]), ln_b=arr([n + ".3.bias" for n in pred]),
            linear_w=t("pitch_predictor.linear.weight"), linear_b=t("pitch_predictor.linear.bias"),
            pos_embed_alpha=t("pitch_predictor.pos_embed_alpha"))
        if self.conv_layers > 0:
            p.enc_in_w, p.enc_in_b = t("mel_encoder.in_proj.weight"), t("mel_encoder.in_proj.bias")
            p.enc_w, p.enc_b = arr([n + ".conv.conv.weight" for n in enc]), arr([n + ".conv.conv.bias" for n in enc])
            p.gn_w, p.gn_b = arr([n + ".norm.weight" for n in enc]), arr([n + ".norm.bias" for n in enc])
            p.enc_out_w, p.enc_out_b = t("mel_encoder.out_proj.weight"), t("mel_encoder.out_proj.bias")
        return p

    def forward(self, mel_input=None):
        """mel_input: [B, T, n_mel_bins] (any strides; dsx_infer's mel_out as it is).  A frame whose bins are all 0 is
        padding.  -> {'pitch_pred': [B, T, 2], 'f0_denorm_pred': [B, T] in Hz}."""
        x = mel_input
        if x is None or x.dim() != 3 or x.shape[-1] != self._cfg.n_mel_bins:
            raise DsxError(f"mel_input must be [B, T, {self._cfg.n_mel_bins}] "
                           f"(got {None if x is None else tuple(x.shape)})")
        if self.training:
            raise DsxError("the dsx pitch extractor runs in eval mode only (call .eval()); training stays with the "
                           "reference's modules")
        _need_cuda(x)
        dev = x.device
        hnd = self._ensure(dev)
        B, T, _ = x.shape
        mel = x.float()
        pitch = torch.empty((B, T, 2), device=dev, dtype=torch.float32)
        f0 = torch.empty((B, T), device=dev, dtype=torch.float32)
        if B > 0 and T > 0:
            with torch.cuda.device(dev):
                check(lib.dsx_pe_forward(hnd, _ptr(mel), _strides_bct(mel, (0, 2, 1)), B, T, _ptr(pitch), _ptr(f0),
                                         _stream(dev)), "dsx_pe_forward")
        return {'pitch_pred': pitch, 'f0_denorm_pred': f0}
