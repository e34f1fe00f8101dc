"""Parallel WaveGAN generator whose forward runs the sm_90a kernels of libdsx.so (dsx_pwg_* in include/dsx.h).

``ParallelWaveGANGenerator(**generator_params)`` keeps the reference's constructor, submodule tree, initialisation and
parameter names (modules/parallel_wavegan/models/parallel_wavegan.py:21-191, layers/residual_block.py,
layers/upsample.py): real ``nn.Conv1d`` / ``nn.Conv2d`` modules under ``weight_norm``, so an official checkpoint loads
strictly, ``fake_task.model_gen`` loads non-strictly, and ``remove_weight_norm()`` leaves the plain names.  The modules
only hold the parameters: ``forward`` packs them into the library (again after every change of the weights) and runs the
whole generator there, in eval mode.  There is no eager or CPU path: a CPU tensor raises ``DsxError``, and so does a
constructor option the kernels do not implement, naming the option.
"""
import logging
import math

import numpy as np
import torch
import torch.nn as nn

from . import _capi
from ._capi import DsxError, check, lib
from .sampler import PackedModule, _need_cuda, _ptr, _stream, _strides_bct

# the widths the kernels implement (every published Parallel WaveGAN config uses them)
WIDTHS = dict(kernel_size=3, residual_channels=64, gate_channels=128, skip_channels=64, aux_channels=80)


class Conv1d(nn.Conv1d):
    """Conv1d with the reference's initialisation (residual_block.py:15-26)."""

    def reset_parameters(self):
        nn.init.kaiming_normal_(self.weight, nonlinearity="relu")
        if self.bias is not None:
            nn.init.constant_(self.bias, 0.0)


class Conv1d1x1(Conv1d):
    """1x1 Conv1d (residual_block.py:29-36)."""

    def __init__(self, in_channels, out_channels, bias):
        super().__init__(in_channels, out_channels, kernel_size=1, padding=0, dilation=1, bias=bias)


class Conv2d(nn.Conv2d):
    """Conv2d with the reference's initialisation (upsample.py:48-60)."""

    def reset_parameters(self):
        self.weight.data.fill_(1. / np.prod(self.kernel_size))
        if self.bias is not None:
            nn.init.constant_(self.bias, 0.0)


class Stretch2d(nn.Module):
    """Nearest-neighbour stretch of the time axis (upsample.py:16-45); it has no parameters."""

    def __init__(self, x_scale, y_scale, mode="nearest"):
        super().__init__()
        self.x_scale, self.y_scale, self.mode = x_scale, y_scale, mode


class UpsampleNetwork(nn.Module):
    """upsample.py:63-124 with nearest interpolation, freq_axis_kernel_size 1 and no nonlinearity."""

    def __init__(self, upsample_scales):
        super().__init__()
        self.use_causal_conv = False
        self.up_layers = nn.ModuleList()
        for scale in upsample_scales:
            self.up_layers += [Stretch2d(scale, 1, "nearest")]
            self.up_layers += [Conv2d(1, 1, kernel_size=(1, scale * 2 + 1), padding=(0, scale), bias=False)]


class ConvInUpsampleNetwork(nn.Module):
    """upsample.py:127-183: conv_in (2w + 1 taps, no padding) and the UpsampleNetwork."""

    def __init__(self, upsample_scales, aux_channels=80, aux_context_window=0):
        super().__init__()
        self.aux_context_window = aux_context_window
        self.use_causal_conv = False
        self.conv_in = Conv1d(aux_channels, aux_channels, kernel_size=2 * aux_context_window + 1, bias=False)
        self.upsample = UpsampleNetwork(upsample_scales)


class ResidualBlock(nn.Module):
    """residual_block.py:39-91: the dilated conv, the auxiliary 1x1 conv and the 1x1 output and skip convs."""

    def __init__(self, kernel_size=3, residual_channels=64, gate_channels=128, skip_channels=64, aux_channels=80,
                 dropout=0.0, dilation=1, bias=True):
        super().__init__()
        self.dropout = dropout
        self.use_causal_conv = False
        padding = (kernel_size - 1) // 2 * dilation
        self.conv = Conv1d(residual_channels, gate_channels, kernel_size, padding=padding, dilation=dilation, bias=bias)
        self.conv1x1_aux = Conv1d1x1(aux_channels, gate_channels, bias=False)
        self.conv1x1_out = Conv1d1x1(gate_channels // 2, residual_channels, bias=bias)
        self.conv1x1_skip = Conv1d1x1(gate_channels // 2, skip_channels, bias=bias)


def _unsupported(option, value, supported):
    raise DsxError(f"unsupported {option}={value!r}: the dsx PWG kernels implement {supported}")


class ParallelWaveGANGenerator(PackedModule):
    def __init__(self, in_channels=1, out_channels=1, kernel_size=3, layers=30, stacks=3, residual_channels=64,
                 gate_channels=128, skip_channels=64, aux_channels=80, aux_context_window=2, dropout=0.0, bias=True,
                 use_weight_norm=True, use_causal_conv=False, upsample_conditional_features=True,
                 upsample_net="ConvInUpsampleNetwork", upsample_params={"upsample_scales": [4, 4, 4, 4]},
                 use_pitch_embed=False):
        super().__init__()
        up = dict(upsample_params)
        scales = list(up.get("upsample_scales", []))
        for option, value, ok, supported in (
                ("in_channels", in_channels, in_channels == 1, "1"),
                ("out_channels", out_channels, out_channels == 1, "1"),
                ("bias", bias, bias is True, "True"),
                ("use_causal_conv", use_causal_conv, not use_causal_conv, "False"),
                ("upsample_conditional_features", upsample_conditional_features, upsample_conditional_features is True,
                 "True"),
                ("upsample_net", upsample_net, upsample_net == "ConvInUpsampleNetwork", "'ConvInUpsampleNetwork'"),
                ("nonlinear_activation", up.get("nonlinear_activation"), up.get("nonlinear_activation") is None, "None"),
                ("interpolate_mode", up.get("interpolate_mode", "nearest"),
                 up.get("interpolate_mode", "nearest") == "nearest", "'nearest'"),
                ("freq_axis_kernel_size", up.get("freq_axis_kernel_size", 1), up.get("freq_axis_kernel_size", 1) == 1,
                 "1"),
                ("use_causal_conv (upsample_params)", up.get("use_causal_conv", False), not up.get("use_causal_conv"),
                 "False"),
                ("layers", layers, 1 <= layers <= 64, "1..64"),
                ("stacks", stacks, stacks >= 1 and layers % stacks == 0 and layers // stacks <= 16,
                 "a divisor of layers with layers / stacks <= 16"),
                ("upsample_scales", scales, 1 <= len(scales) <= 4 and all(1 <= s <= 16 for s in scales)
                 and math.prod(scales) <= 1024, "1..4 scales of 1..16 with a product <= 1024"),
                ("aux_context_window", aux_context_window, 0 <= aux_context_window <= 16, "0..16")):
            if not ok:
                _unsupported(option, value, supported)
        for option, want in WIDTHS.items():
            value = locals()[option]
            if value != want:
                _unsupported(option, value, str(want))
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.aux_channels = aux_channels
        self.layers = layers
        self.stacks = stacks
        self.kernel_size = kernel_size
        self.aux_context_window = aux_context_window
        self.upsample_scales = scales
        self.dropout = dropout
        layers_per_stack = layers // stacks

        self.first_conv = Conv1d1x1(in_channels, residual_channels, bias=True)
        self.upsample_net = ConvInUpsampleNetwork(scales, aux_channels=aux_channels, aux_context_window=aux_context_window)
        self.conv_layers = nn.ModuleList()
        for layer in range(layers):
            self.conv_layers += [ResidualBlock(kernel_size, residual_channels, gate_channels, skip_channels, aux_channels,
                                               dropout, 2 ** (layer % layers_per_stack), bias)]
        self.last_conv_layers = nn.ModuleList([
            nn.ReLU(inplace=True),
            Conv1d1x1(skip_channels, skip_channels, bias=True),
            nn.ReLU(inplace=True),
            Conv1d1x1(skip_channels, out_channels, bias=True),
        ])
        self.use_pitch_embed = use_pitch_embed
        if use_pitch_embed:
            self.pitch_embed = nn.Embedding(300, aux_channels, 0)
            self.c_proj = nn.Linear(2 * aux_channels, aux_channels)
        if use_weight_norm:
            self.apply_weight_norm()

    def remove_weight_norm(self):
        """parallel_wavegan.py:174-183"""
        def _remove_weight_norm(m):
            try:
                torch.nn.utils.remove_weight_norm(m)
            except ValueError:  # this module didn't have weight norm
                return

        self.apply(_remove_weight_norm)

    def apply_weight_norm(self):
        """parallel_wavegan.py:185-191"""
        def _apply_weight_norm(m):
            if isinstance(m, torch.nn.Conv1d) or isinstance(m, torch.nn.Conv2d):
                torch.nn.utils.weight_norm(m)
                logging.debug(f"Weight norm is applied to {m}.")

        self.apply(_apply_weight_norm)

    # -- library handle ---------------------------------------------------------------------------
    _lib_create, _lib_load, _lib_destroy = lib.dsx_pwg_create, lib.dsx_pwg_load, lib.dsx_pwg_destroy

    def hop(self):
        return math.prod(self.upsample_scales)

    def _config(self):
        cfg = _capi.PwgConfig(layers=self.layers, stacks=self.stacks, aux_context_window=self.aux_context_window,
                              num_scales=len(self.upsample_scales), use_pitch_embed=1 if self.use_pitch_embed else 0,
                              **WIDTHS)
        for i, s in enumerate(self.upsample_scales):
            cfg.upsample_scales[i] = int(s)
        return cfg

    def _params(self, sd, t, arr):
        def conv(name):      # (w, g): weight_v / weight_g of a weight-normalised conv, or (weight, NULL)
            if name + ".weight_g" in sd:
                return t(name + ".weight_v"), t(name + ".weight_g")
            return t(name + ".weight"), None

        def convs(names):
            wg = [conv(n) for n in names]
            return arr([w for w, _ in wg]), arr([g for _, g in wg])

        L = self.layers
        first_w, first_g = conv("first_conv")
        in_w, in_g = conv("upsample_net.conv_in")
        up_w, up_g = convs([f"upsample_net.upsample.up_layers.{2 * i + 1}" for i in range(len(self.upsample_scales))])
        layer = lambda sub: [f"conv_layers.{l}.{sub}" for l in range(L)]
        conv_w, conv_g = convs(layer("conv"))
        aux_w, aux_g = convs(layer("conv1x1_aux"))
        out_w, out_g = convs(layer("conv1x1_out"))
        skip_w, skip_g = convs(layer("conv1x1_skip"))
        l1_w, l1_g = conv("last_conv_layers.1")
        l3_w, l3_g = conv("last_conv_layers.3")
        p = _capi.PwgParams(
            first_w=first_w, first_g=first_g, first_b=t("first_conv.bias"), conv_in_w=in_w, conv_in_g=in_g,
            up_w=up_w, up_g=up_g, conv_w=conv_w, conv_g=conv_g, conv_b=arr([n + ".bias" for n in layer("conv")]),
            aux_w=aux_w, aux_g=aux_g, out_w=out_w, out_g=out_g, out_b=arr([n + ".bias" for n in layer("conv1x1_out")]),
            skip_w=skip_w, skip_g=skip_g, skip_b=arr([n + ".bias" for n in layer("conv1x1_skip")]),
            last1_w=l1_w, last1_g=l1_g, last1_b=t("last_conv_layers.1.bias"),
            last3_w=l3_w, last3_g=l3_g, last3_b=t("last_conv_layers.3.bias"))
        if self.use_pitch_embed:
            p.pitch_embed, p.c_proj_w, p.c_proj_b = t("pitch_embed.weight"), t("c_proj.weight"), t("c_proj.bias")
        return p

    def forward(self, x, c=None, pitch=None, **kwargs):
        """x: noise [B, 1, T * hop]; c: [B, 80, T + 2w] (any strides, edge-padded by w = aux_context_window frames);
        pitch: int64 [B, T + 2w] coarse pitch, read only with use_pitch_embed (as in the reference).
        -> wav [B, 1, T * hop]."""
        if c is None:
            raise DsxError("the dsx PWG generator needs the auxiliary features c (upsample_conditional_features)")
        if self.training and self.dropout > 0:
            raise DsxError("the dsx PWG generator runs in eval mode only (dropout > 0 in training mode)")
        _need_cuda(x, c, pitch if self.use_pitch_embed else None)
        w, hop = self.aux_context_window, self.hop()
        if x.dim() != 3 or x.shape[1] != 1 or c.dim() != 3 or c.shape[1] != self.aux_channels:
            raise DsxError(f"x must be [B, 1, T * hop] and c [B, {self.aux_channels}, T + 2w] (got {tuple(x.shape)}, "
                           f"{tuple(c.shape)})")
        B, Tp = c.shape[0], c.shape[2]
        T = Tp - 2 * w
        if x.shape[0] != B or T < 1 or x.shape[2] != T * hop:
            raise DsxError(f"x {tuple(x.shape)} and c {tuple(c.shape)} disagree: c has T + 2w frames (w = {w}) and x "
                           f"T * hop samples (hop = {hop})")
        dev = x.device
        hnd = self._ensure(dev)
        z = x.to(torch.float32).contiguous()
        cf = c.to(torch.float32)
        p = None
        if self.use_pitch_embed:
            if pitch is None:
                raise DsxError("this generator has a pitch embedding (use_pitch_embed): pitch is required")
            if tuple(pitch.shape) != (B, Tp):
                raise DsxError(f"pitch must have shape {(B, Tp)} (got {tuple(pitch.shape)})")
            p = pitch.to(device=dev, dtype=torch.int64).contiguous()
        wav = torch.empty((B, 1, T * hop), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib.dsx_pwg_forward(hnd, _ptr(z), _ptr(cf), _strides_bct(cf, (0, 1, 2)), _ptr(p), B, T, _ptr(wav),
                                      _stream(dev)), "dsx_pwg_forward")
        return wav
