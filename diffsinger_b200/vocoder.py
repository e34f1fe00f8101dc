"""HiFi-GAN (NSF) generator whose forward runs the sm_90a kernels of libdsx.so (dsx_hifigan_* in include/dsx.h).

``HifiGanGenerator(h, c_out=1)`` keeps the reference's constructor, submodule names and parameter shapes
(modules/hifigan/hifigan.py:30-179), so a reference checkpoint loads strictly, in weight-norm form (``weight_g`` /
``weight_v``) or after ``remove_weight_norm()``.  The modules only hold the parameters: ``forward`` packs them into the
library (once per storage and version, so again after ``load_state_dict``, ``remove_weight_norm`` or ``.to()``) and
runs the whole generator there.  There is no eager or CPU path: a CPU tensor raises ``DsxError``.
"""
import numpy as np
import torch
import torch.nn as nn
from torch.nn import Conv1d, ConvTranspose1d
from torch.nn.utils import remove_weight_norm, weight_norm

from . import _capi
from ._capi import DsxError, check, lib
from .sampler import PackedModule, _need_cuda, _ptr, _stream, _strides_bct

HARMONIC_NUM = 8


def get_padding(kernel_size, dilation=1):
    return int((kernel_size * dilation - dilation) / 2)


def _init_weights(m, mean=0.0, std=0.01):
    if m.__class__.__name__.find("Conv") != -1:
        m.weight.data.normal_(mean, std)


class ResBlock1(nn.Module):
    def __init__(self, h, channels, kernel_size=3, dilation=(1, 3, 5)):
        super().__init__()
        self.h = h
        self.convs1 = nn.ModuleList([weight_norm(Conv1d(channels, channels, kernel_size, 1, dilation=d,
                                                        padding=get_padding(kernel_size, d))) for d in dilation[:3]])
        self.convs1.apply(_init_weights)
        self.convs2 = nn.ModuleList([weight_norm(Conv1d(channels, channels, kernel_size, 1, dilation=1,
                                                        padding=get_padding(kernel_size, 1))) for _ in range(3)])
        self.convs2.apply(_init_weights)

    def remove_weight_norm(self):
        for l in list(self.convs1) + list(self.convs2):
            remove_weight_norm(l)


class ResBlock2(nn.Module):
    def __init__(self, h, channels, kernel_size=3, dilation=(1, 3)):
        super().__init__()
        self.h = h
        self.convs = nn.ModuleList([weight_norm(Conv1d(channels, channels, kernel_size, 1, dilation=d,
                                                       padding=get_padding(kernel_size, d))) for d in dilation[:2]])
        self.convs.apply(_init_weights)

    def remove_weight_norm(self):
        for l in self.convs:
            remove_weight_norm(l)


class SourceModuleHnNSF(nn.Module):
    """Parameters of the NSF harmonic source (modules/parallel_wavegan/models/source.py): l_linear merges the 9 harmonics."""

    def __init__(self, sampling_rate, harmonic_num=HARMONIC_NUM):
        super().__init__()
        self.sampling_rate = sampling_rate
        self.l_linear = nn.Linear(harmonic_num + 1, 1)


class HifiGanGenerator(PackedModule):
    def __init__(self, h, c_out=1):
        super().__init__()
        self.h = h
        self.c_out = c_out
        self.num_kernels = len(h['resblock_kernel_sizes'])
        self.num_upsamples = len(h['upsample_rates'])
        if h['use_pitch_embed']:
            self.harmonic_num = HARMONIC_NUM
            self.f0_upsamp = nn.Upsample(scale_factor=float(np.prod(h['upsample_rates'])))
            self.m_source = SourceModuleHnNSF(sampling_rate=h['audio_sample_rate'], harmonic_num=self.harmonic_num)
            self.noise_convs = nn.ModuleList()
        self.conv_pre = weight_norm(Conv1d(80, h['upsample_initial_channel'], 7, 1, padding=3))
        resblock = ResBlock1 if h['resblock'] == '1' else ResBlock2
        self.ups = nn.ModuleList()
        for i, (u, k) in enumerate(zip(h['upsample_rates'], h['upsample_kernel_sizes'])):
            c_cur = h['upsample_initial_channel'] // (2 ** (i + 1))
            self.ups.append(weight_norm(ConvTranspose1d(c_cur * 2, c_cur, k, u, padding=(k - u) // 2)))
            if h['use_pitch_embed']:
                if i + 1 < len(h['upsample_rates']):
                    s = int(np.prod(h['upsample_rates'][i + 1:]))
                    self.noise_convs.append(Conv1d(1, c_cur, kernel_size=s * 2, stride=s, padding=s // 2))
                else:
                    self.noise_convs.append(Conv1d(1, c_cur, kernel_size=1))
        self.resblocks = nn.ModuleList()
        for i in range(len(self.ups)):
            ch = h['upsample_initial_channel'] // (2 ** (i + 1))
            for k, d in zip(h['resblock_kernel_sizes'], h['resblock_dilation_sizes']):
                self.resblocks.append(resblock(h, ch, k, d))
        self.conv_post = weight_norm(Conv1d(ch, c_out, 7, 1, padding=3))
        self.ups.apply(_init_weights)
        self.conv_post.apply(_init_weights)

    def remove_weight_norm(self):
        for l in self.ups:
            remove_weight_norm(l)
        for l in self.resblocks:
            l.remove_weight_norm()
        remove_weight_norm(self.conv_pre)
        remove_weight_norm(self.conv_post)

    # -- library handle ---------------------------------------------------------------------------
    _lib_create, _lib_load, _lib_destroy = lib.dsx_hifigan_create, lib.dsx_hifigan_load, lib.dsx_hifigan_destroy

    def _config(self):
        h = self.h
        cfg = _capi.HifiganConfig()
        rates, ks = list(h['upsample_rates']), list(h['upsample_kernel_sizes'])
        rk, rd = list(h['resblock_kernel_sizes']), [list(d) for d in h['resblock_dilation_sizes']]
        if not (1 <= len(rates) <= 4 and len(ks) == len(rates) and 1 <= len(rk) <= 3 and len(rd) == len(rk)
                and all(1 <= len(d) for d in rd)):
            raise DsxError("unsupported HiFi-GAN topology: 1..4 upsample stages and 1..3 resblock kernels")
        cfg.num_upsamples = len(rates)
        for i, (u, k) in enumerate(zip(rates, ks)):
            cfg.upsample_rates[i], cfg.upsample_kernel_sizes[i] = int(u), int(k)
        cfg.upsample_initial_channel = int(h['upsample_initial_channel'])
        cfg.resblock = 1 if h['resblock'] == '1' else 2       # as the reference picks the block class
        cfg.num_kernels = len(rk)
        for j, (k, d) in enumerate(zip(rk, rd)):
            cfg.resblock_kernel_sizes[j] = int(k)
            for q, dv in enumerate(d[:3]):
                cfg.resblock_dilation_sizes[j][q] = int(dv)
        cfg.audio_sample_rate = int(h['audio_sample_rate'])
        cfg.use_pitch_embed = 1 if h['use_pitch_embed'] else 0
        return cfg

    def _params(self, sd, t, arr):
        def conv(name):      # (w, g): weight_v / weight_g of a weight-normalised conv, or (weight, NULL)
            if name + ".weight_g" in sd:
                return t(name + ".weight_v"), t(name + ".weight_g")
            return t(name + ".weight"), None

        nu, nk = self.num_upsamples, self.num_kernels
        per_block = ["convs1.0", "convs1.1", "convs1.2", "convs2.0", "convs2.1", "convs2.2"] \
            if self.h['resblock'] == '1' else ["convs.0", "convs.1"]
        ups = [conv(f"ups.{i}") for i in range(nu)]
        rb_names = [f"resblocks.{b}.{c}" for b in range(nu * nk) for c in per_block]
        rb = [conv(n) for n in rb_names]
        pre_w, pre_g = conv("conv_pre")
        post_w, post_g = conv("conv_post")
        p = _capi.HifiganParams(
            conv_pre_w=pre_w, conv_pre_g=pre_g, conv_pre_b=t("conv_pre.bias"),
            ups_w=arr([w for w, _ in ups]), ups_g=arr([g for _, g in ups]), ups_b=arr([f"ups.{i}.bias" for i in range(nu)]),
            rb_w=arr([w for w, _ in rb]), rb_g=arr([g for _, g in rb]), rb_b=arr([n + ".bias" for n in rb_names]),
            conv_post_w=post_w, conv_post_g=post_g, conv_post_b=t("conv_post.bias"))
        if self.h['use_pitch_embed']:
            p.noise_w = arr([f"noise_convs.{i}.weight" for i in range(nu)])
            p.noise_b = arr([f"noise_convs.{i}.bias" for i in range(nu)])
            p.source_w, p.source_b = t("m_source.l_linear.weight"), t("m_source.l_linear.bias")
        return p

    def forward(self, x, f0=None, *, lengths=None, phase0=None, src_noise=None, seed=0):
        """x: mel [B, 80, T] (any strides); f0: [B, T] Hz or None; lengths: [B] frames or None; phase0 [B, 9] and
        src_noise [B, T * hop, 9] replace the in-kernel Philox draws of the NSF source.  -> wav [B, 1, T * hop]."""
        if x.dim() != 3 or x.shape[1] != 80:
            raise DsxError(f"mel must be [B, 80, T] (got {tuple(x.shape)}); pass dsx_infer's [B, T, 80] output as "
                           ".transpose(1, 2)")
        _need_cuda(x, f0, lengths, phase0, src_noise)
        if self.c_out != 1:
            raise DsxError(f"the dsx vocoder writes one waveform channel (c_out = {self.c_out})")
        dev = x.device
        hnd = self._ensure(dev)
        B, _, T = x.shape
        hop = int(np.prod(self.h['upsample_rates']))
        mel = x.float()
        c = lambda v: None if v is None else v.to(device=dev, dtype=torch.float32).contiguous()
        f0, phase0, src_noise = c(f0), c(phase0), c(src_noise)
        lens = None if lengths is None else lengths.to(device=dev, dtype=torch.int32).contiguous()
        for name, v, shape in (("f0", f0, (B, T)), ("lengths", lens, (B,)), ("phase0", phase0, (B, HARMONIC_NUM + 1)),
                               ("src_noise", src_noise, (B, T * hop, HARMONIC_NUM + 1))):
            if v is not None and tuple(v.shape) != shape:
                raise DsxError(f"{name} must have shape {shape} (got {tuple(v.shape)})")
        wav = torch.empty((B, 1, T * hop), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib.dsx_hifigan_forward(hnd, _ptr(mel), _strides_bct(mel, (0, 1, 2)), _ptr(f0), _ptr(lens), _ptr(phase0),
                                          _ptr(src_noise), int(seed), B, T, _ptr(wav), _stream(dev)), "dsx_hifigan_forward")
        return wav
