"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's HiFi-GAN (NSF) generator, the next row of the hot-path
scope table (the vocoder that follows the sampler).  No kernel exists for it yet; this file and
tests/golden/hifigan_*.npz pin the algorithm so that a kernel can be held to it.

Functional torch-CPU fp32 (the ATen kernels the reference itself runs), every function citing the reference lines it
restates.  Pinned: oracle/gen_golden_hifigan.py imports the live reference and asserts bit-exact agreement (same RNG stream
for the NSF source's random phase / noise draws); tests/test_oracle_hifigan.py re-checks the committed fixtures.

    generator(sd, h, mel, f0=None)        modules/hifigan/hifigan.py:104-171   HifiGanGenerator.forward
    resblock1 / resblock2                  modules/hifigan/hifigan.py:30-99
    nsf_source(sd, f0_up, rate, ...)       modules/parallel_wavegan/models/source.py  SineGen.forward + SourceModuleHnNSF.forward
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

LRELU_SLOPE = 0.1          # hifigan.py:11


def conv_weight(sd, name):
    """weight of a (possibly weight-normalised) conv: w = g * v / ||v|| over every dim but 0 (torch.nn.utils.weight_norm,
    dim=0, as applied in hifigan.py:33-49,117,125,143); plain `.weight` after remove_weight_norm()."""
    if name + ".weight" in sd:
        return sd[name + ".weight"]
    return torch._weight_norm(sd[name + ".weight_v"], sd[name + ".weight_g"], 0)      # the ATen op the reference's hook calls


def get_padding(kernel_size, dilation=1):                      # hifigan.py:26-27
    return int((kernel_size * dilation - dilation) / 2)


def resblock1(sd, pre, x, k, dil):
    """ResBlock1.forward, hifigan.py:54-62 (note `x = xt + x` is executed once per pair in the reference)."""
    for j, d in enumerate(dil):
        xt = F.leaky_relu(x, LRELU_SLOPE)
        xt = F.conv1d(xt, conv_weight(sd, f"{pre}.convs1.{j}"), sd[f"{pre}.convs1.{j}.bias"], dilation=d, padding=get_padding(k, d))
        xt = F.leaky_relu(xt, LRELU_SLOPE)
        xt = F.conv1d(xt, conv_weight(sd, f"{pre}.convs2.{j}"), sd[f"{pre}.convs2.{j}.bias"], dilation=1, padding=get_padding(k, 1))
        x = xt + x
    return x


def resblock2(sd, pre, x, k, dil):
    """ResBlock2.forward, hifigan.py:85-90."""
    for j, d in enumerate(dil):
        xt = F.leaky_relu(x, LRELU_SLOPE)
        xt = F.conv1d(xt, conv_weight(sd, f"{pre}.convs.{j}"), sd[f"{pre}.convs.{j}.bias"], dilation=d, padding=get_padding(k, d))
        x = xt + x
    return x


def sine_gen(f0, rate, harmonic_num, sine_amp=0.1, noise_std=0.003, voiced_threshold=0.0):
    """SineGen.forward with flag_for_pulse=False (source.py:44-74,105-134).  f0 [B, L, 1] -> (sine_waves [B, L, H+1], uv).
    Draws, in the reference's order: torch.rand(B, H+1) (initial phases), torch.randn_like(sine_waves) (additive noise)."""
    B, L, _ = f0.shape
    dim = harmonic_num + 1
    f0_buf = torch.zeros(B, L, dim)
    f0_buf[:, :, 0] = f0[:, :, 0]
    for idx in range(harmonic_num):
        f0_buf[:, :, idx + 1] = f0_buf[:, :, 0] * (idx + 2)
    rad_values = (f0_buf / rate) % 1
    rand_ini = torch.rand(B, dim)
    rand_ini[:, 0] = 0
    rad_values[:, 0, :] = rad_values[:, 0, :] + rand_ini
    tmp_over_one = torch.cumsum(rad_values, 1) % 1
    tmp_over_one_idx = (tmp_over_one[:, 1:, :] - tmp_over_one[:, :-1, :]) < 0
    cumsum_shift = torch.zeros_like(rad_values)
    cumsum_shift[:, 1:, :] = tmp_over_one_idx * -1.0
    sines = torch.sin(torch.cumsum(rad_values + cumsum_shift, dim=1) * 2 * np.pi)
    sine_waves = sines * sine_amp
    uv = torch.ones_like(f0) * (f0 > voiced_threshold)
    noise_amp = uv * noise_std + (1 - uv) * sine_amp / 3
    noise = noise_amp * torch.randn_like(sine_waves)
    return sine_waves * uv + noise, uv


def nsf_source(sd, f0_up, rate, harmonic_num=8, sine_amp=0.1):
    """SourceModuleHnNSF.forward (source.py: l_sin_gen -> l_linear -> tanh; then one more torch.randn_like(uv) draw for the
    noise branch, which the generator does not use but which advances the RNG)."""
    sine_wavs, uv = sine_gen(f0_up, rate, harmonic_num, sine_amp)
    sine_merge = torch.tanh(F.linear(sine_wavs, sd["m_source.l_linear.weight"], sd["m_source.l_linear.bias"]))
    noise = torch.randn_like(uv) * sine_amp / 3
    return sine_merge, noise, uv


def generator(sd, h, mel, f0=None):
    """HifiGanGenerator.forward (hifigan.py:149-171): mel [B, 80, T] (+ f0 [B, T] in Hz, 0 = unvoiced) -> wav [B, 1, T * prod(rates)]."""
    rates, ksz = h["upsample_rates"], h["upsample_kernel_sizes"]
    nk = len(h["resblock_kernel_sizes"])
    block = resblock1 if h["resblock"] == "1" else resblock2
    har = None
    if f0 is not None:
        up = int(np.prod(rates))
        f0_up = F.interpolate(f0[:, None], scale_factor=float(up), mode="nearest").transpose(1, 2)     # torch.nn.Upsample, :115,152
        har, _, _ = nsf_source(sd, f0_up, h["audio_sample_rate"])
        har = har.transpose(1, 2)
    x = F.conv1d(mel, conv_weight(sd, "conv_pre"), sd["conv_pre.bias"], padding=3)
    for i, (u, k) in enumerate(zip(rates, ksz)):
        x = F.leaky_relu(x, LRELU_SLOPE)
        x = F.conv_transpose1d(x, conv_weight(sd, f"ups.{i}"), sd[f"ups.{i}.bias"], stride=u, padding=(k - u) // 2)
        if har is not None:
            if i + 1 < len(rates):
                s = int(np.prod(rates[i + 1:]))
                x = x + F.conv1d(har, sd[f"noise_convs.{i}.weight"], sd[f"noise_convs.{i}.bias"], stride=s, padding=s // 2)
            else:
                x = x + F.conv1d(har, sd[f"noise_convs.{i}.weight"], sd[f"noise_convs.{i}.bias"])
        xs = None
        for j, (rk, rd) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
            r = block(sd, f"resblocks.{i * nk + j}", x, rk, rd)
            xs = r if xs is None else xs + r
        x = xs / nk
    x = F.leaky_relu(x)                                   # (default slope 0.01, as the reference: hifigan.py:167)
    x = F.conv1d(x, conv_weight(sd, "conv_post"), sd["conv_post.bias"], padding=3)
    return torch.tanh(x)


def flops_per_frame(h, c_in=80):
    """Algorithmic FLOPs of one mel frame through the generator (2 per multiply-add): the roofline numerator a kernel would
    be measured against."""
    c = h["upsample_initial_channel"]
    total, per_frame = 2 * c_in * c * 7, 1
    for u, k in zip(h["upsample_rates"], h["upsample_kernel_sizes"]):
        c_out = c // 2
        per_frame *= u
        total += per_frame * 2 * c * c_out * k / u                   # transposed conv: k / u taps per output sample
        for rk, rd in zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"]):
            n_conv = 2 * len(rd) if h["resblock"] == "1" else len(rd)
            total += per_frame * n_conv * 2 * c_out * c_out * rk
        c = c_out
    total += per_frame * 2 * c * 7
    return total


HPARAMS_TTS = dict(resblock="1", upsample_rates=[8, 8, 2, 2], upsample_kernel_sizes=[16, 16, 4, 4], upsample_initial_channel=128,
                   resblock_kernel_sizes=[3, 7, 11], resblock_dilation_sizes=[[1, 3, 5]] * 3, use_pitch_embed=True,
                   audio_sample_rate=24000)     # configs/tts/hifigan.yaml:3-10 + the NSF switch the singing vocoder sets
