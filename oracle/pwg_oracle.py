"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the reference's Parallel WaveGAN generator, the vocoder that
configs/tts/base.yaml selects (`vocoder: pwg`) and vocoders/pwg.py runs.

Functional torch-CPU fp32 (the ATen kernels the reference itself runs), every function citing the reference lines it
restates.  Pinned: oracle/gen_golden_pwg.py imports the live reference and asserts bit-exact agreement;
tests/test_oracle_pwg.py re-checks the committed fixtures.

    generator(sd, cfg, z, c, pitch=None)  modules/parallel_wavegan/models/parallel_wavegan.py:139-172  forward
    upsample(sd, cfg, c)                  modules/parallel_wavegan/layers/upsample.py:107-183  ConvInUpsampleNetwork
    residual_block(...)                   modules/parallel_wavegan/layers/residual_block.py:94-129  ResidualBlock.forward
"""
import math

import torch
import torch.nn.functional as F

# configs/tts/pwg.yaml generator_params (the shipped generator)
CONFIG_SHIPPED = dict(in_channels=1, out_channels=1, kernel_size=3, layers=30, stacks=3, residual_channels=64,
                      gate_channels=128, skip_channels=64, aux_channels=80, aux_context_window=2, dropout=0.0,
                      use_weight_norm=True, upsample_net="ConvInUpsampleNetwork",
                      upsample_params={"upsample_scales": [4, 4, 4, 4]}, use_pitch_embed=False)


def conv_weight(sd, name):
    """weight of a (possibly weight-normalised) conv: w = g * v / ||v|| over every dim but 0 (torch.nn.utils.weight_norm,
    dim=0, as parallel_wavegan.py:182-189 applies it to every Conv1d and Conv2d); plain `.weight` after
    remove_weight_norm()."""
    if name + ".weight" in sd:
        return sd[name + ".weight"]
    return torch._weight_norm(sd[name + ".weight_v"], sd[name + ".weight_g"], 0)      # the ATen op the reference's hook calls


def scales(cfg):
    return list(cfg["upsample_params"]["upsample_scales"])


def hop(cfg):
    return math.prod(scales(cfg))


def _round(fp16):
    """fp16=True: a GEMM operand as the dsx kernels read it, rounded to fp16 (and back to the tensor's own dtype)"""
    return (lambda t: t.half().to(t.dtype)) if fp16 else (lambda t: t)


def upsample(sd, cfg, c):
    """ConvInUpsampleNetwork.forward (upsample.py:169-183): conv_in (no padding: the caller edge-pads c by
    aux_context_window frames), then UpsampleNetwork.forward (:107-124): per scale s, Stretch2d (nearest, :33-45) and
    Conv2d(1, 1, (1, 2s + 1), padding (0, s), bias=False)."""
    c = F.conv1d(c, conv_weight(sd, "upsample_net.conv_in"), None)
    c = c.unsqueeze(1)
    for i, s in enumerate(scales(cfg)):
        c = F.interpolate(c, scale_factor=(1, s), mode="nearest")
        c = F.conv2d(c, conv_weight(sd, f"upsample_net.upsample.up_layers.{2 * i + 1}"), None, padding=(0, s))
    return c.squeeze(1)


def residual_block(sd, pre, x, c, dilation, fp16=False):
    """ResidualBlock.forward in eval mode (residual_block.py:94-129; dropout is the identity): -> (x, s)."""
    r = _round(fp16)
    residual = x
    x = F.conv1d(r(x), r(conv_weight(sd, f"{pre}.conv")), sd[f"{pre}.conv.bias"], padding=dilation, dilation=dilation)
    xa, xb = x.split(x.size(1) // 2, dim=1)
    c = F.conv1d(r(c), r(conv_weight(sd, f"{pre}.conv1x1_aux")), None)
    ca, cb = c.split(c.size(1) // 2, dim=1)
    xa, xb = xa + ca, xb + cb
    x = torch.tanh(xa) * torch.sigmoid(xb)
    s = F.conv1d(r(x), r(conv_weight(sd, f"{pre}.conv1x1_skip")), sd[f"{pre}.conv1x1_skip.bias"])
    x = (F.conv1d(r(x), r(conv_weight(sd, f"{pre}.conv1x1_out")), sd[f"{pre}.conv1x1_out.bias"]) + residual) * math.sqrt(0.5)
    return x, s


def generator(sd, cfg, z, c, pitch=None, fp16=False):
    """ParallelWaveGANGenerator.forward (parallel_wavegan.py:139-172): z [B, 1, T * hop], c [B, aux, T + 2w] (edge-padded
    by w = aux_context_window, as vocoders/pwg.py:91-93 does), pitch int64 [B, T + 2w] or None -> wav [B, 1, T * hop].
    pitch is read only with use_pitch_embed, as in the reference.
    fp16=True: the x taps, the upsampled c, the gate output z and the weights of the residual layers' GEMMs rounded to
    fp16, as the dsx kernels read them; the conditioning network, first_conv, the sums and the head stay fp32."""
    if cfg.get("use_pitch_embed"):
        p = F.embedding(pitch, sd["pitch_embed.weight"], 0)
        c = F.linear(torch.cat([c.transpose(1, 2), p], -1), sd["c_proj.weight"], sd["c_proj.bias"]).transpose(1, 2)
    c = upsample(sd, cfg, c)
    assert c.size(-1) == z.size(-1), (c.size(-1), z.size(-1))
    x = F.conv1d(z, conv_weight(sd, "first_conv"), sd["first_conv.bias"])
    layers, lps = cfg["layers"], cfg["layers"] // cfg["stacks"]
    skips = 0
    for l in range(layers):
        x, h = residual_block(sd, f"conv_layers.{l}", x, c, 2 ** (l % lps), fp16)
        skips += h
    skips *= math.sqrt(1.0 / layers)
    x = F.relu(skips)
    x = F.conv1d(x, conv_weight(sd, "last_conv_layers.1"), sd["last_conv_layers.1.bias"])
    x = F.relu(x)
    return F.conv1d(x, conv_weight(sd, "last_conv_layers.3"), sd["last_conv_layers.3.bias"])


def flops_per_sample(cfg):
    """Algorithmic FLOPs of one output sample (2 per multiply-add): the residual layers, the head, first_conv and the
    conditioning network (frame-rate work spread over hop samples).  The roofline numerator of bench_pwg.py."""
    R, G, S, A = cfg["residual_channels"], cfg["gate_channels"], cfg["skip_channels"], cfg["aux_channels"]
    k, w, sc = cfg["kernel_size"], cfg["aux_context_window"], scales(cfg)
    layer = 2 * G * R * k + 2 * G * A + 2 * (G // 2) * (R + S)
    head = 2 * S * S + 2 * S * cfg["out_channels"]
    first = 2 * R
    frame = 2 * A * A * (2 * w + 1) + (2 * (2 * A) * A if cfg.get("use_pitch_embed") else 0)
    up, f = 0.0, 1
    for s in sc:
        f *= s
        up += f * 2 * (2 * s + 1) * A          # per frame: stage output samples x (2s + 1) taps x aux channels
    return cfg["layers"] * layer + head + first + (frame + up) / hop(cfg)
