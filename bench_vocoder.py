"""Throughput of the HiFi-GAN (NSF) vocoder on one GPU: mel frames and audio seconds per second at B = 16, T = 1024.

    python bench_vocoder.py [--iters N] [--kernels]

Two widths, both with f0 and the rates of configs/tts/hifigan.yaml (hop 256): 128 is that config; 512 stands in for a large
NSF checkpoint.  Times come from CUDA events around whole generator calls.  Baselines in the same process: the
reference's generator (oracle/hifigan_oracle.py, the ATen ops the reference runs) in PyTorch eager, fp32 with TF32
off, and the same in fp16.  The dsx output is compared with the eager fp32 output at the timed size, with the draws of
the NSF source injected so both see the same noise.  Share of peak is the larger of the FLOP floor (flops_per_frame at
989 TFLOP/s, the H100 SXM data-sheet dense FP16 rate) and the compulsory-bytes floor (mel + f0 in, wav out at 3.35 TB/s)
over the measured time.  --kernels adds the summed device time per kernel name of one dsx call (torch.profiler).
Width 128 runs every ResBlock through the chained kernel (stage widths 64 / 32 / 16 / 8); width 512 runs its first two
stages (256 and 128 channels) one launch per conv and its last two chained, so the benchmark covers both sides of that
choice.  The card's name, power limit and max SM clock are read once; the SM clock again right after each dsx loop.
Prints one JSON line; writes nothing.
"""
import argparse
import json
import re
import subprocess

import numpy as np
import torch
import torch.nn.functional as F

import diffsinger_b200 as dsx
from oracle import hifigan_oracle as H

PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12
B, T = 16, 1024


def gpu_info(q="name,power.limit,clocks.max.sm"):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def eager(sd, h, mel, har):
    """HifiGanGenerator.forward in eager PyTorch (the oracle's restatement) in the dtype of sd / mel; the NSF source
    `har` [B, 1, L] is computed in fp32 beforehand (it is not a conv) and cast."""
    block = H.resblock1 if h["resblock"] == "1" else H.resblock2
    rates, nk = h["upsample_rates"], len(h["resblock_kernel_sizes"])
    har = har.to(mel.dtype)
    x = F.conv1d(mel, H.conv_weight(sd, "conv_pre"), sd["conv_pre.bias"], padding=3)
    for i, (u, k) in enumerate(zip(rates, h["upsample_kernel_sizes"])):
        x = F.conv_transpose1d(F.leaky_relu(x, H.LRELU_SLOPE), H.conv_weight(sd, f"ups.{i}"), sd[f"ups.{i}.bias"], stride=u,
                               padding=(k - u) // 2)
        s = int(np.prod(rates[i + 1:])) if i + 1 < len(rates) else 1
        x = x + F.conv1d(har, sd[f"noise_convs.{i}.weight"], sd[f"noise_convs.{i}.bias"], stride=s,
                         padding=s // 2 if i + 1 < len(rates) else 0)
        xs = None
        for j, (rk, rd) in enumerate(zip(h["resblock_kernel_sizes"], h["resblock_dilation_sizes"])):
            r = block(sd, f"resblocks.{i * nk + j}", x, rk, rd)
            xs = r if xs is None else xs + r
        x = xs / nk
    return torch.tanh(F.conv1d(F.leaky_relu(x), H.conv_weight(sd, "conv_post"), sd["conv_post.bias"], padding=3))


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, out


def kernel_times(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tot = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            m = re.search(r"k_\w+(<\d+>)?", ev.name)
            name = m.group(0) if m else ev.name[:60]
            tot[name] = tot.get(name, 0.0) + ev.device_time_total / 1e3
    return {k: round(v, 3) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])}


def run_width(width, iters, kernels):
    dev = torch.device("cuda", 0)
    h = dict(H.HPARAMS_TTS, upsample_initial_channel=width)
    hop = int(np.prod(h["upsample_rates"]))
    torch.manual_seed(0)
    gen_mod = dsx.HifiGanGenerator(h)
    sd = {k: v.detach().clone() for k, v in gen_mod.state_dict().items()}
    gen_mod = gen_mod.to(dev)
    g = torch.Generator().manual_seed(1)
    mel = torch.randn(B, 80, T, generator=g).to(dev)
    f0 = (torch.rand(B, T, generator=g) * 300 + 100).to(dev)
    f0[:, 100:140] = 0
    torch.manual_seed(2)
    ph = torch.rand(B, 9, device=dev)
    ph[:, 0] = 0
    noise = torch.randn(B, T * hop, 9, device=dev)

    with torch.no_grad():
        t_dsx, _ = timed(lambda: gen_mod(mel, f0, seed=3), iters)
        sm_clock = gpu_info("clocks.sm")      # read right after the timed loop, while the clock is still under load
        wav = gen_mod(mel, f0, phase0=ph, src_noise=noise)
        # the NSF source of the eager baseline, with the same draws
        f0_up = f0[:, :, None].repeat_interleave(hop, dim=1)
        rad = (f0_up * torch.arange(1, 10, device=dev, dtype=torch.float32) / h["audio_sample_rate"]) % 1
        rad[:, 0, :] += ph
        over = torch.cumsum(rad, 1) % 1
        shift = torch.zeros_like(rad)
        shift[:, 1:, :] = ((over[:, 1:, :] - over[:, :-1, :]) < 0) * -1.0
        uv = (f0_up > 0).float()
        sines = torch.sin(torch.cumsum(rad + shift, 1) * 2 * np.pi) * 0.1
        src = sines * uv + (uv * 0.003 + (1 - uv) * 0.1 / 3) * noise
        har = torch.tanh(F.linear(src, sd["m_source.l_linear.weight"].to(dev), sd["m_source.l_linear.bias"].to(dev))).transpose(1, 2)
        sd32 = {k: v.to(dev) for k, v in sd.items()}
        sd16 = {k: v.to(dev).half() for k, v in sd.items()}
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        t32, ref = timed(lambda: eager(sd32, h, mel, har), max(1, iters // 4))
        t16, _ = timed(lambda: eager(sd16, h, mel.half(), har), max(1, iters // 2))
        d = (wav - ref).abs()
        peak = ref.abs().max().item()
    flops = H.flops_per_frame(h) * B * T
    bytes_ = (B * T * 80 + B * T + B * T * hop) * 4
    floor_f, floor_b = flops / PEAK_FLOPS, bytes_ / PEAK_BW
    res = dict(width=width, sm_clock_after_dsx_loop=sm_clock, dsx_ms=round(t_dsx, 3), eager_fp32_ms=round(t32, 3), eager_fp16_ms=round(t16, 3),
               mel_frames_per_s=round(B * T / (t_dsx / 1e3)), audio_s_per_s=round(B * T * hop / h["audio_sample_rate"] / (t_dsx / 1e3), 1),
               speedup_vs_eager_fp32=round(t32 / t_dsx, 2), speedup_vs_eager_fp16=round(t16 / t_dsx, 2),
               flops_per_frame=H.flops_per_frame(h), share_of_peak=round(max(floor_f, floor_b) / (t_dsx / 1e3), 4),
               bound="flops" if floor_f >= floor_b else "bytes",
               max_abs_diff_vs_fp32=d.max().item(), mean_abs_diff_vs_fp32=d.mean().item(), ref_peak=peak,
               within_bound=bool(d.max().item() <= 4e-3 * peak and d.mean().item() <= 1e-3 * peak))
    if kernels:
        with torch.no_grad():
            res["dsx_kernel_ms"] = kernel_times(lambda: gen_mod(mel, f0, seed=3))
    del sd32, sd16, ref, wav, noise, har
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vocoder.py needs a CUDA device")
    out = dict(metric="hifigan_nsf_vocoder", B=B, T=T, gpu=gpu_info(),
               widths=[run_width(w, a.iters, a.kernels) for w in (128, 512)])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
