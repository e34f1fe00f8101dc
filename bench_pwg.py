"""Throughput of the Parallel WaveGAN vocoder on one GPU: the shipped generator (configs/tts/pwg.yaml: 30 layers, 3 stacks,
hop 256, aux_context_window 2) at 22.05 kHz.

    python bench_pwg.py [--iters N] [--kernels]

Two workloads: B = 16, T = 1024 (the batch of bench_vocoder.py) and B = 1, T = 800 (the single-utterance call
vocoders/pwg.py:spec2wav makes).  Times come from CUDA events around whole generator calls.  Baselines in the same
process: the reference's generator (oracle/pwg_oracle.py, the ATen ops the reference runs) in PyTorch eager, fp32 with
TF32 off, and the same in fp16.  The dsx output is compared with the eager fp32 output at the timed size against the
bound test_gpu_pwg.py sets for the shipped topology.  Share of peak is the larger of the FLOP floor (flops_per_sample at
989 TFLOP/s, the H100 SXM data-sheet dense FP16 rate) and the compulsory-bytes floor (z, c and wav at 3.35 TB/s) over
the measured time.  --kernels adds the summed device time per kernel name of one dsx call (torch.profiler).  The card's
name, power limit and max SM clock are read once; the SM clock again right after each dsx loop.  Prints one JSON line;
writes nothing.
"""
import argparse
import json
import re
import subprocess

import numpy as np
import torch

import diffsinger_b200 as dsx
from oracle import pwg_oracle as P

PEAK_FLOPS, PEAK_BW = 989e12, 3.35e12
SAMPLE_RATE = 22050
BOUND_MAX, BOUND_MEAN = 3 * 7e-4, 3 * 1.3e-4      # test_gpu_pwg.py, the shipped topology (relative to the peak)
WORKLOADS = ((16, 1024), (1, 800))


def gpu_info(q="name,power.limit,clocks.max.sm"):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


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
            m = re.search(r"k_\w+", ev.name)
            name = m.group(0) if m else ev.name[:60]
            tot[name] = tot.get(name, 0.0) + ev.device_time_total / 1e3
    return {k: round(v, 3) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])}


def run(B, T, iters, kernels):
    dev = torch.device("cuda", 0)
    cfg = P.CONFIG_SHIPPED
    hop, w = P.hop(cfg), cfg["aux_context_window"]
    torch.manual_seed(0)
    gen_mod = dsx.ParallelWaveGANGenerator(**cfg)
    sd = {k: v.detach().clone() for k, v in gen_mod.state_dict().items()}
    gen_mod = gen_mod.eval().to(dev)
    g = torch.Generator().manual_seed(1)
    z = torch.randn(B, 1, T * hop, generator=g).to(dev)
    mel = torch.randn(B, T, 80, generator=g)
    c = torch.from_numpy(np.pad(mel.numpy(), ((0, 0), (w, w), (0, 0)), "edge")).to(dev).transpose(1, 2)
    with torch.no_grad():
        t_dsx, _ = timed(lambda: gen_mod(z, c), iters)
        sm_clock = gpu_info("clocks.sm")      # read right after the timed loop, while the clock is still under load
        wav = gen_mod(z, c)
        plain = {k: v.to(dev) for k, v in sd.items() if not k.endswith((".weight_g", ".weight_v"))}
        for k in sd:
            if k.endswith(".weight_g"):
                name = k[:-len(".weight_g")]
                plain[name + ".weight"] = P.conv_weight(sd, name).to(dev)
        sd16 = {k: v.half() for k, v in plain.items()}
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        t32, ref = timed(lambda: P.generator(plain, cfg, z, c), max(1, iters // 4))
        t16, _ = timed(lambda: P.generator(sd16, cfg, z.half(), c.half()), max(1, iters // 2))
        d = (wav - ref).abs()
        peak = ref.abs().max().item()
    fps = P.flops_per_sample(cfg)
    samples = B * T * hop
    bytes_ = (samples * 2 + B * (T + 2 * w) * 80) * 4
    floor_f, floor_b = fps * samples / PEAK_FLOPS, bytes_ / PEAK_BW
    res = dict(B=B, T=T, sm_clock_after_dsx_loop=sm_clock, dsx_ms=round(t_dsx, 3), eager_fp32_ms=round(t32, 3),
               eager_fp16_ms=round(t16, 3), mel_frames_per_s=round(B * T / (t_dsx / 1e3)),
               audio_s_per_s=round(samples / SAMPLE_RATE / (t_dsx / 1e3), 1),
               speedup_vs_eager_fp32=round(t32 / t_dsx, 2), speedup_vs_eager_fp16=round(t16 / t_dsx, 2),
               flops_per_sample=fps, share_of_peak=round(max(floor_f, floor_b) / (t_dsx / 1e3), 4),
               bound="flops" if floor_f >= floor_b else "bytes",
               max_abs_diff_vs_fp32=d.max().item(), mean_abs_diff_vs_fp32=d.mean().item(), ref_peak=peak,
               within_bound=bool(d.max().item() <= BOUND_MAX * peak and d.mean().item() <= BOUND_MEAN * peak))
    if kernels:
        with torch.no_grad():
            res["dsx_kernel_ms"] = kernel_times(lambda: gen_mod(z, c))
    del plain, sd16, ref, wav
    gen_mod.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pwg.py needs a CUDA device")
    out = dict(metric="pwg_vocoder", gpu=gpu_info(), workloads=[run(B, T, a.iters, a.kernels) for B, T in WORKLOADS])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
