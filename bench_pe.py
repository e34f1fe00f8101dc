"""Throughput of the pitch extractor on one GPU: mel frames per second at hidden_size 256.

    python bench_pe.py [--iters N] [--kernels]

Two sizes: B = 16, T = 1024 (a batch) and B = 1, T = 2000 (one sung phrase at hop 128).  The model is the shipped
e2e configuration (hidden_size 256, predictor_kernel 5, two GroupNorm conv blocks, 'SAME' padding, log pitch with uv)
with seeded weights and normalisation parameters; the second utterance of the batch has a zero-padded tail.  Times come
from CUDA events around whole calls.  Baselines in the same process: the reference's pitch extractor
(oracle/pe_oracle.py, the ATen ops the reference runs, the position table cached as the module caches it) in PyTorch
eager -- fp32 with TF32 off, fp32 with cuDNN's defaults (TF32 convolutions: what the reference runs on an H100), and
`.half()`.  The dsx output is compared with the eager fp32 TF32-off output.  Share of peak is the FLOP floor
(flops_per_frame at 989 TFLOP/s, the H100 SXM data-sheet dense FP16 rate) over the measured time.  --kernels adds the
summed device time per kernel name of one dsx call (torch.profiler).  The card's name, power limit and max SM clock are
read once; the SM clock again right after each dsx loop.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import re
import subprocess

import torch

import diffsinger_b200 as dsx
from oracle import pe_oracle as O

PEAK_FLOPS = 989e12
SIZES = ((16, 1024), (1, 2000))


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
            m = re.search(r"k_\w+(<\d+>)?", ev.name)
            name = m.group(0) if m else ev.name[:60]
            tot[name] = tot.get(name, 0.0) + ev.device_time_total / 1e3
    return {k: round(v, 3) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])}


def run_size(B, T, iters, kernels):
    dev = torch.device("cuda", 0)
    hp, L = dict(O.HPARAMS_E2E), 2
    torch.manual_seed(0)
    pe = dsx.PitchExtractor(80, L, hparams=hp)
    sd = O.random_state_dict(pe.state_dict(), 1)
    pe.load_state_dict(sd, strict=True)
    pe = pe.eval().to(dev)
    mel = (torch.randn(B, T, 80, generator=torch.Generator().manual_seed(2)) * 1.5 - 4.0).to(dev)
    if B > 1:
        mel[1, T - T // 4:] = 0
    table = O.sinusoidal_table(max(4096, T + 1), hp["hidden_size"])
    with torch.no_grad():
        t_dsx, _ = timed(lambda: pe(mel), iters)
        sm_clock = gpu_info("clocks.sm")      # read right after the timed loop, while the clock is still under load
        out = pe(mel)
        sd32 = {k: v.to(dev) for k, v in sd.items()}
        sd16 = {k: (v.to(dev).half() if v.is_floating_point() else v.to(dev)) for k, v in sd.items()}
        tab32, tab16 = table.to(dev), table.to(dev).half()
        eager = lambda s, m, t: O.pitch_extractor(s, m, hp, L, table=t)
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = False, False
        t32, ref = timed(lambda: eager(sd32, mel, tab32), iters)
        torch.backends.cudnn.allow_tf32 = True                 # cuDNN's default: TF32 convolutions
        t_tf32, ref_tf32 = timed(lambda: eager(sd32, mel, tab32), iters)
        t16, ref16 = timed(lambda: eager(sd16, mel.half(), tab16), iters)
        torch.backends.cudnn.allow_tf32 = False
    err = lambda a: {f"ch{c}": [round((a[..., c].float() - ref[0][..., c]).abs().max().item(), 5),
                                round((a[..., c].float() - ref[0][..., c]).abs().mean().item(), 6)] for c in range(2)}
    fps = lambda ms: round(B * T / (ms / 1e3))
    flops = O.flops_per_frame() * B * T
    res = dict(B=B, T=T, sm_clock_after_dsx_loop=sm_clock, dsx_ms=round(t_dsx, 3), eager_fp32_ms=round(t32, 3),
               eager_cudnn_default_ms=round(t_tf32, 3), eager_fp16_ms=round(t16, 3), mel_frames_per_s=fps(t_dsx),
               eager_fp32_frames_per_s=fps(t32), eager_cudnn_default_frames_per_s=fps(t_tf32), eager_fp16_frames_per_s=fps(t16),
               speedup_vs_eager_fp32=round(t32 / t_dsx, 2), speedup_vs_eager_cudnn_default=round(t_tf32 / t_dsx, 2),
               speedup_vs_eager_fp16=round(t16 / t_dsx, 2), flops_per_frame=O.flops_per_frame(),
               share_of_fp16_peak=round(flops / PEAK_FLOPS / (t_dsx / 1e3), 4),
               dsx_err_vs_fp32=err(out['pitch_pred']), cudnn_default_err_vs_fp32=err(ref_tf32[0]), fp16_err_vs_fp32=err(ref16[0]))
    if kernels:
        with torch.no_grad():
            res["dsx_kernel_ms"] = kernel_times(lambda: pe(mel))
    pe.close()
    del sd32, sd16, ref, ref_tf32, ref16, out
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pe.py needs a CUDA device")
    out = dict(metric="pitch_extractor", hidden_size=256, gpu=gpu_info(),
               sizes=[run_size(B, T, a.iters, a.kernels) for B, T in SIZES])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
