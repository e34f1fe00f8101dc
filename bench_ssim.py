"""Times the SSIM mel loss (FastSpeech2Task.ssim_loss's ssim(), modules/commons/ssim.py:383-391) forward + backward on dsx
against eager PyTorch in fp32 with TF32 off and under PyTorch's defaults (cuDNN convolutions in TF32), and one training
step of the dsx FastSpeech2 decoder (dsx_train) + mel_out + the singing configs' `ssim:0.5|l1:0.5` mel loss as
add_mel_loss computes it + backward, with the SSIM half eager (defaults), on dsx, and left out (the L1 half alone), so
the SSIM share of the step is (with - without) / with.

Sizes: 32 x 1000, 16 x 1024 and 4 x 4500 mel frames of 80 bins (LJ's 32k-frame batches, singing segments) and
32 x 1000 x 10 (cwt_loss over 10 CWT scales).  The least time the hardware allows per SSIM call is the larger of its
bytes (x, y read twice, map, d_map, d_x, d_y: 32 per pixel) over 3.35 TB/s and its fp32 operations (FLOPS_PER_PIXEL,
counting an FMA as two) over 67 TFLOP/s, the H100 SXM data-sheet figures at 700 W.  Prints one JSON line with the
card, its power limit and SM clock.  --kernels adds per-kernel CUDA times from torch.profiler for one dsx call at
each size, so the kernels can be told apart from the host's share of the call.

    python bench_ssim.py [--steps 20] [--warmup 5] [--kernels]
"""
import argparse
import json
import os
import re
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import fs2dec_oracle as F  # noqa: E402
from oracle import ssim_oracle as O  # noqa: E402

SSIM_SIZES = [(32, 1000, 80), (16, 1024, 80), (4, 4500, 80), (32, 1000, 10)]
STEP_SIZES = [(32, 1000), (16, 1024)]
DEV = torch.device("cuda", 0)
HBM_BYTES_PER_S, FP32_FLOPS = 3.35e12, 67e12
BYTES_PER_PIXEL = 32
# forward: 5 fields x 2 passes x 11 FMAs, 3 products, ~15 for the formula; backward: the forward's moments again, ~30 for
# the partials, 4 fields x 2 passes x 11 FMAs, 8 for d_x and d_y
FLOPS_PER_PIXEL = (5 * 2 * 11 * 2 + 3 + 15) * 2 + 30 + 4 * 2 * 11 * 2 + 8
HP = dict(F.HPARAMS_POPCS, dsx_train=True)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    name, power, sm, sm_max = [v.strip() for v in q[0].split(",")] if q else ("?", "?", "?", "?")
    return {"card": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(steps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / steps


def kernel_times(fn):
    """CUDA time per kernel of one call, from torch.profiler in a run of its own"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    agg = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            k = re.sub(r"^void |\(anonymous namespace\)::|<.*$|\(.*$", "", e.name)
            agg[k] = agg.get(k, 0.0) + e.device_time / 1e3
    return {k: round(v, 4) for k, v in sorted(agg.items(), key=lambda kv: -kv[1])}


def set_tf32(mode):
    """'fp32': TF32 off everywhere; 'defaults': PyTorch's (cuDNN convolutions TF32, matmuls fp32)"""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = mode == "defaults"


def ssim_call(ssim_fn, B, H, W):
    gen = torch.Generator().manual_seed(0)
    y = (torch.rand(B, 1, H, W, generator=gen) * 7 - 5.5).to(DEV) + 6
    x = (y + 0.3 * torch.randn(B, 1, H, W, generator=gen).to(DEV)).requires_grad_(True)

    def fn():
        x.grad = None
        ssim_fn(x, y, size_average=False).mean().backward()
    return fn


def step_case(ssim_fn, B, T, losses):
    from diffsinger_b200 import FastspeechDecoder
    torch.manual_seed(0)
    dec = FastspeechDecoder(hparams=HP)
    dec.load_state_dict(F.random_state_dict(0, HP), strict=True)
    dec = dec.to(DEV).train()
    mel_out = torch.nn.Linear(HP["hidden_size"], 80).to(DEV)
    x = F.fixture_input(1, B, T, HP["hidden_size"], tail=T * 3 // 4).to(DEV)
    target = torch.randn(B, T, 80, device=DEV)
    target[1, T * 3 // 4:] = 0

    def fn():
        dec.zero_grad(set_to_none=True)
        mel_out.zero_grad(set_to_none=True)
        O.mel_loss(mel_out(dec(x)), target, losses, ssim_fn=ssim_fn).backward()
    return fn, dec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    from diffsinger_b200 import ssim
    assert torch.cuda.is_available(), "bench_ssim.py measures on the GPU"
    res = dict(card(), workload="SSIM mel loss (11 x 11 Gaussian, sigma 1.5) forward + backward", ssim={}, step={})
    for B, H, W in SSIM_SIZES:
        n = B * H * W
        least = max(n * BYTES_PER_PIXEL / HBM_BYTES_PER_S, n * FLOPS_PER_PIXEL / FP32_FLOPS) * 1e3
        r = {"least_ms": least, "least_bound": "bytes" if n * BYTES_PER_PIXEL / HBM_BYTES_PER_S >
             n * FLOPS_PER_PIXEL / FP32_FLOPS else "flops"}
        set_tf32("defaults")
        call = ssim_call(ssim, B, H, W)
        r["dsx_ms"] = time_ms(call, a.steps, a.warmup)
        if a.kernels:
            r["dsx_kernels_ms"] = kernel_times(call)
        for mode in ("fp32", "defaults"):
            set_tf32(mode)
            r[f"eager_{mode}_ms"] = time_ms(ssim_call(O.ssim, B, H, W), a.steps, a.warmup)
        r["dsx_share_of_least"] = least / r["dsx_ms"]
        res["ssim"][f"{B}x{H}x{W}"] = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}
        torch.cuda.empty_cache()
    set_tf32("defaults")
    for B, T in STEP_SIZES:
        r = {}
        for name, fn_ssim, losses in (("eager_ssim", O.ssim, {"ssim": 0.5, "l1": 0.5}),
                                      ("dsx_ssim", ssim, {"ssim": 0.5, "l1": 0.5}),
                                      ("l1_only", None, {"l1": 0.5})):
            fn, dec = step_case(fn_ssim, B, T, losses)
            r[f"{name}_ms"] = time_ms(fn, a.steps, a.warmup)
            dec.close()
            del fn, dec
            torch.cuda.empty_cache()
        r["ssim_share_eager"] = (r["eager_ssim_ms"] - r["l1_only_ms"]) / r["eager_ssim_ms"]
        r["ssim_share_dsx"] = (r["dsx_ssim_ms"] - r["l1_only_ms"]) / r["dsx_ssim_ms"]
        res["step"][f"{B}x{T}"] = {k: round(v, 4) for k, v in r.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
