"""Times one DiffNet training step -- forward, L1 loss against noise, backward to every parameter and to cond -- on the
dsx training step and on eager PyTorch (fp32 with TF32 off, cuDNN's defaults, and autocast bf16), L = 20, cycle 4.

    python bench_train.py [--sizes 16x1024,4x2048] [--steps 10] [--warmup 3] [--kernels]

Prints one JSON line per size: ms per step, mel-frames/s, the share of dense FP16 peak that the FLOP floor (3x the
forward's 2 L (3 C 2C + H 2C + C 2C) per frame) implies, and peak memory above the inputs from max_memory_allocated
(dsx: the tape, the workspace and the gradients, all from PyTorch's allocator; eager: autograd's saved tensors and the
gradients).  --kernels adds per-kernel device times from torch.profiler.  The card's name, power limit and SM clock
are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

FP16_PEAK = 989e12   # H100 SXM dense FP16 (data sheet, 700 W)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm, smax = [s.strip() for s in out.split(",")]
        return dict(name=name, power_limit=pl, sm_clock=sm, sm_clock_max=smax)
    except Exception as e:  # pragma: no cover
        return dict(name=torch.cuda.get_device_name(0), error=str(e))


def flops_per_frame(L=20, C=256, H=256, M=80):
    return 3 * 2 * (L * (3 * C * 2 * C + H * 2 * C + C * 2 * C) + M * C + C * C + C * M)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16x1024,4x2048")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernels", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train.py needs a CUDA device")
    import diffsinger_b200 as dsx
    dev = torch.device("cuda", 0)
    info = card()
    hp = dict(hidden_size=256, residual_layers=20, residual_channels=256, dilation_cycle_length=4)
    torch.manual_seed(0)
    net = dsx.DiffNet(80, hparams=hp, train=True)
    torch.nn.init.normal_(net.output_projection.weight, std=0.02)
    net = net.to(dev).train()

    def step_fn(mode, spec, t, cond, noise):
        c = cond.requires_grad_(True)
        if mode == "dsx":
            eps = net(spec, t, c)
        elif mode == "autocast_bf16":
            with torch.autocast("cuda", dtype=torch.bfloat16):
                eps = net._forward_autograd(spec, t, c)
        else:
            eps = net._forward_autograd(spec, t, c)
        loss = (noise - eps.float()).abs().mean()
        loss.backward()
        c.grad = None
        net.zero_grad(set_to_none=True)

    for size in args.sizes.split(","):
        B, T = map(int, size.split("x"))
        g = torch.Generator(device=dev).manual_seed(1)
        spec = torch.randn(B, 1, 80, T, device=dev, generator=g)
        cond = torch.randn(B, 256, T, device=dev, generator=g)
        noise = torch.randn(B, 1, 80, T, device=dev, generator=g)
        t = torch.randint(0, 100, (B,), device=dev, generator=g)
        res = dict(B=B, T=T, L=20, cycle=4, card=info)
        for mode in ("dsx", "fp32_tf32_off", "cudnn_defaults", "autocast_bf16"):
            tf32 = mode == "cudnn_defaults"
            torch.backends.cudnn.allow_tf32 = tf32 or mode in ("dsx", "autocast_bf16")
            torch.backends.cuda.matmul.allow_tf32 = False
            if mode == "fp32_tf32_off":
                torch.backends.cudnn.allow_tf32 = False
            for _ in range(args.warmup):
                step_fn(mode, spec, t, cond.clone(), noise)
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step_fn(mode, spec, t, cond.clone(), noise)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            fps = B * T / (ms / 1e3)
            res[mode] = dict(ms=round(ms, 3), frames_per_s=round(fps), fp16_peak_share=round(
                fps * flops_per_frame() / FP16_PEAK, 4), peak_mem_mb=round((torch.cuda.max_memory_allocated() - base) / 2**20, 1))
        res["tape_mb"] = round(net._dsx_train_step().tape_bytes(dev, B, T) / 2**20, 1)
        res["workspace_mb"] = round(net._dsx_train_step().workspace(dev, B, T).numel() / 2**20, 1)
        res["dsx_speedup_vs_cudnn_defaults"] = round(res["cudnn_defaults"]["ms"] / res["dsx"]["ms"], 3)
        if args.kernels:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                step_fn("dsx", spec, t, cond.clone(), noise)
                torch.cuda.synchronize()
            ev = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" or getattr(e, "self_device_time_total", 0):
                    ev[e.key] = dict(us=round(getattr(e, "self_device_time_total", 0.0), 1), calls=e.count)
            res["kernels"] = dict(sorted(ev.items(), key=lambda kv: -kv[1]["us"])[:25])
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
