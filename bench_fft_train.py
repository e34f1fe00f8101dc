"""Times one FFT denoiser training step -- FFT forward on x_noisy, L1 against the noise (p_losses), backward with the
gradient of cond -- with the dsx training step (diffsinger_b200.FFT under dsx_train) against eager PyTorch: fp32 with
TF32 off, PyTorch's defaults (cuDNN convolutions in TF32, matmuls in fp32), TF32 everywhere (matmuls too), and
autocast(bfloat16).  The denoiser is the shipped one (H 256, 4 layers, 2 heads, k 9, SAME, GELU, residual_channels 256,
dropout 0.1).  Sizes: 32 x 1000 (LJ's 32k-frame batches), 16 x 1024 and 4 x 4500 (long singing segments, where the T^2
term of the attention matters).  Prints one JSON line with the card, its power limit and SM clock, per-size times, and
peak memory above the inputs (the dsx tape and workspace broken out).  --kernels adds per-kernel CUDA times from
torch.profiler for the dsx step at each size.

    python bench_fft_train.py [--steps 10] [--warmup 3] [--kernels]
"""
import argparse
import json
import re
import sys

import torch

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.abspath(__file__)))
from bench_fs2dec_train import card, time_step  # noqa: E402
from oracle import fft_oracle as O  # noqa: E402
from oracle.fft_train_oracle import forward_train  # noqa: E402

HP = dict(O.HPARAMS_POPCS)
SIZES = [(32, 1000), (16, 1024), (4, 4500)]
DEV = torch.device("cuda", 0)


def batch(B, T):
    g = torch.Generator().manual_seed(1)
    spec = torch.randn(B, 1, 80, T, generator=g).to(DEV)
    t = torch.randint(0, 100, (B,), generator=g).to(DEV)
    cond = torch.randn(B, 256, T, generator=g).to(DEV).requires_grad_(True)   # d_cond is computed, as in DiffSinger
    noise = torch.randn(B, 1, 80, T, generator=g).to(DEV)
    return spec, t, cond, noise


def dsx_case(B, T):
    from diffsinger_b200 import FFT
    m = FFT(hparams=dict(HP, dsx_train=True))
    m.load_state_dict(O.random_state_dict(0, HP), strict=True)
    m = m.to(DEV).train()
    spec, t, cond, noise = batch(B, T)

    def step():
        (m(spec, t, cond) - noise).abs().mean().backward()
    return step, m


def eager_case(B, T, mode):
    sd = {k: v.to(DEV).requires_grad_(True) for k, v in O.random_state_dict(0, HP).items()
          if k != "embed_positions._float_tensor"}
    spec, t, cond, noise = batch(B, T)
    p = HP['dropout']

    def step():
        masks = [torch.rand(B, T, 4 * 256 if s > 0 and s % 3 == 2 else 256, device=DEV) >= p
                 for s in range(1 + 3 * HP['dec_layers'])]
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=(mode == "bf16")):
            loss = (forward_train(sd, spec, t, cond, HP, masks, p) - noise).abs().mean()
        loss.backward()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    res = dict(card(), workload="FFT denoiser training step (H 256, L 4, heads 2, k 9, dim 256, p 0.1) + L1 to the noise",
               sizes={})
    for B, T in SIZES:
        r = {}
        torch.cuda.empty_cache()
        step, m = dsx_case(B, T)
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        r["dsx_ms"] = time_step(step, a.steps, a.warmup)
        r["dsx_peak_mib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
        st = m._dsx_train_step()
        r["dsx_tape_mib"] = st.tape_bytes(DEV, B, T) / 2 ** 20
        r["dsx_workspace_mib"] = st.workspace(DEV, B, T).numel() / 2 ** 20
        if a.kernels:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                step()
                torch.cuda.synchronize()
            agg = {}
            for e in prof.events():
                if e.device_type.name == "CUDA":
                    k = re.sub(r"^void |\(anonymous namespace\)::|<.*$|\(.*$", "", e.name)
                    agg[k] = agg.get(k, 0.0) + e.device_time / 1e3
            r["dsx_kernels_ms"] = dict(sorted(((k, round(v, 3)) for k, v in agg.items()), key=lambda kv: -kv[1])[:20])
        del step, m
        for mode in ("fp32", "defaults", "tf32", "bf16"):
            torch.cuda.empty_cache()
            torch.backends.cuda.matmul.allow_tf32 = mode in ("tf32", "bf16")
            torch.backends.cudnn.allow_tf32 = mode != "fp32"
            step = eager_case(B, T, mode)
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            r[f"eager_{mode}_ms"] = time_step(step, a.steps, a.warmup)
            r[f"eager_{mode}_peak_mib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
            del step
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.allow_tf32 = True
        r = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()}
        res["sizes"][f"{B}x{T}"] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
