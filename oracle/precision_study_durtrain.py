"""TEST INFRASTRUCTURE ONLY -- CPU emulation behind the duration predictor training step's operand format and gradient
scale (dsx_durtrain.cu).

    python oracle/precision_study_durtrain.py [--sizes 16x250,4x1000] [--target 5] [--layers 5]

The workload is ds100_adj_rel's predictor (256 -> 256, 5 layers, k 3, SAME, p 0.5, seeded masks) on padded batches,
with the masked pdur MSE as the loss.  Everything runs in float64; only the convolutions' operands are rounded, as a
format would round them:
  forward   each conv's input and weight (fp16 is what dsx_durpred_forward uses, so the training forward must use it too)
  backward  the gradient at each conv's output, scaled by S (the power of two with S amax |d_xs * !mask| in
            [2^target, 2^(target + 1))), rounded and divided by S again, and the weight and input operands it meets
Formats: fp16 (10-bit mantissa, smallest normal 2^-14, subnormals to 2^-24), TF32 (10-bit mantissa, fp32 range), bf16
(7-bit mantissa, fp32 range), and exact.  For each (forward, backward) pair it prints the worst per-tensor relative
Frobenius error over xs, d_x and every gradient against the exact float64 step.  For the scaled gradient operand of each
layer it prints log2(65504 / (S amax)), the headroom below fp16's maximum, and the fraction of nonzero values below
2^-14 and below 2^-24.  It also prints, per layer, the largest LayerNorm rstd over real tokens (eps 1e-12) and the
fraction of ReLU inputs whose sign the forward's rounding flips."""
import argparse
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.fs2enc_oracle import DUR_LN_EPS  # noqa: E402
from oracle.gen_golden_durpred_train import random_state_dict  # noqa: E402

P_DROP, K, C = 0.5, 3, 256


def rnd(v, fmt):
    """v (float64) rounded to fmt, round to nearest even"""
    if fmt == "exact":
        return v
    if fmt == "fp16":
        return v.half().double()
    if fmt == "bf16":
        return v.bfloat16().double()
    f = v.float()                                        # tf32: fp32 with the 13 low mantissa bits rounded off
    i = f.view(torch.int32)
    i = (i + 0xFFF + ((i >> 13) & 1)) & ~0x1FFF
    return i.view(torch.float32).double()


class Conv(torch.autograd.Function):
    """conv1d (SAME, k taps) with the forward operands rounded to ffmt and the backward's to bfmt: the output gradient
    scaled by S, rounded and unscaled; records the scaled operand in `log`"""

    @staticmethod
    def forward(ctx, x, w, b, ffmt, bfmt, S, log):
        xr, wr = rnd(x, ffmt), rnd(w, ffmt)
        ctx.save_for_backward(xr, wr)
        ctx.bfmt, ctx.S, ctx.log = bfmt, S, log
        return F.conv1d(F.pad(xr, (K // 2, K // 2)), wr, b)

    @staticmethod
    def backward(ctx, g):
        xr, wr = ctx.saved_tensors
        gs = g * ctx.S
        ctx.log.append(gs.detach())
        gq = rnd(gs, ctx.bfmt) / ctx.S
        xq, wq = rnd(xr, ctx.bfmt), rnd(wr, ctx.bfmt)
        with torch.enable_grad():
            x_ = xq.detach().requires_grad_(True)
            w_ = wq.detach().requires_grad_(True)
            y = F.conv1d(F.pad(x_, (K // 2, K // 2)), w_)
            dx, dw = torch.autograd.grad(y, (x_, w_), gq)
        return dx, dw, gq.sum((0, 2)), None, None, None, None


def forward(sd, x, mask, masks, L, ffmt, bfmt, S, log, stats=None):
    keep = (1 - mask.double())
    h = x.transpose(1, 2)
    for i in range(L):
        pre = f"conv.{i}."
        u = Conv.apply(h, sd[pre + "1.weight"], sd[pre + "1.bias"], ffmt, bfmt, S, log)
        if stats is not None:
            stats.append(u.detach())
        r = torch.relu(u)
        y = F.layer_norm(r.transpose(1, 2), (C,), sd[pre + "3.weight"], sd[pre + "3.bias"], DUR_LN_EPS).transpose(1, 2)
        h = y * masks[i].transpose(1, 2).double() / (1 - P_DROP) * keep[:, None, :]
    return (F.linear(h.transpose(1, 2), sd["linear.weight"], sd["linear.bias"]).squeeze(-1)) * keep


def step(sd0, x0, mask, masks, dur, L, ffmt, bfmt, S, stats=None):
    sd = {k: v.clone().requires_grad_(True) for k, v in sd0.items()}
    x = x0.clone().requires_grad_(True)
    log = []
    xs = forward(sd, x, mask, masks, L, ffmt, bfmt, S, log, stats)
    nonpad = (~mask).double()
    loss = (((xs - torch.log(dur + 1)) ** 2) * nonpad).sum() / nonpad.sum()
    loss.backward()
    names = sorted(sd)
    return [xs.detach(), x.grad] + [sd[k].grad for k in names], log[::-1]


def rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def study(B, T, target, L):
    g = torch.Generator().manual_seed(B * 7 + T)
    sd = {k: v.double() for k, v in random_state_dict(0, C, L, C, K).items()}
    x = torch.randn(B, T, C, generator=g, dtype=torch.float64)
    mask = torch.zeros(B, T, dtype=torch.bool)
    for b in range(1, B, 2):
        mask[b, T - T // 4:] = True
    dur = torch.randint(1, 20, (B, T), generator=g).double()
    masks = [torch.rand(B, T, C, generator=g) >= P_DROP for _ in range(L)]
    # S from amax |d_xs * !mask| as the kernels choose it: d_xs of the pdur MSE
    nonpad = (~mask).double()
    with torch.no_grad():
        xs = forward({k: v for k, v in sd.items()}, x, mask, masks, L, "fp16", "exact", 1.0, [])
        dxs = 2 * (xs - torch.log(dur + 1)) * nonpad / nonpad.sum()
    amax = dxs.abs().max().item()
    S = 2.0 ** (target - math.frexp(amax)[1] + 1)
    exact_stats, f16_stats = [], []
    ref, _ = step(sd, x, mask, masks, dur, L, "exact", "exact", S, exact_stats)
    _, log = step(sd, x, mask, masks, dur, L, "fp16", "fp16", S, f16_stats)
    print(f"B {B} x T {T}, {L} layers: amax |d_xs| = {amax:.3e}, S = 2^{int(math.log2(S))}")
    real = (~mask).reshape(-1)
    for i, (gs, ue, uf) in enumerate(zip(log, exact_stats, f16_stats)):
        gs = gs.transpose(1, 2).reshape(-1, C)[real]
        nz = gs[gs != 0].abs()
        head = math.log2(65504 / nz.max().item()) if nz.numel() else float("inf")
        sub = (nz < 2 ** -14).double().mean().item() if nz.numel() else 0.0
        flush = (nz < 2 ** -24).double().mean().item() if nz.numel() else 0.0
        r = torch.relu(ue).transpose(1, 2).reshape(-1, C)[real]
        rstd = (1 / torch.sqrt(r.var(-1, unbiased=False) + DUR_LN_EPS)).max().item()
        flips = ((ue > 0) != (uf > 0)).transpose(1, 2).reshape(-1, C)[real].double().mean().item()
        print(f"  layer {i}: scaled gradient operand headroom 2^{head:.1f}, below 2^-14 {sub:.2e}, below 2^-24 "
              f"{flush:.2e}; LayerNorm rstd max {rstd:.1f}; ReLU sign flips from the fp16 forward {flips:.2e}")
    for ffmt, bfmt in (("fp16", "fp16"), ("fp16", "exact"), ("exact", "fp16"), ("tf32", "tf32"), ("fp16", "tf32"),
                       ("fp16", "bf16"), ("bf16", "bf16")):
        res, _ = step(sd, x, mask, masks, dur, L, ffmt, bfmt, S)
        errs = [rel(a, b) for a, b in zip(res, ref)]
        print(f"  forward {ffmt:5s} backward {bfmt:5s}: worst {max(errs):.2e}  xs {errs[0]:.1e}  d_x {errs[1]:.1e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16x250,4x1000")
    ap.add_argument("--target", type=int, default=5)
    ap.add_argument("--layers", type=int, default=5)
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count() or 1)
    for s in a.sizes.split(","):
        B, T = (int(v) for v in s.split("x"))
        study(B, T, a.target, a.layers)


if __name__ == "__main__":
    main()
