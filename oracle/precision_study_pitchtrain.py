"""TEST INFRASTRUCTURE ONLY -- CPU emulation behind the pitch predictor training step's operand format and gradient scale
(dsx_pitchtrain.cu, on the duration predictor step's backward in dsx_durtrain.cu), and the source of the parity bounds of
tests/test_gpu_pitchpred_train.py.

    python oracle/precision_study_pitchtrain.py [--cases frame,ph,cwt,left] [--seeds 3]

The workloads are the four configurations of oracle/gen_golden_pitchpred_train.py at the GPU test's sizes: frame
(aux_rel, 256 -> 256, 5 layers, k 5, odim 2) at 4 x 1000 frames, ph (2 layers, odim 1) at 8 x 120, cwt (idim 128, 2
layers, odim 11) at 8 x 300 and left (3 layers, LEFT) at 4 x 200, each with padding tails of zero frames, seeded p = 0.5
masks and a standard normal d_out, as the GPU test draws them.  Everything runs in float64; only the convolutions'
operands are rounded, as a format would round them:
  forward   each conv's input (x + alpha table[pos] for layer 0) and weight
  backward  the gradient at each conv's output, scaled by S (the power of two with S amax |d_out| over every column in
            [2^5, 2^6), as k_scale chooses it), rounded and divided by S again, and the operands it meets
The GPU test's reference is this step with fp16 forward operands and an exact backward.  The study prints, per case and
seed, the worst per-tensor relative Frobenius error of the fp16 backward against it (out, d_x and every gradient but
pos_embed_alpha's), and the same for a TF32 backward and for a forward computed in fp32 (fp16 operands, fp32
accumulation and LayerNorm, which is what dsx and TF32 autograd both do).  d pos_embed_alpha = sum d_in . table[pos] is
printed against |d alpha| and against the Cauchy-Schwarz bound |d_in error| |table[pos]|.  For the scaled gradient
operand of each layer it prints log2(65504 / (S amax)), the headroom below fp16's maximum, and the fraction of nonzero
values below 2^-14 (fp16 subnormals).  The fp32 forward is run under ORDERS random orders of each conv's input channels.

Result over seeds 0..2 (STUDY below; DESIGN.md §3l):
  * The fp16 backward, with S from amax |d_out| over every column and no mask, costs at most 4.9e-4 in every
    configuration, the 11-column CWT head included (3.6e-4), the same as a TF32 backward; d alpha moves by at most
    1.6e-3 of |d alpha|.  The scaled operand keeps 2^5.9 or more of headroom below 65504 (layer 0, the smallest) and
    at most 2.1e-3 of its nonzero values are fp16 subnormals.
  * A forward in fp32 arithmetic, with the same fp16 operands, moves the step by up to 1.4e-2 (frame), 8.7e-3 (ph,
    left) and 1.7e-4 (cwt) depending only on its summation order: it flips ReLUs and LayerNorm rows near zero, and
    d alpha, a sum that cancels, by up to 3 % of itself.  This depends on the instance, so the GPU test measures it on
    each case (fp32 autograd under hidden-channel relabelings, and TF32 autograd) and bounds the step by twice that
    plus the fp16 backward's cost."""
import argparse
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.fs2enc_oracle import DUR_LN_EPS  # noqa: E402
from oracle.gen_golden_pitchpred_train import CASES, random_state_dict  # noqa: E402
from oracle.pe_oracle import make_positions, sinusoidal_table  # noqa: E402
from oracle.precision_study_durtrain import rnd  # noqa: E402

P_DROP = 0.5
ORDERS = 4                     # fp32 summation orders tried per seed
# case -> (B, T, tails) at the GPU test's sizes (frame at 4 of its 16 utterances: the CPU is slow in float64)
SIZES = {"frame": (4, 1000, [(1, 963), (2, 926), (3, 889)]), "ph": (8, 120, [(1, 70), (5, 3)]),
         "cwt": (8, 300, [(3, 200)]), "left": (4, 200, [(2, 150)])}
# what this study printed per case over seeds 0..2 (relative Frobenius, against the fp16-forward exact-backward step):
# (the fp16 backward's worst, the fp32 forward's worst over ORDERS summation orders)
STUDY = {"frame": (4.9e-4, 1.4e-2), "ph": (4.0e-4, 8.7e-3), "cwt": (3.6e-4, 1.7e-4), "left": (4.1e-4, 8.7e-3)}


class Conv(torch.autograd.Function):
    """conv1d with taps (pad_l, pad_r) of zeros, forward operands rounded to ffmt (computed in float32 when f32), the
    backward's to bfmt: the output gradient scaled by S, rounded and unscaled; records the scaled operand in `log`"""

    @staticmethod
    def forward(ctx, x, w, b, pad, ffmt, f32, bfmt, S, log):
        xr, wr = rnd(x, ffmt), rnd(w, ffmt)
        ctx.save_for_backward(xr, wr)
        ctx.pad, ctx.bfmt, ctx.S, ctx.log = pad, bfmt, S, log
        if f32:         # f32 = a generator: the input channels in a random order, so another fp32 summation order
            perm = torch.randperm(xr.shape[1], generator=f32)
            return F.conv1d(F.pad(xr[:, perm].float(), pad), wr[:, perm].float(), b.float()).double()
        return F.conv1d(F.pad(xr, pad), wr, b)

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
            y = F.conv1d(F.pad(x_, ctx.pad), w_)
            dx, dw = torch.autograd.grad(y, (x_, w_), gq)
        return dx, dw, gq.sum((0, 2)), None, None, None, None, None, None


def forward(sd, x, masks, k, padding, ffmt, f32, bfmt, S, log, table, pos):
    B, T, H = x.shape
    pad = ((k - 1) // 2, (k - 1) // 2) if padding == 'SAME' else (k - 1, 0)
    h = (x + sd["pos_embed_alpha"] * table.index_select(0, pos.view(-1)).view(B, T, H)).transpose(1, 2)
    for i, m in enumerate(masks):
        pre = f"conv.{i}."
        u = Conv.apply(h, sd[pre + "1.weight"], sd[pre + "1.bias"], pad, ffmt, f32, bfmt, S, log)
        r = torch.relu(u)
        C = r.shape[1]
        if f32:
            y = F.layer_norm(r.transpose(1, 2).float(), (C,), sd[pre + "3.weight"].float(), sd[pre + "3.bias"].float(),
                             DUR_LN_EPS).double().transpose(1, 2)
        else:
            y = F.layer_norm(r.transpose(1, 2), (C,), sd[pre + "3.weight"], sd[pre + "3.bias"], DUR_LN_EPS).transpose(1, 2)
        h = y * m.transpose(1, 2).double() / (1 - P_DROP)
    return F.linear(h.transpose(1, 2), sd["linear.weight"], sd["linear.bias"])


def step(sd0, x0, masks, d_out, k, padding, ffmt, f32, bfmt, S, table, pos):
    sd = {n: v.clone().requires_grad_(True) for n, v in sd0.items()}
    x = x0.clone().requires_grad_(True)
    log = []
    out = forward(sd, x, masks, k, padding, ffmt, f32, bfmt, S, log, table, pos)
    out.backward(d_out)
    names = sorted(n for n in sd if n != "pos_embed_alpha")
    return [out.detach(), x.grad] + [sd[n].grad for n in names], sd["pos_embed_alpha"].grad.item(), log[::-1]


def rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-300)).item()


def study(case, seed):
    cfg = dict((c, f) for c, _, _, f in CASES)[case]
    idim, L, C, odim, k, padding = cfg
    B, T, tails = SIZES[case]
    g = torch.Generator().manual_seed(1000 * seed + 17)
    sd = {n: v.double() for n, v in random_state_dict(seed, idim, L, C, odim, k).items()
          if n != "embed_positions._float_tensor"}
    x = torch.randn(B, T, idim, generator=g, dtype=torch.float64)
    for b, t in tails:
        x[b, t:] = 0
    masks = [torch.rand(B, T, C, generator=g) >= P_DROP for _ in range(L)]
    d_out = torch.randn(B, T, odim, generator=g, dtype=torch.float64)
    amax = d_out.abs().max().item()
    S = 2.0 ** (6 - math.frexp(amax)[1])
    table = sinusoidal_table(max(4096, 1 + T), idim, dtype=torch.float64)
    pos = make_positions(x[..., 0])
    t_norm = table.index_select(0, pos.view(-1)).norm().item()
    ref, a_ref, _ = step(sd, x, masks, d_out, k, padding, "fp16", False, "exact", S, table, pos)
    res, a16, log = step(sd, x, masks, d_out, k, padding, "fp16", False, "fp16", S, table, pos)
    e16 = [rel(a, b) for a, b in zip(res, ref) if b.norm() > 0]
    tf, _, _ = step(sd, x, masks, d_out, k, padding, "fp16", False, "tf32", S, table, pos)
    etf = [rel(a, b) for a, b in zip(tf, ref) if b.norm() > 0]
    e32, a32 = [0.0], a_ref
    for r in range(ORDERS):
        f32, a, _ = step(sd, x, masks, d_out, k, padding, "fp16", torch.Generator().manual_seed(r), "exact", S, table, pos)
        e = [rel(u, v) for u, v in zip(f32, ref) if v.norm() > 0]
        e32, a32 = (e, a) if max(e) > max(e32) else (e32, a32)
    cs = (res[1] - ref[1]).norm().item() * t_norm
    print(f"{case} seed {seed}: B {B} x T {T}, amax |d_out| {amax:.2f}, S = 2^{int(math.log2(S))}")
    print(f"  fp16 backward: worst {max(e16):.2e} (out {e16[0]:.1e}, d_x {e16[1]:.1e}); TF32 backward: worst "
          f"{max(etf):.2e}; fp32 forward, worst of {ORDERS} summation orders: {max(e32):.2e}")
    print(f"  d alpha {a_ref:.4e}: fp16 backward off by {abs(a16 - a_ref):.2e} ({abs(a16 - a_ref) / abs(a_ref):.1e} of "
          f"|d alpha|, Cauchy-Schwarz bound {cs:.2e}); fp32 forward off by {abs(a32 - a_ref):.2e}")
    for i, gs in enumerate(log):
        nz = gs[gs != 0].abs()
        head = math.log2(65504 / nz.max().item()) if nz.numel() else float("inf")
        sub = (nz < 2 ** -14).double().mean().item() if nz.numel() else 0.0
        print(f"  layer {i}: scaled gradient operand headroom 2^{head:.1f}, below 2^-14 {sub:.2e}")
    return max(e16), max(e32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="frame,ph,cwt,left")
    ap.add_argument("--seeds", type=int, default=3)
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count() or 1)
    for case in a.cases.split(","):
        r = [study(case, s) for s in range(a.seeds)]
        print(f"{case} over {a.seeds} seeds: fp16 backward {max(v[0] for v in r):.2e} (STUDY {STUDY[case][0]:.1e}), fp32 "
              f"forward {max(v[1] for v in r):.2e} (STUDY {STUDY[case][1]:.1e})")


if __name__ == "__main__":
    main()
