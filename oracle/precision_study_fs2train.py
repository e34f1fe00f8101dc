"""TEST INFRASTRUCTURE ONLY -- CPU emulation behind the FastSpeech2 decoder training step's gradient scale
(dsx_fs2train.cu): where the backward's fp16 operands sit in fp16's range once they are scaled by S, the power of two
with S amax |d_out| in [2^5, 2^6).

    python oracle/precision_study_fs2train.py [--sizes 32x1000,4x4500] [--target 5]

The workload is the training one: the shipped decoder (H 256, L 4, 2 heads, k 9, GELU, dropout 0.1) + mel_out
(Linear 256 -> 80) + L1, in fp32 autograd with the attention written out so that every operand the kernels round to fp16
can be hooked: gY2 (ffn_2's output gradient after dropout), gC (ffn_1's output gradient, after act' and k^-0.5), gY
(out_proj's output gradient after dropout), dO, dS = P (dP - D), dQ (times D^-0.5), dK and dV.  For each it prints
log2(65504 / (S amax)) -- the headroom below fp16's maximum -- and the fraction of nonzero scaled values below fp16's
smallest normal 2^-14 (held with reduced precision) and below 2^-24 (flushed to 0)."""
import argparse
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import fs2dec_oracle as O  # noqa: E402
from oracle.pe_oracle import make_positions, sinusoidal_table  # noqa: E402

HP = dict(O.HPARAMS_POPCS)


def decoder_hooked(sd, x, hp, p, hook, gen):
    """oracle.fs2dec_train_oracle.decoder_train with the attention written out and every fp16 operand hooked"""
    B, T, H = x.shape
    heads = int(hp['num_heads'])
    D, k = H // heads, int(hp['dec_ffn_kernel_size'])
    drop = lambda v: v * (torch.rand(v.shape, generator=gen) >= p).to(v.dtype).div_(1 - p)
    pad = O.padding_mask(x)
    keep = (~pad).to(x.dtype)[..., None]
    table = sinusoidal_table(max(2000, 1 + T), H)
    x = x + sd["pos_embed_alpha"] * table.index_select(0, make_positions(x[..., 0]).view(-1)).view(B, T, -1)
    x = drop(x) * keep
    kbias = torch.zeros(B, 1, 1, T).masked_fill(pad[:, None, None, :], float("-inf"))

    def hooked(v, name):
        v.register_hook(hook(name))
        return v

    for i in range(int(hp['dec_layers'])):
        pre = f"layers.{i}.op."
        y = F.layer_norm(x, (H,), sd[pre + "layer_norm1.weight"], sd[pre + "layer_norm1.bias"], O.LN_EPS)
        q, kk, v = (y @ sd[pre + "self_attn.in_proj_weight"].t()).split(H, -1)
        q = hooked(q, "dQ") * D ** -0.5
        q = q.view(B, T, heads, D).transpose(1, 2)
        kk = hooked(kk, "dK").view(B, T, heads, D).transpose(1, 2)
        v = hooked(v, "dV").view(B, T, heads, D).transpose(1, 2)
        s = hooked(q @ kk.transpose(-1, -2) + kbias, "dS")
        o = hooked((torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, T, H), "dO")
        a = hooked(o @ sd[pre + "self_attn.out_proj.weight"].t(), "gY")
        x = (x + drop(a)) * keep
        y = F.layer_norm(x, (H,), sd[pre + "layer_norm2.weight"], sd[pre + "layer_norm2.bias"], O.LN_EPS)
        w = O._ffn1_key(hp, i)
        c = F.conv1d(y.transpose(1, 2), sd[w + "weight"], sd[w + "bias"], padding=k // 2).transpose(1, 2) * k ** -0.5
        c = hooked(c, "gC")
        f2 = hooked(drop(F.gelu(c)) @ sd[pre + "ffn.ffn_2.weight"].t() + sd[pre + "ffn.ffn_2.bias"], "gY2")
        x = (x + drop(f2)) * keep
    return F.layer_norm(x, (H,), sd["layer_norm.weight"], sd["layer_norm.bias"], O.LN_EPS) * keep


def study(B, T, target):
    torch.manual_seed(0)
    gen = torch.Generator().manual_seed(1)
    sd = {kk: v.requires_grad_(True) for kk, v in O.random_state_dict(0, HP).items()}
    head = torch.nn.Linear(256, 80)
    x = O.fixture_input(1, B, T, 256, tail=T * 3 // 4 if B > 1 else None)
    y = torch.randn(B, T, 80, generator=gen)
    S = []
    rows = {}      # name -> [max of S |g|, values, below 2^-14, below 2^-24] over nonzero values

    def record(name, g):
        a = g.detach().abs().reshape(-1) * S[0]
        a = a[a > 0]
        r = rows.setdefault(name, [0.0, 0, 0, 0])
        r[0] = max(r[0], a.max().item())
        r[1] += a.numel()
        r[2] += (a < 2.0 ** -14).sum().item()
        r[3] += (a < 2.0 ** -24).sum().item()

    def on_out(g):
        e = math.frexp(g.abs().max().item())[1]       # amax in [2^(e-1), 2^e)
        S.append(2.0 ** (target + 1 - e))             # S amax in [2^target, 2^(target+1))
        record("d_out", g)

    out = decoder_hooked(sd, x, HP, HP['dropout'], lambda name: (lambda g: record(name, g)), gen)
    out.register_hook(on_out)
    (head(out) - y).abs().mean().backward()
    print(f"\nB x T = {B} x {T}: S = 2^{int(math.log2(S[0]))}")
    print(f"{'operand':8s} {'S amax':>10s} {'headroom':>9s} {'< 2^-14':>9s} {'< 2^-24':>9s}")
    for name, (m, n, sub, zero) in rows.items():
        print(f"{name:8s} {m:10.3e} {math.log2(65504 / m):8.1f}b {sub / n:9.2e} {zero / n:9.2e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="32x1000,4x4500")
    ap.add_argument("--target", type=int, default=5)
    a = ap.parse_args()
    torch.set_grad_enabled(True)
    for s in a.sizes.split(","):
        B, T = map(int, s.split("x"))
        study(B, T, a.target)


if __name__ == "__main__":
    main()
