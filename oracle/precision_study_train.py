"""TEST INFRASTRUCTURE ONLY -- CPU emulation of the operand formats of the DiffNet training step, to choose its precision.

Every conv operand of a DiffNet training step (activations, weights and the incoming gradients on the way back) is
rounded to a format, with fp32 accumulation, and the L1 loss and every parameter gradient and d_cond are compared with
fp32 autograd as relative Frobenius errors.  L = 20, cycle 4, seeded weights with a nonzero final projection.

    python oracle/precision_study_train.py {tf32|fp16|fp16scaled|fp16dyn|bf16} B T [target]

fp16scaled multiplies the incoming gradients by a fixed 2^14 before rounding them and divides it out after.  fp16dyn is
the kernels' dynamic scale: the power of two S that puts S amax |d eps| in [2^(target-1), 2^target) (target 10 by
default), and it reports the largest scaled gradient operand of the backward and its headroom below the fp16 maximum
(65504): an operand past it would be inf.  tf32 rounds to TF32 as cuDNN's defaults do on an H100."""
import math, sys
import torch
import torch.nn.functional as F

torch.manual_seed(0)
DT = {"bf16": torch.bfloat16, "fp16": torch.float16, "fp16scaled": torch.float16, "fp16dyn": torch.float16,
      "tf32": None}[sys.argv[1]]
GS = 2.0 ** 14 if sys.argv[1] == "fp16scaled" else 1.0
TARGET = int(sys.argv[4]) if len(sys.argv) > 4 else 10
PEAK = [0.0]   # largest |scaled gradient operand| of the backward
B, T, M, C, H, L, CYC = int(sys.argv[2]), int(sys.argv[3]), 80, 256, 256, 20, 4


def tf32(x):
    i = x.contiguous().view(torch.int32)
    i = (i + 0x1000 + ((i >> 13) & 1) - 1) & ~0x1FFF
    return i.view(torch.float32)


class R(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return tf32(x) if DT is None else x.to(DT).float()

    @staticmethod
    def backward(ctx, g):
        if DT is None:
            return tf32(g)
        PEAK[0] = max(PEAK[0], (g * GS).abs().max().item())
        return (g * GS).to(DT).float() / GS


class RW(R):
    """A weight operand: rounded in the forward; its gradient is an fp32 accumulation over frames, never rounded."""
    @staticmethod
    def backward(ctx, g):
        return g


def r(x, on):
    return R.apply(x) if on else x


def rw(x, on):
    return RW.apply(x) if on else x


def params():
    p = {}
    kn = lambda *s: torch.nn.init.kaiming_normal_(torch.empty(*s))
    lin = lambda o, i: (torch.randn(o, i) / math.sqrt(i), torch.randn(o) * 0.02)
    p["in_w"], p["in_b"] = kn(C, M, 1), torch.randn(C) * 0.02
    p["m0_w"], p["m0_b"] = lin(4 * C, C)
    p["m2_w"], p["m2_b"] = lin(C, 4 * C)
    for l in range(L):
        p[f"dil_w{l}"], p[f"dil_b{l}"] = kn(2 * C, C, 3), torch.randn(2 * C) * 0.02
        p[f"dif_w{l}"], p[f"dif_b{l}"] = lin(C, C)
        p[f"cond_w{l}"], p[f"cond_b{l}"] = kn(2 * C, H, 1), torch.randn(2 * C) * 0.02
        p[f"out_w{l}"], p[f"out_b{l}"] = kn(2 * C, C, 1), torch.randn(2 * C) * 0.02
    p["skip_w"], p["skip_b"] = kn(C, C, 1), torch.randn(C) * 0.02
    p["fin_w"], p["fin_b"] = kn(M, C, 1) * 0.1, torch.randn(M) * 0.02   # nonzero: the reference zero-inits it
    return p


def net(p, spec, t, cond, q):
    x = F.relu(F.conv1d(r(spec, q), rw(p["in_w"], q), p["in_b"]))
    half = C // 2
    e = math.log(10000) / (half - 1)
    e = t[:, None].float() * torch.exp(torch.arange(half) * -e)[None]
    e = torch.cat((e.sin(), e.cos()), -1)
    e = F.linear(e, p["m0_w"], p["m0_b"])
    e = e * torch.tanh(F.softplus(e))
    e = F.linear(e, p["m2_w"], p["m2_b"])
    skips = 0
    for l in range(L):
        d = 2 ** (l % CYC)
        y = x + F.linear(e, p[f"dif_w{l}"], p[f"dif_b{l}"])[:, :, None]
        y = F.conv1d(r(y, q), rw(p[f"dil_w{l}"], q), p[f"dil_b{l}"], padding=d, dilation=d) + \
            F.conv1d(r(cond, q), rw(p[f"cond_w{l}"], q), p[f"cond_b{l}"])
        g, f = torch.chunk(y, 2, 1)
        z = torch.sigmoid(g) * torch.tanh(f)
        y = F.conv1d(r(z, q), rw(p[f"out_w{l}"], q), p[f"out_b{l}"])
        res, s = torch.chunk(y, 2, 1)
        x = (x + res) / math.sqrt(2.0)
        skips = skips + s
    x = skips / math.sqrt(L)
    x = F.relu(F.conv1d(r(x, q), rw(p["skip_w"], q), p["skip_b"]))
    return F.conv1d(r(x, q), rw(p["fin_w"], q), p["fin_b"])


p = params()
spec = torch.randn(B, M, T)
noise = torch.randn(B, M, T)
cond = torch.randn(B, H, T)
t = torch.randint(0, 100, (B,))
res = {}
for q in (False, True):
    pp = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    c = cond.clone().requires_grad_(True)
    eps = net(pp, spec, t, c, q)
    loss = (noise - eps).abs().mean()
    if q and sys.argv[1] == "fp16dyn":
        d_eps, = torch.autograd.grad(loss, eps, retain_graph=True)
        e = math.frexp(d_eps.abs().max().item())[1]          # amax in [2^(e-1), 2^e)
        GS = 2.0 ** (TARGET - e)
        PEAK[0] = d_eps.abs().max().item() * GS
        eps.backward(d_eps)
    else:
        loss.backward()
    res[q] = (loss.item(), {k: v.grad for k, v in pp.items()}, c.grad)
l0, g0, c0 = res[False]
l1, g1, c1 = res[True]
print(f"{sys.argv[1]} B={B} T={T}: loss {l0:.6f} vs {l1:.6f} rel {abs(l1 - l0) / l0:.2e}")
rel = {k: ((g1[k] - g0[k]).norm() / g0[k].norm()).item() for k in g0}
worst = sorted(rel.items(), key=lambda kv: -kv[1])[:6]
print("worst rel-Frobenius grad errors:", ", ".join(f"{k} {v:.2e}" for k, v in worst))
print("median", sorted(rel.values())[len(rel) // 2], " dcond", ((c1 - c0).norm() / c0.norm()).item())
if sys.argv[1] == "fp16dyn":
    print(f"target 2^{TARGET}: largest scaled gradient operand {PEAK[0]:.4g}, headroom below 65504 "
          f"2^{math.log2(65504 / PEAK[0]):.1f}")
print("grad magnitudes: |dL/deps| =", 1.0 / (B * M * T), " min |g| over params (abs max)",
      min(v.abs().max().item() for v in g0.values()))
