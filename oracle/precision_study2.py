"""TEST INFRASTRUCTURE ONLY -- round-2 CPU emulation of cheaper tensor-core operand schemes.

Question: how few MMA passes keep the K-step loop inside |d| < 1e-3?  The weight rounding error of a single
fp16 pass is the same at every diffusion step (coherent: it accumulates ~linearly in K), whereas the rounding of
the running activations is fresh every step.  Schemes tried here:

  rn      round-to-nearest fp16 weights (one set, used at every step)
  sr<R>   R independently *stochastically rounded* fp16 weight sets, step j uses set j % R (E[w_sr] = w, so the
          weight error decorrelates across steps and accumulates ~sqrt(K))
  hl      hi+lo fp16 pair (2 passes)

    python -m oracle.precision_study2 [K100|K1000]
"""
import math, os, sys, time
import numpy as np, torch, torch.nn.functional as F
from . import diffnet_oracle as O
from .gen_golden import rs_normal, OUT


rn16, hl16, sr16 = O.rn16, O.hl16, O.sr16


def make_sets(P, mode1, mode2, R, seed=1234):
    """Weight sets for the residual layers: mode per GEMM in {'rn','sr','hl'}."""
    gen = np.random.RandomState(seed)
    sets = []
    n = R if ("sr" in (mode1, mode2)) else 1
    for r in range(n):
        Pw = {}
        for k, v in P.items():
            if not (k.endswith("weight") and v.dim() == 3 and k.startswith("residual_layers")):
                continue
            if "conditioner_projection" in k:
                continue
            m = mode2 if "output_projection" in k else mode1
            Pw[k] = rn16(v) if m == "rn" else (hl16(v) if m == "hl" else sr16(v, gen))
        sets.append(Pw)
    return sets


def forward(P, Pw, Ph, spec, t, cond, cycle, act_round=True):
    L = O.num_layers(P)
    x = F.relu(F.conv1d(hl16(spec[:, 0]), Ph["input_projection.weight"], P["input_projection.bias"]))
    e = O.step_embedding(P, t)
    skip = 0
    a = rn16 if act_round else (lambda v: v)
    for i in range(L):
        p = f"residual_layers.{i}."
        d = F.linear(e, P[p + "diffusion_projection.weight"], P[p + "diffusion_projection.bias"]).unsqueeze(-1)
        dil = 2 ** (i % cycle)
        cp = F.conv1d(cond, P[p + "conditioner_projection.weight"], P[p + "conditioner_projection.bias"])
        y = F.conv1d(a(x + d), Pw[p + "dilated_conv.weight"], P[p + "dilated_conv.bias"], padding=dil, dilation=dil) + cp
        g, f = torch.chunk(y, 2, dim=1)
        z = torch.sigmoid(g) * torch.tanh(f)
        o = F.conv1d(a(z), Pw[p + "output_projection.weight"], P[p + "output_projection.bias"])
        r, s = torch.chunk(o, 2, dim=1)
        x = (x + r) / math.sqrt(2.0)
        skip = skip + s
    x = skip / math.sqrt(L)
    x = F.relu(F.conv1d(hl16(x), Ph["skip_projection.weight"], P["skip_projection.bias"]))
    x = F.conv1d(hl16(x), Ph["output_projection.weight"], P["output_projection.bias"])
    return x[:, None]


def run(name, P, S, sets, Ph, xT, cond, noise, x0, K, cycle):
    x, b = xT.clone(), xT.shape[0]
    t0 = time.time()
    with torch.no_grad():
        for j, t in enumerate(reversed(range(K))):
            eps = forward(P, sets[j % len(sets)], Ph, x, torch.full((b,), t), cond, cycle)
            xr = (S["sqrt_recip_alphas_cumprod"][t] * x - S["sqrt_recipm1_alphas_cumprod"][t] * eps).clamp(-1, 1)
            mean = S["posterior_mean_coef1"][t] * xr + S["posterior_mean_coef2"][t] * x
            x = mean + (0.0 if t == 0 else 1.0) * (0.5 * S["posterior_log_variance_clipped"][t]).exp() * noise[j]
    d = (x - x0).abs()
    print(f"{name}: max {d.max():.2e} MAE {d.mean():.2e} frac>5e-4 {(d > 5e-4).float().mean():.2e} ({time.time() - t0:.0f}s)",
          flush=True)


def main(which):
    torch.set_num_threads(8)
    P = O.build_state_dict(0, dilation_cycle_length=1)
    Ph = {k: (hl16(v) if k.endswith("weight") and v.dim() == 3 else v) for k, v in P.items()}
    if which == "K100":
        g = np.load(os.path.join(OUT, "ddpm_lj_K100.npz"))
        cond, xT, x0 = (torch.from_numpy(g[k]) for k in ("cond", "xT", "x0"))
        K = 100
        noise = rs_normal(int(g["noise_seed"]), (K,) + tuple(xT.shape))
        S = O.make_schedule(O.linear_beta_schedule(100, 0.06))
    else:
        K = 1000
        S = O.make_schedule(O.linear_beta_schedule(1000, 0.02))
        cond, xT = rs_normal(71, (1, 256, 96)), rs_normal(72, (1, 1, 80, 96))
        noise = rs_normal(73, (K, 1, 1, 80, 96))
        with torch.no_grad():
            x0 = O.sample_ddpm(P, S, xT, cond, K, noise, 1)
    schemes = (("W1 rn, W2 hl", "rn", "hl", 1), ("W1 hl, W2 hl (fp16x2)", "hl", "hl", 1),
               ("W1 sr16, W2 hl", "sr", "hl", 16), ("W1 sr64, W2 hl", "sr", "hl", 64),
               ("W1 sr64, W2 sr64", "sr", "sr", 64), ("W1 sr16, W2 sr16", "sr", "sr", 16),
               ("W1 rn, W2 rn (fp16)", "rn", "rn", 1), ("W1 sr4, W2 sr4", "sr", "sr", 4))
    for name, m1, m2, R in schemes:
        sets = make_sets(P, m1, m2, R)
        run(name, P, S, sets, Ph, xT, cond, noise, x0, K, 1)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "K100")
