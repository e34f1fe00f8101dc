"""TEST INFRASTRUCTURE ONLY -- CPU oracle for the DiffSinger denoiser hot path.

A functional (no nn.Module, no global ``hparams``) fp32 restatement of

  * ``DiffNet.forward``              usr/diff/net.py:107-130
  * ``ResidualBlock.forward``        usr/diff/net.py:66-78
  * ``SinusoidalPosEmb`` / ``Mish``  usr/diff/net.py:32-44, usr/diff/diffusion.py:68-70
  * schedule buffers                 usr/diff/shallow_diffusion_tts.py:44-62, 90-123
  * ``p_sample`` (DDPM)              usr/diff/shallow_diffusion_tts.py:134-166
  * ``p_sample_plms`` (PNDM)         usr/diff/shallow_diffusion_tts.py:168-204
  * the K-step inference loop        usr/diff/shallow_diffusion_tts.py:248-275
  * ``norm_spec`` / ``denorm_spec`` / ``q_sample``   :206-211, :278-282

Weights are passed as a dict keyed by the reference's own state-dict names
(``residual_layers.3.dilated_conv.weight`` ...), so a checkpoint's ``denoise_fn.*``
entries can be fed in directly.  Arithmetic is torch CPU fp32 (the same ATen CPU kernels
the reference runs on), which is what "the reference's own CPU path" means for this repo.

Pinning: ``oracle/gen_golden.py`` compares every function here against the live
reference modules imported from a checkout of the reference (bit-exact or <=1e-6) and writes the
vectors in ``tests/golden``; ``tests/test_oracle.py`` re-checks the oracle against those
vectors wherever the tests run.

Operand formats (``fmt=``).  ``diffnet_forward`` and every sampler built on it take ``fmt``: ``None`` is the
reference computation above, unchanged; ``"fp16"``, ``"fp16x2"``, ``"fp16x3"`` and ``"fp16s"`` simulate what the
tensor-core step kernel (dsx_hopper.cu) rounds in that precision, in the dtype of the inputs (float64 for a simulation
whose only error is the operand rounding).  The simulation follows the kernel's header:

  * conditioner projection: 3-pass, taken as exact;
  * dilated conv and output projection: P = 1 (fp16) uses round-to-nearest fp16 weights, P = 2 (fp16x2) hi + lo fp16
    weights, both with y = x + d and z rounded to fp16; P = 3 (fp16x3) also splits y and z into hi + lo; fp16s uses R
    sets of stochastically rounded fp16 weights, evaluation row j (the FiLM-table row: the step of a loop, the
    warm-up's second evaluation at row n, 0 for a single evaluation) on set j % R, with y and z rounded to fp16;
  * input projection and head: hi + lo operands (HP = 3) except fp16 (HP = 1: both rounded to fp16); skip / sqrt(L)
    reaches the head as hi + lo (S16), or its hi plane alone at HP = 1.

The stochastic sets are drawn on the CPU (``OperandFormat(P, "fp16s", seed=...)``), not with the kernel's Philox
stream, so a bound built on them takes the worst of a few draws.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------
# parameters
# --------------------------------------------------------------------------------------
def build_state_dict(seed=0, in_dims=80, residual_channels=256, encoder_hidden=256,
                     residual_layers=20, dilation_cycle_length=1, out_std=0.02):
    """Random DiffNet weights created exactly the way the reference constructor does
    (module creation order and init calls of usr/diff/net.py:47-50, 58-64, 82-105), so
    ``torch.manual_seed(seed)`` gives the same numbers as ``DiffNet(in_dims)``.

    ``out_std``: the reference zero-initialises the last projection (net.py:105), which
    makes eps independent of x; fixtures re-draw it N(0, out_std) afterwards
    Pass ``None`` to keep the zeros.
    """
    import torch.nn as nn

    def conv(cin, cout, k, **kw):
        layer = nn.Conv1d(cin, cout, k, **kw)
        nn.init.kaiming_normal_(layer.weight)
        return layer

    C, H = residual_channels, encoder_hidden
    torch.manual_seed(seed)
    sd = OrderedDict()

    def put(prefix, mod):
        sd[prefix + ".weight"] = mod.weight.detach().clone()
        sd[prefix + ".bias"] = mod.bias.detach().clone()

    put("input_projection", conv(in_dims, C, 1))
    put("mlp.0", nn.Linear(C, C * 4))
    put("mlp.2", nn.Linear(C * 4, C))
    for i in range(residual_layers):
        d = 2 ** (i % dilation_cycle_length)
        put(f"residual_layers.{i}.dilated_conv", conv(C, 2 * C, 3, padding=d, dilation=d))
        put(f"residual_layers.{i}.diffusion_projection", nn.Linear(C, C))
        put(f"residual_layers.{i}.conditioner_projection", conv(H, 2 * C, 1))
        put(f"residual_layers.{i}.output_projection", conv(C, 2 * C, 1))
    put("skip_projection", conv(C, C, 1))
    last = conv(C, in_dims, 1)
    nn.init.zeros_(last.weight)
    if out_std is not None:
        nn.init.normal_(last.weight, std=out_std)
    put("output_projection", last)
    return sd


def num_layers(P):
    n = 0
    while f"residual_layers.{n}.dilated_conv.weight" in P:
        n += 1
    return n


# --------------------------------------------------------------------------------------
# DiffNet
# --------------------------------------------------------------------------------------
def sinusoidal_embedding(t, dim):
    """net.py:37-44.  t: [B] (int64 or float) -> [B, dim]."""
    half = dim // 2
    emb = math.log(10000) / (half - 1)
    emb = torch.exp(torch.arange(half) * -emb)
    emb = t[:, None] * emb[None, :]
    return torch.cat((emb.sin(), emb.cos()), dim=-1)


def mish(x):
    """diffusion.py:68-70."""
    return x * torch.tanh(F.softplus(x))


def step_embedding(P, t):
    """net.py:119-120: e(t) = mlp(SinusoidalPosEmb(t)) -> [B, C]."""
    C = P["mlp.2.weight"].shape[0]
    e = sinusoidal_embedding(t, C).to(P["mlp.0.weight"].dtype)     # integer t in a float64 model: fp32 angles
    e = F.linear(e, P["mlp.0.weight"], P["mlp.0.bias"])
    e = mish(e)
    return F.linear(e, P["mlp.2.weight"], P["mlp.2.bias"])


def dilated_conv(y, w, b, dilation):
    """The residual layers' conv (kernel 3, zero padding = dilation).  A dilation of at least T reaches wholly outside
    the utterance with both outer taps, so only the centre tap remains; above 1024 (dilation cycles > 11) that is
    computed directly rather than through a padding of 2 x dilation frames.  (Below, the padded conv is kept: the
    centre-tap conv sums in another order.)"""
    if dilation >= max(y.shape[-1], 1024):
        return F.conv1d(y, w[..., 1:2], b)
    return F.conv1d(y, w, b, padding=dilation, dilation=dilation)


def residual_block(P, i, x, cond, e, dilation):
    """net.py:66-78.  Returns ((x + residual)/sqrt2, skip)."""
    p = f"residual_layers.{i}."
    d = F.linear(e, P[p + "diffusion_projection.weight"], P[p + "diffusion_projection.bias"]).unsqueeze(-1)
    c = F.conv1d(cond, P[p + "conditioner_projection.weight"], P[p + "conditioner_projection.bias"])
    y = x + d
    y = dilated_conv(y, P[p + "dilated_conv.weight"], P[p + "dilated_conv.bias"], dilation) + c
    gate, filt = torch.chunk(y, 2, dim=1)
    y = torch.sigmoid(gate) * torch.tanh(filt)
    y = F.conv1d(y, P[p + "output_projection.weight"], P[p + "output_projection.bias"])
    residual, skip = torch.chunk(y, 2, dim=1)
    return (x + residual) / math.sqrt(2.0), skip


# --------------------------------------------------------------------------------------
# operand formats of the tensor-core kernels (see the module docstring)
# --------------------------------------------------------------------------------------
FORMATS = ("fp16", "fp16x2", "fp16x3", "fp16s")


def rn16(x):
    """round to nearest fp16, returned in x's dtype"""
    return x.half().to(x.dtype)


def hl16(x):
    """hi + lo fp16 pair of x, summed in x's dtype"""
    hi = rn16(x)
    return hi + rn16(x - hi)


def sr16(x, gen):
    """Stochastic rounding to fp16 (returned in x's dtype): P(up) = distance to the lower neighbour / ulp.
    gen: numpy RandomState."""
    a = x.detach().cpu().numpy().astype(np.float32)
    h = a.astype(np.float16)
    hf = h.astype(np.float32)
    up = np.nextafter(h, np.float16(np.inf)).astype(np.float32)
    dn = np.nextafter(h, np.float16(-np.inf)).astype(np.float32)
    lo = np.where(hf <= a, hf, dn)
    hi = np.where(hf <= a, up, hf)
    p = np.where(hi > lo, (a - lo) / np.maximum(hi - lo, 1e-30), 0.0)
    u = gen.random_sample(a.shape).astype(np.float32)
    return torch.from_numpy(np.where(u < p, hi, lo).astype(np.float32)).to(x.dtype)


class OperandFormat:
    """What one tensor-core precision rounds: ``act`` (y and z of the residual layers), ``head`` (operands of the input
    projection and the head) and ``weights(row)`` (the residual layers' conv and output-projection weights of FiLM-table
    row ``row``).  fp16s draws set r = row % sr_sets on first use, from numpy RandomState(seed + r)."""

    def __init__(self, P, name, sr_sets=64, seed=0):
        assert name in FORMATS, name
        self.P, self.name, self.sr_sets, self.seed = P, name, sr_sets, seed
        self.act = hl16 if name == "fp16x3" else rn16
        self.head = rn16 if name == "fp16" else hl16
        self._sets = {}

    def weights(self, row):
        key = row % self.sr_sets if self.name == "fp16s" else 0
        if key not in self._sets:
            gen = np.random.RandomState(self.seed + key)
            rnd = {"fp16": rn16, "fp16x2": hl16, "fp16x3": hl16, "fp16s": lambda w: sr16(w, gen)}[self.name]
            self._sets[key] = {k: rnd(v) for k, v in self.P.items()
                               if k.startswith("residual_layers.") and
                               k.endswith(("dilated_conv.weight", "output_projection.weight"))}
        return self._sets[key]


def operand_format(P, fmt):
    """None, a name in FORMATS, or an OperandFormat (kept: a loop's stochastic sets persist across its steps)"""
    return OperandFormat(P, fmt) if isinstance(fmt, str) else fmt


# Steps of the simulated evaluation, one function each (oracle/diffnet_edge_sensitivity.py replaces them with
# bug-shaped variants)
def sim_input_projection(P, spec, f):
    return F.relu(F.conv1d(f.head(spec[:, 0]), f.head(P["input_projection.weight"]), P["input_projection.bias"]))


def sim_film(P, e, i):
    """layer i's FiLM vectors d_i(t_b), [B, C, 1]"""
    p = f"residual_layers.{i}."
    return F.linear(e, P[p + "diffusion_projection.weight"], P[p + "diffusion_projection.bias"]).unsqueeze(-1)


def sim_dilated_conv(y, w, b, dilation):
    return dilated_conv(y, w, b, dilation)


def sim_skip_sum(skips):
    return sum(skips)


def _forward_fmt(P, spec, t, cond, cycle, f, row):
    L = num_layers(P)
    W = f.weights(row)
    x = sim_input_projection(P, spec, f)
    e = step_embedding(P, t)
    skips = []
    for i in range(L):
        p = f"residual_layers.{i}."
        c = F.conv1d(cond, P[p + "conditioner_projection.weight"], P[p + "conditioner_projection.bias"])
        y = sim_dilated_conv(f.act(x + sim_film(P, e, i)), W[p + "dilated_conv.weight"], P[p + "dilated_conv.bias"],
                             2 ** (i % cycle)) + c
        gate, filt = torch.chunk(y, 2, dim=1)
        z = torch.sigmoid(gate) * torch.tanh(filt)
        o = F.conv1d(f.act(z), W[p + "output_projection.weight"], P[p + "output_projection.bias"])
        residual, skip = torch.chunk(o, 2, dim=1)
        x = (x + residual) / math.sqrt(2.0)
        skips.append(skip)
    x = f.head(sim_skip_sum(skips) / math.sqrt(L))
    x = F.relu(F.conv1d(x, f.head(P["skip_projection.weight"]), P["skip_projection.bias"]))
    x = F.conv1d(f.head(x), f.head(P["output_projection.weight"]), P["output_projection.bias"])
    return x[:, None, :, :]


def diffnet_forward(P, spec, t, cond, dilation_cycle_length=1, taps=None, fmt=None, row=0):
    """net.py:107-130.  spec [B,1,M,T], t [B] int64, cond [B,H,T] -> eps [B,1,M,T].

    ``taps``: optional dict that receives the per-layer residual streams (``x{l}``: input of
    layer l, ``x{L}``: after the last layer) and the skip sum, for layer-by-layer checks.
    ``fmt`` / ``row``: simulate a tensor-core precision (module docstring) at FiLM-table row ``row``.
    """
    if fmt is not None:
        return _forward_fmt(P, spec, t, cond, dilation_cycle_length, operand_format(P, fmt), row)
    L = num_layers(P)
    x = spec[:, 0]
    x = F.relu(F.conv1d(x, P["input_projection.weight"], P["input_projection.bias"]))
    e = step_embedding(P, t)
    skips = []
    for i in range(L):
        if taps is not None:
            taps[f"x{i}"] = x.clone()
        x, skip = residual_block(P, i, x, cond, e, 2 ** (i % dilation_cycle_length))
        skips.append(skip)
    skip_sum = torch.sum(torch.stack(skips), dim=0)     # same reduction as net.py:126
    if taps is not None:
        taps[f"x{L}"] = x.clone()
        taps["skip_sum"] = skip_sum.clone()
    x = skip_sum / math.sqrt(L)
    x = F.relu(F.conv1d(x, P["skip_projection.weight"], P["skip_projection.bias"]))
    x = F.conv1d(x, P["output_projection.weight"], P["output_projection.bias"])
    return x[:, None, :, :]


# --------------------------------------------------------------------------------------
# schedule (float64 numpy -> fp32 buffers, exactly like the constructor)
# --------------------------------------------------------------------------------------
def linear_beta_schedule(timesteps, max_beta=0.01):
    """shallow_diffusion_tts.py:44-49."""
    return np.linspace(1e-4, max_beta, timesteps)


def cosine_beta_schedule(timesteps, s=0.008):
    """shallow_diffusion_tts.py:52-62."""
    steps = timesteps + 1
    x = np.linspace(0, steps, steps)
    ac = np.cos(((x / steps) + s) / (1 + s) * np.pi * 0.5) ** 2
    ac = ac / ac[0]
    betas = 1 - (ac[1:] / ac[:-1])
    return np.clip(betas, a_min=0, a_max=0.999)


SCHEDULE_BUFFERS = (
    "betas", "alphas_cumprod", "alphas_cumprod_prev", "sqrt_alphas_cumprod",
    "sqrt_one_minus_alphas_cumprod", "log_one_minus_alphas_cumprod",
    "sqrt_recip_alphas_cumprod", "sqrt_recipm1_alphas_cumprod", "posterior_variance",
    "posterior_log_variance_clipped", "posterior_mean_coef1", "posterior_mean_coef2",
)


def make_schedule(betas):
    """shallow_diffusion_tts.py:90-123: the 12 registered fp32 buffers, as a dict."""
    betas = np.asarray(betas, dtype=np.float64)
    alphas = 1. - betas
    ac = np.cumprod(alphas, axis=0)
    ac_prev = np.append(1., ac[:-1])
    pv = betas * (1. - ac_prev) / (1. - ac)
    f = lambda a: torch.tensor(a, dtype=torch.float32)
    return {
        "betas": f(betas),
        "alphas_cumprod": f(ac),
        "alphas_cumprod_prev": f(ac_prev),
        "sqrt_alphas_cumprod": f(np.sqrt(ac)),
        "sqrt_one_minus_alphas_cumprod": f(np.sqrt(1. - ac)),
        "log_one_minus_alphas_cumprod": f(np.log(1. - ac)),
        "sqrt_recip_alphas_cumprod": f(np.sqrt(1. / ac)),
        "sqrt_recipm1_alphas_cumprod": f(np.sqrt(1. / ac - 1)),
        "posterior_variance": f(pv),
        "posterior_log_variance_clipped": f(np.log(np.maximum(pv, 1e-20))),
        "posterior_mean_coef1": f(betas * np.sqrt(ac_prev) / (1. - ac)),
        "posterior_mean_coef2": f((1. - ac_prev) * np.sqrt(alphas) / (1. - ac)),
    }


# --------------------------------------------------------------------------------------
# samplers.  All batch items share the step index (the reference always calls with
# torch.full((b,), i)), so t is a python int here.
# --------------------------------------------------------------------------------------
def _tvec(t, b):
    return torch.full((b,), int(t), dtype=torch.long)


def p_sample(P, S, x, t, cond, noise, dilation_cycle_length=1, clip_denoised=True, fmt=None, row=0):
    """shallow_diffusion_tts.py:149-166 with the noise passed in (noise_like is :38-41)."""
    b = x.shape[0]
    eps = diffnet_forward(P, x, _tvec(t, b), cond, dilation_cycle_length, fmt=fmt, row=row)
    x_recon = S["sqrt_recip_alphas_cumprod"][t] * x - S["sqrt_recipm1_alphas_cumprod"][t] * eps
    if clip_denoised:
        x_recon = x_recon.clamp(-1., 1.)
    mean = S["posterior_mean_coef1"][t] * x_recon + S["posterior_mean_coef2"][t] * x
    nonzero = 0.0 if t == 0 else 1.0
    return mean + nonzero * (0.5 * S["posterior_log_variance_clipped"][t]).exp() * noise


def plms_x_pred(S, x, noise_t, t, interval):
    """get_x_pred, shallow_diffusion_tts.py:174-185 (fp32 tensor ops, same order)."""
    a_t = S["alphas_cumprod"][t].reshape(1, 1, 1, 1)
    if t < interval:
        a_prev = torch.ones_like(a_t)
    else:
        a_prev = S["alphas_cumprod"][max(t - interval, 0)].reshape(1, 1, 1, 1)
    a_t_sq, a_prev_sq = a_t.sqrt(), a_prev.sqrt()
    x_delta = (a_prev - a_t) * ((1 / (a_t_sq * (a_t_sq + a_prev_sq))) * x
                                - 1 / (a_t_sq * (((1 - a_prev) * a_t).sqrt() + ((1 - a_t) * a_prev).sqrt())) * noise_t)
    return x + x_delta


def plms_prime(noise_pred, noise_list):
    """the linear multistep combination of the current eps with the history, after the warm-up (:191-197)"""
    n = len(noise_list)
    if n == 1:
        return (3 * noise_pred - noise_list[-1]) / 2
    if n == 2:
        return (23 * noise_pred - 16 * noise_list[-1] + 5 * noise_list[-2]) / 12
    return (55 * noise_pred - 59 * noise_list[-1] + 37 * noise_list[-2] - 9 * noise_list[-3]) / 24


def p_sample_plms(P, S, x, t, interval, cond, noise_list, dilation_cycle_length=1, fmt=None, row=0, warm_row=1):
    """shallow_diffusion_tts.py:168-204.  ``noise_list`` is the caller-owned history (list).
    ``fmt``: a simulated precision; the evaluation at t is at table row ``row``, the warm-up's second at ``warm_row``."""
    b = x.shape[0]
    noise_pred = diffnet_forward(P, x, _tvec(t, b), cond, dilation_cycle_length, fmt=fmt, row=row)
    if len(noise_list) == 0:
        x_pred = plms_x_pred(S, x, noise_pred, t, interval)
        noise_pred_prev = diffnet_forward(P, x_pred, _tvec(max(t - interval, 0), b), cond, dilation_cycle_length,
                                          fmt=fmt, row=warm_row)
        prime = (noise_pred + noise_pred_prev) / 2
    else:
        prime = plms_prime(noise_pred, noise_list)
    x_prev = plms_x_pred(S, x, prime, t, interval)
    noise_list.append(noise_pred)
    if len(noise_list) > 4:          # deque(maxlen=4), :99
        del noise_list[0]
    return x_prev


def sample_ddpm(P, S, x, cond, K, noise, dilation_cycle_length=1, fmt=None, n_steps=None):
    """Loop :269-270.  noise[j] is used at the j-th executed step (t = K-1-j), step j at table row j.
    ``n_steps``: stop after that many steps (t = K-1 .. K-n_steps), as dsx_sample_ddpm does."""
    fmt = operand_format(P, fmt)
    for j, t in enumerate(reversed(range(0, K))):
        if n_steps is not None and j == n_steps:
            break
        x = p_sample(P, S, x, t, cond, noise[j], dilation_cycle_length, fmt=fmt, row=j)
    return x


def sample_plms(P, S, x, cond, K, interval, dilation_cycle_length=1, fmt=None):
    """Loop :261-267.  Step j at table row j, the warm-up's second evaluation at row n (the number of steps)."""
    fmt = operand_format(P, fmt)
    hist = []
    steps = list(reversed(range(0, K, interval)))
    for j, t in enumerate(steps):
        x = p_sample_plms(P, S, x, t, interval, cond, hist, dilation_cycle_length, fmt=fmt, row=j, warm_row=len(steps))
    return x


def norm_spec(x, spec_min, spec_max):
    """:278-279.  x [B,T,M]; spec_min/max [1,1,M]."""
    return (x - spec_min) / (spec_max - spec_min) * 2 - 1


def denorm_spec(x, spec_min, spec_max):
    """:281-282."""
    return (x + 1) / 2 * (spec_max - spec_min) + spec_min


def q_sample(S, x_start, t, noise):
    """:206-211."""
    return S["sqrt_alphas_cumprod"][t] * x_start + S["sqrt_one_minus_alphas_cumprod"][t] * noise


def infer_loop(P, S, cond, K_step, spec_min, spec_max, *, fs2_mel=None, start_noise=None,
               x_start=None, step_noise=None, pndm_speedup=None, mel2ph=None,
               dilation_cycle_length=1, fmt=None):
    """The infer branch of GaussianDiffusion.forward, :248-275, after ``self.fs2``.

    cond [B,H,T].  Shallow start: fs2_mel [B,T,M] + start_noise [B,1,M,T];
    gaussian start: x_start [B,1,M,T].  Returns mel_out [B,T,M] (denormalised, masked).
    """
    if x_start is None:
        m = norm_spec(fs2_mel, spec_min, spec_max).transpose(1, 2)[:, None, :, :]
        x = q_sample(S, m, K_step - 1, start_noise)
    else:
        x = x_start
    if pndm_speedup:
        x = sample_plms(P, S, x, cond, K_step, pndm_speedup, dilation_cycle_length, fmt=fmt)
    else:
        x = sample_ddpm(P, S, x, cond, K_step, step_noise, dilation_cycle_length, fmt=fmt)
    x = x[:, 0].transpose(1, 2)
    out = denorm_spec(x, spec_min, spec_max)
    if mel2ph is not None:
        out = out * ((mel2ph > 0).float()[:, :, None])
    return out
