"""TEST INFRASTRUCTURE ONLY -- functional torch fp32 restatement of the reference's FFT diffusion denoiser
(usr/diff/candidate_decoder.py:35-100: FastspeechDecoder with an input projection, the DiffNet step embedding,
get_decode_inp and get_mel_out) and of the sampling loops of GaussianDiffusion around it
(usr/diff/shallow_diffusion_tts.py:134-275), over a state dict ``sd`` with the reference's names.  ``hp`` holds the
decoder's hparams (oracle.fs2dec_oracle) plus residual_channels and audio_num_mel_bins.

``forward_fp16_sim`` rounds operands as the dsx kernels do, for sizing the GPU tests' bounds; ``loop_error`` applies it to
a whole sampling loop.  Run this file to print that simulation for the shipped configuration."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import diffnet_oracle as N
from oracle import fs2dec_oracle as D

HPARAMS_POPCS = dict(D.HPARAMS_POPCS, residual_channels=256, audio_num_mel_bins=80)
MEL_OUT = 80            # get_mel_out = Linear(hidden_size, 80)


def extra_shapes(hp):
    """name -> shape of the parameters FFT adds to the decoder, in the reference's order"""
    H, dim, M = int(hp['hidden_size']), int(hp['residual_channels']), int(hp['audio_num_mel_bins'])
    return {"input_projection.weight": (dim, M, 1), "input_projection.bias": (dim,),
            "mlp.0.weight": (4 * dim, dim), "mlp.0.bias": (4 * dim,), "mlp.2.weight": (dim, 4 * dim), "mlp.2.bias": (dim,),
            "get_mel_out.weight": (MEL_OUT, H), "get_mel_out.bias": (MEL_OUT,),
            "get_decode_inp.weight": (H, H + 2 * dim), "get_decode_inp.bias": (H,)}


def state_dict_shapes(hp):
    return dict(D.state_dict_shapes(hp), **extra_shapes(hp))


def random_state_dict(seed, hp):
    """The decoder's seeded parameters (fs2dec_oracle.random_state_dict(seed)), then the FFT's own from
    RandomState(seed + 1): Xavier-uniform weights, biases 0.05 * normal."""
    out = D.random_state_dict(seed, hp)
    rs = np.random.RandomState(seed + 1)
    for name, shape in extra_shapes(hp).items():
        if name.endswith("bias"):
            v = 0.05 * rs.standard_normal(shape)
        else:
            rf = int(np.prod(shape[2:]))
            a = np.sqrt(6.0 / (shape[1] * rf + shape[0] * rf))
            v = rs.uniform(-a, a, shape)
        out[name] = torch.from_numpy(np.asarray(v, np.float32))
    return out


def _p(w):
    # a module's weight requires grad, and ATen picks how it folds a strided 3-d input by that (see fs2dec_oracle._ffn)
    return w if w.requires_grad else torch.nn.Parameter(w, requires_grad=True)


def step_embedding(sd, t, dim):
    """mlp(SinusoidalPosEmb(dim)(t)), candidate_decoder.py:14-26 and :41-46 (Mish of usr/diff/diffusion.py)"""
    half = dim // 2
    emb = math.log(10000) / (half - 1)
    emb = torch.exp(torch.arange(half, device=t.device) * -emb)
    emb = t[:, None] * emb[None, :]
    e = torch.cat((emb.sin(), emb.cos()), dim=-1)
    e = F.linear(e, _p(sd["mlp.0.weight"]), sd["mlp.0.bias"])
    e = N.mish(e)
    return F.linear(e, _p(sd["mlp.2.weight"]), sd["mlp.2.bias"])


def decode_inp(sd, spec, t, cond, hp):
    """candidate_decoder.py:57-70: get_decode_inp(cat[input_projection(x), cond, mlp(emb(t)) over T]) -> [B, T, H]"""
    x = F.conv1d(spec[:, 0], _p(sd["input_projection.weight"]), sd["input_projection.bias"]).permute([0, 2, 1])
    e = step_embedding(sd, t, int(hp['residual_channels']))
    c = cond.permute([0, 2, 1])
    te = e[:, None, :].repeat([1, c.shape[1], 1])
    return F.linear(torch.cat([x, c, te], dim=-1), _p(sd["get_decode_inp.weight"]), sd["get_decode_inp.bias"])


def forward(sd, spec, t, cond, hp):
    """FFT.forward(spec [B, 1, 80, T], t [B], cond [B, H, T]) -> [B, 1, 80, T]"""
    x = D.decoder(sd, decode_inp(sd, spec, t, cond, hp), hp)
    return F.linear(x, _p(sd["get_mel_out.weight"]), sd["get_mel_out.bias"]).permute([0, 2, 1])[:, None, :, :]


def forward_fp16_sim(sd, spec, t, cond, hp):
    """forward with the dsx kernels' operand rounding: decoder_inp in fp32 (its GEMMs use hi+lo fp16 pairs), the decoder
    stack as fs2dec_oracle.decoder_fp16_sim, and get_mel_out over fp16 LayerNorm outputs and fp16 weights."""
    r = lambda v: v.half().float()
    x = D.decoder_fp16_sim(sd, decode_inp(sd, spec, t, cond, hp), hp)
    return (r(x) @ r(sd["get_mel_out.weight"]).t() + sd["get_mel_out.bias"]).permute([0, 2, 1])[:, None, :, :]


# ---- sampling loops (shallow_diffusion_tts.py), as oracle.diffnet_oracle restates them for DiffNet ----------------
def p_sample(fn, S, x, t, cond, noise):
    """:149-166 with the noise passed in; fn(spec, t [B], cond) is the denoiser"""
    eps = fn(x, N._tvec(t, x.shape[0]).to(x.device), cond)
    x_recon = S["sqrt_recip_alphas_cumprod"][t] * x - S["sqrt_recipm1_alphas_cumprod"][t] * eps
    x_recon = x_recon.clamp(-1., 1.)
    mean = S["posterior_mean_coef1"][t] * x_recon + S["posterior_mean_coef2"][t] * x
    nonzero = 0.0 if t == 0 else 1.0
    return mean + nonzero * (0.5 * S["posterior_log_variance_clipped"][t]).exp() * noise


def p_sample_plms(fn, S, x, t, interval, cond, noise_list):
    """:168-204; noise_list is the caller-owned history"""
    b = x.shape[0]
    tv = lambda v: N._tvec(v, b).to(x.device)
    noise_pred = fn(x, tv(t), cond)
    n = len(noise_list)
    if n == 0:
        x_pred = N.plms_x_pred(S, x, noise_pred, t, interval)
        prime = (noise_pred + fn(x_pred, tv(max(t - interval, 0)), cond)) / 2
    elif n == 1:
        prime = (3 * noise_pred - noise_list[-1]) / 2
    elif n == 2:
        prime = (23 * noise_pred - 16 * noise_list[-1] + 5 * noise_list[-2]) / 12
    else:
        prime = (55 * noise_pred - 59 * noise_list[-1] + 37 * noise_list[-2] - 9 * noise_list[-3]) / 24
    x_prev = N.plms_x_pred(S, x, prime, t, interval)
    noise_list.append(noise_pred)
    if len(noise_list) > 4:
        del noise_list[0]
    return x_prev


def infer_loop(fn, S, cond, K_step, spec_min, spec_max, *, fs2_mel, start_noise, step_noise=None, pndm_speedup=None,
               mel2ph=None):
    """The infer branch of GaussianDiffusion.forward (:248-275) after self.fs2, shallow start -> mel_out [B, T, M].
    S: the schedule buffers on the device of the inputs."""
    x = N.q_sample(S, N.norm_spec(fs2_mel, spec_min, spec_max).transpose(1, 2)[:, None, :, :], K_step - 1, start_noise)
    if pndm_speedup:
        hist = []
        for t in reversed(range(0, K_step, pndm_speedup)):
            x = p_sample_plms(fn, S, x, t, pndm_speedup, cond, hist)
    else:
        for j, t in enumerate(reversed(range(0, K_step))):
            x = p_sample(fn, S, x, t, cond, step_noise[j])
    out = N.denorm_spec(x[:, 0].transpose(1, 2), spec_min, spec_max)
    if mel2ph is not None:
        out = out * ((mel2ph > 0).float()[:, :, None])
    return out


def fixture_inputs(seed, B, T, hp):
    """cond [B, H, T] (seeded normals, utterance 1 zero from 3T/4: a padded tail of decoder_inp), fs2_mel [B, T, 80]
    around the popcs spectrum range, mel2ph [B, T] (0 on the same tail), start noise [B, 1, 80, T]"""
    rs = np.random.RandomState(seed)
    H = int(hp['hidden_size'])
    cond = torch.from_numpy(rs.standard_normal((B, H, T)).astype(np.float32))
    fs2_mel = torch.from_numpy((rs.standard_normal((B, T, 80)) * 1.5 - 4.0).astype(np.float32))
    start = torch.from_numpy(rs.standard_normal((B, 1, 80, T)).astype(np.float32))
    mel2ph = torch.ones(B, T, dtype=torch.long)
    if B > 1:
        cond[1, :, 3 * T // 4:] = 0
        mel2ph[1, 3 * T // 4:] = 0
    return cond, fs2_mel, mel2ph, start


def step_noise(seed, K, B, T):
    return torch.from_numpy(np.random.RandomState(seed).standard_normal((K, B, 1, 80, T)).astype(np.float32))


def loop_error(sd, hp, S, B=2, T=200, K=51, seed=5):
    """DDPM K-step infer loop with forward_fp16_sim against fp32 forward: (max, mean) |d| of mel_out, and of eps after
    one evaluation."""
    cond, fs2_mel, mel2ph, start = fixture_inputs(seed, B, T, hp)
    noise = step_noise(seed + 1, K, B, T)
    smin, smax = torch.full((1, 1, 80), -6.0), torch.full((1, 1, 80), 1.5)
    with torch.no_grad():
        args = dict(fs2_mel=fs2_mel, start_noise=start, step_noise=noise, mel2ph=mel2ph)
        ref = infer_loop(lambda *a: forward(sd, *a, hp), S, cond, K, smin, smax, **args)
        sim = infer_loop(lambda *a: forward_fp16_sim(sd, *a, hp), S, cond, K, smin, smax, **args)
        x = torch.randn(B, 1, 80, T, generator=torch.Generator().manual_seed(seed))
        t = torch.tensor([K - 1, 3][:B])
        e = (forward(sd, x, t, cond, hp) - forward_fp16_sim(sd, x, t, cond, hp)).abs()
    d = (ref - sim).abs()
    return d.max().item(), d.mean().item(), e.max().item(), e.mean().item(), ref.abs().max().item()


if __name__ == "__main__":
    torch.set_num_threads(8)
    hp = HPARAMS_POPCS
    sd = random_state_dict(31, hp)
    S = N.make_schedule(N.linear_beta_schedule(100, 0.06))
    print("K=51 DDPM mel max/mean |d|, one-eval eps max/mean |d|, |mel| max: %.3e %.3e %.3e %.3e %.2f" %
          loop_error(sd, hp, S))
