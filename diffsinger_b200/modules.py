"""Host-side mirror of the reference's class surface for the hot path:

  * ``DiffNet``            usr/diff/net.py:81-130        (same ctor, parameter names, forward contract)
  * ``GaussianDiffusion``  usr/diff/shallow_diffusion_tts.py:71-282 (same ctor, buffers, forward / ret dict)

Same state-dict keys (``denoise_fn.residual_layers.{l}.dilated_conv.weight`` ...), so reference
checkpoints load with ``strict=True``.  Under ``torch.no_grad`` / ``infer=True`` every evaluation goes
to the sm_90a kernels through the C ABI and fails loudly on CPU tensors.  The training branch
(``p_losses`` under autograd) is outside this round's scope (section 8f rank 4): it keeps the module
graph in plain PyTorch ops so existing training code still runs, and is never used for inference.
"""
import math
from collections import deque
from functools import partial

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _capi
from .sampler import DsxSampler, DsxError, _need_cuda


def _get_hparams(hp):
    if hp is not None:
        return hp
    try:                                   # inside the reference tree: the process-global config dict
        from utils.hparams import hparams  # type: ignore
        return hparams
    except Exception as e:                 # pragma: no cover
        raise DsxError("no hparams given and the reference's utils.hparams is not importable") from e


class Mish(nn.Module):
    """usr/diff/diffusion.py:68-70"""

    def forward(self, x):
        return x * torch.tanh(F.softplus(x))


class SinusoidalPosEmb(nn.Module):
    """usr/diff/net.py:32-44"""

    def __init__(self, dim):
        super().__init__()
        self.dim = dim

    def forward(self, x):
        half = self.dim // 2
        emb = math.log(10000) / (half - 1)
        emb = torch.exp(torch.arange(half, device=x.device) * -emb)
        emb = x[:, None] * emb[None, :]
        return torch.cat((emb.sin(), emb.cos()), dim=-1)


def Conv1d(*args, **kwargs):
    layer = nn.Conv1d(*args, **kwargs)
    nn.init.kaiming_normal_(layer.weight)
    return layer


class ResidualBlock(nn.Module):
    """Parameter container with the reference's names (usr/diff/net.py:58-64); the autograd forward is
    only used by the training branch."""

    def __init__(self, encoder_hidden, residual_channels, dilation):
        super().__init__()
        self.dilated_conv = Conv1d(residual_channels, 2 * residual_channels, 3, padding=dilation, dilation=dilation)
        self.diffusion_projection = nn.Linear(residual_channels, residual_channels)
        self.conditioner_projection = Conv1d(encoder_hidden, 2 * residual_channels, 1)
        self.output_projection = Conv1d(residual_channels, 2 * residual_channels, 1)

    def forward(self, x, conditioner, diffusion_step):
        d = self.diffusion_projection(diffusion_step).unsqueeze(-1)
        y = self.dilated_conv(x + d) + self.conditioner_projection(conditioner)
        gate, filt = torch.chunk(y, 2, dim=1)
        y = self.output_projection(torch.sigmoid(gate) * torch.tanh(filt))
        residual, skip = torch.chunk(y, 2, dim=1)
        return (x + residual) / math.sqrt(2.0), skip


class DiffNet(nn.Module):
    """Drop-in for usr.diff.net.DiffNet: ``DiffNet(in_dims=80)`` reads ``hidden_size``,
    ``residual_layers``, ``residual_channels``, ``dilation_cycle_length`` from hparams (net.py:84-89)."""

    def __init__(self, in_dims=80, hparams=None, precision=None):
        super().__init__()
        hp = _get_hparams(hparams)
        self.params = params = dict(
            encoder_hidden=hp["hidden_size"], residual_layers=hp["residual_layers"],
            residual_channels=hp["residual_channels"], dilation_cycle_length=hp["dilation_cycle_length"])
        C = params["residual_channels"]
        self.input_projection = Conv1d(in_dims, C, 1)
        self.diffusion_embedding = SinusoidalPosEmb(C)
        self.mlp = nn.Sequential(nn.Linear(C, C * 4), Mish(), nn.Linear(C * 4, C))
        self.residual_layers = nn.ModuleList([
            ResidualBlock(params["encoder_hidden"], C, 2 ** (i % params["dilation_cycle_length"]))
            for i in range(params["residual_layers"])])
        self.skip_projection = Conv1d(C, C, 1)
        self.output_projection = Conv1d(C, in_dims, 1)
        nn.init.zeros_(self.output_projection.weight)
        self._dsx = None
        self._dsx_precision = precision or hp.get("dsx_precision")

    @property
    def dsx(self):
        if self._dsx is None:
            object.__setattr__(self, "_dsx", DsxSampler(self, self._dsx_precision, self.params["dilation_cycle_length"]))
        return self._dsx

    def forward(self, spec, diffusion_step, cond):
        """spec [B,1,M,T], diffusion_step [B], cond [B,H,T] -> [B,1,M,T] (net.py:107-130).

        Training mode (``self.training``: p_losses under autograd) or an input that itself requires grad keeps the module
        graph in plain PyTorch ops; everything else -- ``model.eval()``, with or without ``torch.no_grad()`` -- is inference
        and goes to libdsx (no silent PyTorch path: CPU tensors / a missing library raise)."""
        if self.training or (torch.is_grad_enabled() and spec.requires_grad):
            return self._forward_autograd(spec, diffusion_step, cond)
        return self.dsx.diffnet_forward(spec, diffusion_step, cond)

    def __getstate__(self):
        # the lazily created sampler holds a ctypes handle: copies (EMA deepcopy, torch.save of the module) rebuild theirs
        state = self.__dict__.copy()
        state["_dsx"] = None
        return state

    def _forward_autograd(self, spec, diffusion_step, cond):
        # training branch only (p_losses); not a fallback for inference
        x = F.relu(self.input_projection(spec[:, 0]))
        e = self.mlp(self.diffusion_embedding(diffusion_step))
        skip = []
        for layer in self.residual_layers:
            x, s = layer(x, cond, e)
            skip.append(s)
        x = torch.sum(torch.stack(skip), dim=0) / math.sqrt(len(self.residual_layers))
        x = self.output_projection(F.relu(self.skip_projection(x)))
        return x[:, None, :, :]


# ---- schedules (usr/diff/shallow_diffusion_tts.py:44-68) -------------------------------------------
def linear_beta_schedule(timesteps, max_beta=0.01):
    return np.linspace(1e-4, max_beta, timesteps)


def cosine_beta_schedule(timesteps, s=0.008):
    steps = timesteps + 1
    x = np.linspace(0, steps, steps)
    ac = np.cos(((x / steps) + s) / (1 + s) * np.pi * 0.5) ** 2
    ac = ac / ac[0]
    return np.clip(1 - (ac[1:] / ac[:-1]), a_min=0, a_max=0.999)


def register_schedule_buffers(module, betas, spec_min, spec_max, keep_bins):
    """The buffers of GaussianDiffusion.__init__ (shallow_diffusion_tts.py:90-126): float64 numpy -> fp32."""
    alphas = 1. - betas
    ac = np.cumprod(alphas, axis=0)
    ac_prev = np.append(1., ac[:-1])
    f = partial(torch.tensor, dtype=torch.float32)
    reg = module.register_buffer
    reg('betas', f(betas))
    reg('alphas_cumprod', f(ac))
    reg('alphas_cumprod_prev', f(ac_prev))
    reg('sqrt_alphas_cumprod', f(np.sqrt(ac)))
    reg('sqrt_one_minus_alphas_cumprod', f(np.sqrt(1. - ac)))
    reg('log_one_minus_alphas_cumprod', f(np.log(1. - ac)))
    reg('sqrt_recip_alphas_cumprod', f(np.sqrt(1. / ac)))
    reg('sqrt_recipm1_alphas_cumprod', f(np.sqrt(1. / ac - 1)))
    pv = betas * (1. - ac_prev) / (1. - ac)
    reg('posterior_variance', f(pv))
    reg('posterior_log_variance_clipped', f(np.log(np.maximum(pv, 1e-20))))
    reg('posterior_mean_coef1', f(betas * np.sqrt(ac_prev) / (1. - ac)))
    reg('posterior_mean_coef2', f((1. - ac_prev) * np.sqrt(alphas) / (1. - ac)))
    reg('spec_min', torch.FloatTensor(spec_min)[None, None, :keep_bins])
    reg('spec_max', torch.FloatTensor(spec_max)[None, None, :keep_bins])


class DsxInferMixin:
    """The sampling half of GaussianDiffusion, shared by the standalone class below and by the subclass
    that `dropin.install()` derives from the reference's own GaussianDiffusion."""

    def _dsx_sampler(self):
        s = getattr(self.denoise_fn, "dsx", None)
        if s is None:
            s = self.__dict__.get("_dsx_sampler_obj")
            if s is None:
                s = DsxSampler(self.denoise_fn, self._dsx_hparams().get("dsx_precision"))
                self.__dict__["_dsx_sampler_obj"] = s
        return s

    def _dsx_hparams(self):
        return getattr(self, "_hparams", None) or _get_hparams(None)

    def _dsx_ready(self, device):
        s = self._dsx_sampler()
        s.ensure_weights(device)
        s.set_schedule({n: getattr(self, n) for n in _capi.SCHEDULE_BUFFERS})
        return s

    def dsx_infer(self, ret, cond, mel2ph, step_noise=None, start_noise=None, seed=None, fs2_mel=None, x_start=None,
                  K_step=None, keep_fs2_mel=True, allow_pndm=True):
        """Everything after ``self.fs2`` in an infer branch: shallow_diffusion_tts.py:248-275 (defaults), the Offline
        variant :306-322 (fs2_mel given, no mask, DDPM only) and the older sampler diffusion.py:313-320 (x_start given,
        K_step = num_timesteps)."""
        hp = self._dsx_hparams()
        if fs2_mel is None and x_start is None:
            fs2_mel = ret['mel_out']
        _need_cuda(cond, fs2_mel, x_start)
        dev = cond.device
        s = self._dsx_ready(dev)
        if keep_fs2_mel:
            ret['fs2_mel'] = ret['mel_out']
        gaussian = x_start is None and hp.get('gaussian_start') is not None and hp['gaussian_start']
        if seed is None:
            seed = int(torch.randint(0, 2 ** 62, (1,)).item())
        if gaussian:
            print('===> gaussion start.')
            x_start = torch.randn((cond.shape[0], 1, self.mel_bins, cond.shape[2]), device=dev)
        interval = int(hp.get('pndm_speedup') or 0) if allow_pndm else 0
        ret['mel_out'] = s.infer(cond, self.K_step if K_step is None else K_step, self.spec_min, self.spec_max,
                                 fs2_mel=None if x_start is not None else fs2_mel, start_noise=start_noise,
                                 x_start=x_start, step_noise=step_noise, seed=seed, mel2ph=mel2ph,
                                 pndm_interval=interval)
        return ret

    @torch.no_grad()
    def p_sample(self, x, t, cond, clip_denoised=True, repeat_noise=False):
        """One DDPM step (shallow_diffusion_tts.py:159-166); all batch items must share t."""
        assert clip_denoised and not repeat_noise, "only the reference's default arguments are supported"
        tt = int(t[0])
        s = self._dsx_ready(x.device)
        noise = torch.randn((1,) + tuple(x.shape), device=x.device)
        return s.sample_ddpm(x, cond, tt + 1, 1, noise=noise)

    @torch.no_grad()
    def p_sample_plms(self, x, t, interval, cond, clip_denoised=True, repeat_noise=False):
        """One PNDM step with the module-held history (shallow_diffusion_tts.py:168-204).  The fused loop
        is ``dsx_sample_plms``; this per-step form exists for callers that drive the loop themselves."""
        tt = int(t[0])
        s = self._dsx_ready(x.device)
        b = x.shape[0]
        full = lambda v: torch.full((b,), v, device=x.device, dtype=torch.long)
        nl = self.noise_list
        # network evaluations and the multistep algebra both run in libdsx (the conditioner pack + projection are re-used
        # from the previous step's call: DsxSampler._cond_arg)
        noise_pred = s.diffnet_forward(x, full(tt), cond)
        if len(nl) == 0:
            x_mid = s.plms_update(x, [noise_pred], 0, tt, interval)
            noise_pred_prev = s.diffnet_forward(x_mid, full(max(tt - interval, 0)), cond)
            out = s.plms_update(x, [noise_pred, noise_pred_prev], 1, tt, interval)
        else:
            hist = [noise_pred] + [nl[-1 - i] for i in range(min(len(nl), 3))]
            out = s.plms_update(x, hist, len(hist), tt, interval)
        nl.append(noise_pred)
        return out


class GaussianDiffusion(DsxInferMixin, nn.Module):
    """Standalone mirror of usr.diff.shallow_diffusion_tts.GaussianDiffusion.  The conditioner
    (FastSpeech2 / FastSpeech2MIDI, out of scope) is injected as ``fs2``; inside the reference tree
    ``dropin.install()`` gives the subclass of the reference's own class instead."""

    def __init__(self, phone_encoder, out_dims, denoise_fn, timesteps=1000, K_step=1000, loss_type='l1', betas=None,
                 spec_min=None, spec_max=None, fs2=None, hparams=None):
        super().__init__()
        hp = _get_hparams(hparams)
        self._hparams = hp
        self.denoise_fn = denoise_fn
        if fs2 is None:
            raise DsxError("diffsinger_b200.GaussianDiffusion needs the conditioner module as fs2= "
                           "(FastSpeech2 is outside this package's scope); inside the reference tree use "
                           "diffsinger_b200.dropin.install() instead")
        self.fs2 = fs2
        self.mel_bins = out_dims
        if betas is not None:
            betas = betas.detach().cpu().numpy() if isinstance(betas, torch.Tensor) else betas
        elif 'schedule_type' in hp.keys():
            if hp['schedule_type'] == 'linear':
                betas = linear_beta_schedule(timesteps, hp.get('max_beta', 0.01))
            else:
                betas = cosine_beta_schedule(timesteps)
        else:
            betas = cosine_beta_schedule(timesteps)
        self.num_timesteps = int(betas.shape[0])
        self.K_step = K_step
        self.loss_type = loss_type
        self.noise_list = deque(maxlen=4)
        register_schedule_buffers(self, betas, spec_min, spec_max, hp['keep_bins'])

    def q_sample(self, x_start, t, noise=None):
        noise = torch.randn_like(x_start) if noise is None else noise
        e = lambda a: a.gather(-1, t).reshape(t.shape[0], 1, 1, 1)
        return e(self.sqrt_alphas_cumprod) * x_start + e(self.sqrt_one_minus_alphas_cumprod) * noise

    def p_losses(self, x_start, t, cond, noise=None, nonpadding=None):
        noise = torch.randn_like(x_start) if noise is None else noise
        x_recon = self.denoise_fn(self.q_sample(x_start, t, noise), t, cond)
        if self.loss_type == 'l1':
            if nonpadding is not None:
                return ((noise - x_recon).abs() * nonpadding.unsqueeze(1)).mean()
            return (noise - x_recon).abs().mean()
        if self.loss_type == 'l2':
            return F.mse_loss(noise, x_recon)
        raise NotImplementedError()

    def forward(self, txt_tokens, mel2ph=None, spk_embed=None, ref_mels=None, f0=None, uv=None, energy=None,
                infer=False, **kwargs):
        b, device = txt_tokens.shape[0], txt_tokens.device
        dsx_kw = {k: kwargs.pop(k) for k in list(kwargs) if k.startswith('dsx_')}
        ret = self.fs2(txt_tokens, mel2ph, spk_embed, ref_mels, f0, uv, energy, skip_decoder=(not infer),
                       infer=infer, **kwargs)
        cond = ret['decoder_inp'].transpose(1, 2)
        if not infer:
            t = torch.randint(0, self.K_step, (b,), device=device).long()
            x = self.norm_spec(ref_mels).transpose(1, 2)[:, None, :, :]
            ret['diff_loss'] = self.p_losses(x, t, cond)
            return ret
        with torch.no_grad():
            return self.dsx_infer(ret, cond, mel2ph, step_noise=dsx_kw.get('dsx_step_noise'),
                                  start_noise=dsx_kw.get('dsx_start_noise'), seed=dsx_kw.get('dsx_seed'))

    def norm_spec(self, x):
        return (x - self.spec_min) / (self.spec_max - self.spec_min) * 2 - 1

    def denorm_spec(self, x):
        return (x + 1) / 2 * (self.spec_max - self.spec_min) + self.spec_min

    def cwt2f0_norm(self, cwt_spec, mean, std, mel2ph):
        return self.fs2.cwt2f0_norm(cwt_spec, mean, std, mel2ph)

    def out2mel(self, x):
        return x
