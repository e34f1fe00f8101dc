"""Writes a STAND-IN for the reference tree (the few modules `diffsinger_b200.dropin` touches) into a directory, so the
installed subclasses can be driven end to end without a checkout of the reference.

The stand-in keeps the reference's module paths, class names, constructor signatures and attributes
(usr/diff/shallow_diffusion_tts.py:71-126,285-290; usr/diff/diffusion.py:178-232; usr/diff/net.py:81-105; usr/task.py:10-12)
but none of its sampling code: its own `forward` raises, so a test that passes proves the call went through the dropin
subclass into libdsx.  Schedule buffers come from the same float64 formulas (diffsinger_b200.modules), which
tests/test_host_cpu.py pins to the live reference's buffers.
"""
import os
import textwrap

FILES = {
    "utils/__init__.py": "",
    "utils/hparams.py": """
        hparams = {}

        def set_hparams(**kw):
            hparams.update(kw)
    """,
    "usr/__init__.py": "",
    "usr/diff/__init__.py": "",
    "usr/diff/net.py": """
        import torch.nn as nn

        class DiffNet(nn.Module):          # replaced by diffsinger_b200.DiffNet at install time
            def __init__(self, in_dims=80):
                super().__init__()
                raise RuntimeError("stand-in DiffNet: dropin.install() should have replaced this class")
    """,
    "usr/diff/shallow_diffusion_tts.py": """
        from collections import deque
        import torch
        import torch.nn as nn
        from utils.hparams import hparams
        from diffsinger_b200.modules import register_schedule_buffers, linear_beta_schedule, cosine_beta_schedule

        class _NoFS2(nn.Module):
            def forward(self, *a, **k):
                raise RuntimeError("stand-in: set model.fs2 to a stub")

        class GaussianDiffusion(nn.Module):
            def __init__(self, phone_encoder, out_dims, denoise_fn, timesteps=1000, K_step=1000, loss_type='l1', betas=None,
                         spec_min=None, spec_max=None):
                super().__init__()
                self.denoise_fn = denoise_fn
                self.fs2 = _NoFS2()
                self.mel_bins = out_dims
                if betas is not None:
                    betas = betas.detach().cpu().numpy() if isinstance(betas, torch.Tensor) else betas
                elif hparams.get('schedule_type') == 'linear':
                    betas = linear_beta_schedule(timesteps, hparams.get('max_beta', 0.01))
                else:
                    betas = cosine_beta_schedule(timesteps)
                self.num_timesteps = int(betas.shape[0])
                self.K_step = K_step
                self.loss_type = loss_type
                self.noise_list = deque(maxlen=4)
                register_schedule_buffers(self, betas, spec_min, spec_max, hparams['keep_bins'])

            def forward(self, *a, **k):
                raise RuntimeError("stand-in forward: the dropin subclass must handle infer=True")

        class OfflineGaussianDiffusion(GaussianDiffusion):
            pass
    """,
    "usr/diff/diffusion.py": """
        import torch
        import torch.nn as nn
        from utils.hparams import hparams
        from diffsinger_b200.modules import register_schedule_buffers, cosine_beta_schedule

        class GaussianDiffusion(nn.Module):
            def __init__(self, phone_encoder, out_dims, denoise_fn, timesteps=1000, loss_type='l1', betas=None, spec_min=None,
                         spec_max=None):
                super().__init__()
                self.denoise_fn = denoise_fn
                self.fs2 = None
                self.mel_bins = out_dims
                betas = cosine_beta_schedule(timesteps) if betas is None else betas
                self.num_timesteps = int(betas.shape[0])
                self.loss_type = loss_type
                register_schedule_buffers(self, betas, spec_min, spec_max, hparams['keep_bins'])

            def forward(self, *a, **k):
                raise RuntimeError("stand-in forward: the dropin subclass must handle infer=True")
    """,
    "usr/task.py": """
        from .diff.diffusion import GaussianDiffusion
        from .diff.net import DiffNet

        DIFF_DECODERS = {'wavenet': lambda hp: DiffNet(hp['audio_num_mel_bins'])}
    """,
    "usr/diffsinger_task.py": """
        from .diff.shallow_diffusion_tts import GaussianDiffusion, OfflineGaussianDiffusion
        from .diff.net import DiffNet

        DIFF_DECODERS = {'wavenet': lambda hp: DiffNet(hp['audio_num_mel_bins'])}
    """,
}


def write_tree(dst):
    for rel, body in FILES.items():
        path = os.path.join(dst, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as f:
            f.write(textwrap.dedent(body).lstrip("\n"))
    return dst
