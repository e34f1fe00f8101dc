"""Drop-in installation inside the reference tree.

    import diffsinger_b200.dropin as dropin; dropin.install()      # after utils.hparams.set_hparams(...)

replaces, without editing any reference file,
  * ``usr.diff.shallow_diffusion_tts.GaussianDiffusion`` (built by usr/diffspeech_task.py:25, usr/diffsinger_task.py:40),
  * ``usr.diff.shallow_diffusion_tts.OfflineGaussianDiffusion`` (usr/diffsinger_task.py:128) and
  * ``usr.diff.diffusion.GaussianDiffusion`` (the older full-T sampler, usr/task.py:18)
-- and the names bound from them in ``usr.*`` / ``tasks.*`` / ``inference.*`` modules already imported -- by subclasses
whose ``forward(infer=True)`` runs the sm_90a sampler, and the ``'wavenet'`` entry of every ``DIFF_DECODERS`` registry by
``diffsinger_b200.DiffNet``.  Construction arguments, parameter / buffer names, ``p_losses`` and the returned ``ret`` dict
are the reference's own, so the task files run unchanged.
"""
import importlib
import sys

import torch

from .modules import DiffNet, DsxInferMixin

_installed = {}


def _dsx_kwargs(kwargs):
    return {k: kwargs.pop(k) for k in list(kwargs) if k.startswith('dsx_')}


def make_subclass(ref_cls):
    """usr.diff.shallow_diffusion_tts.GaussianDiffusion with the infer branch (:248-275) routed to dsx."""

    class DsxGaussianDiffusion(DsxInferMixin, ref_cls):
        def forward(self, txt_tokens, mel2ph=None, spk_embed=None, ref_mels=None, f0=None, uv=None, energy=None,
                    infer=False, **kwargs):
            if not infer:
                return ref_cls.forward(self, txt_tokens, mel2ph, spk_embed, ref_mels, f0, uv, energy, infer, **kwargs)
            dsx_kw = _dsx_kwargs(kwargs)
            # same call as usr/diff/shallow_diffusion_tts.py:236-238
            ret = self.fs2(txt_tokens, mel2ph, spk_embed, ref_mels, f0, uv, energy, skip_decoder=False, infer=True,
                           **kwargs)
            cond = ret['decoder_inp'].transpose(1, 2)
            with torch.no_grad():
                return self.dsx_infer(ret, cond, mel2ph, step_noise=dsx_kw.get('dsx_step_noise'),
                                      start_noise=dsx_kw.get('dsx_start_noise'), seed=dsx_kw.get('dsx_seed'))

    DsxGaussianDiffusion.__name__ = ref_cls.__name__
    DsxGaussianDiffusion.__qualname__ = ref_cls.__qualname__
    return DsxGaussianDiffusion


def make_offline_subclass(ref_cls):
    """OfflineGaussianDiffusion (:291-323): the shallow start comes from the mel handed in as ref_mels[1]; plain DDPM;
    no mel2ph mask and no ret['fs2_mel']."""

    class DsxOfflineGaussianDiffusion(DsxInferMixin, ref_cls):
        def forward(self, txt_tokens, mel2ph=None, spk_embed=None, ref_mels=None, f0=None, uv=None, energy=None,
                    infer=False, **kwargs):
            if not infer:
                return ref_cls.forward(self, txt_tokens, mel2ph, spk_embed, ref_mels, f0, uv, energy, infer, **kwargs)
            dsx_kw = _dsx_kwargs(kwargs)
            ret = self.fs2(txt_tokens, mel2ph, spk_embed, ref_mels, f0, uv, energy, skip_decoder=True, infer=True, **kwargs)
            cond = ret['decoder_inp'].transpose(1, 2)
            with torch.no_grad():
                return self.dsx_infer(ret, cond, None, fs2_mel=ref_mels[1], keep_fs2_mel=False, allow_pndm=False,
                                      step_noise=dsx_kw.get('dsx_step_noise'), start_noise=dsx_kw.get('dsx_start_noise'),
                                      seed=dsx_kw.get('dsx_seed'))

    DsxOfflineGaussianDiffusion.__name__ = ref_cls.__name__
    DsxOfflineGaussianDiffusion.__qualname__ = ref_cls.__qualname__
    return DsxOfflineGaussianDiffusion


def make_old_subclass(ref_cls):
    """usr.diff.diffusion.GaussianDiffusion (:297-320): gaussian start, num_timesteps DDPM steps, denorm, no mask."""

    class DsxOldGaussianDiffusion(DsxInferMixin, ref_cls):
        def forward(self, txt_tokens, mel2ph=None, spk_embed=None, ref_mels=None, f0=None, uv=None, energy=None,
                    infer=False, **kwargs):
            if not infer:
                return ref_cls.forward(self, txt_tokens, mel2ph, spk_embed, ref_mels, f0, uv, energy, infer)
            dsx_kw = _dsx_kwargs(kwargs)
            ret = self.fs2(txt_tokens, mel2ph, spk_embed, ref_mels, f0, uv, energy, skip_decoder=True, infer=infer)
            cond = ret['decoder_inp'].transpose(1, 2)
            with torch.no_grad():
                x_start = dsx_kw.get('dsx_x_start')
                if x_start is None:
                    x_start = torch.randn((cond.shape[0], 1, self.mel_bins, cond.shape[2]), device=cond.device)
                return self.dsx_infer(ret, cond, None, x_start=x_start, K_step=self.num_timesteps, keep_fs2_mel=False,
                                      allow_pndm=False, step_noise=dsx_kw.get('dsx_step_noise'), seed=dsx_kw.get('dsx_seed'))

    DsxOldGaussianDiffusion.__name__ = ref_cls.__name__
    DsxOldGaussianDiffusion.__qualname__ = ref_cls.__qualname__
    return DsxOldGaussianDiffusion


def install():
    sdt = importlib.import_module("usr.diff.shallow_diffusion_tts")
    old = importlib.import_module("usr.diff.diffusion")
    if not _installed:
        _installed.update(ref_cls=sdt.GaussianDiffusion, ref_off=getattr(sdt, "OfflineGaussianDiffusion", None),
                          ref_old=old.GaussianDiffusion)
        _installed.update(new_cls=make_subclass(_installed["ref_cls"]),
                          new_off=make_offline_subclass(_installed["ref_off"]) if _installed["ref_off"] else None,
                          new_old=make_old_subclass(_installed["ref_old"]))
    sdt.GaussianDiffusion = _installed["new_cls"]
    if _installed["new_off"] is not None:
        sdt.OfflineGaussianDiffusion = _installed["new_off"]
    old.GaussianDiffusion = _installed["new_old"]
    net_mod = importlib.import_module("usr.diff.net")
    _installed.setdefault("ref_net", net_mod.DiffNet)
    net_mod.DiffNet = DiffNet
    wavenet = lambda hp: DiffNet(hp['audio_num_mel_bins'])
    swap = {id(_installed[r]): _installed[n] for r, n in (("ref_cls", "new_cls"), ("ref_off", "new_off"), ("ref_old", "new_old"))
            if _installed[r] is not None}
    for name, mod in list(sys.modules.items()):
        if mod is None or not (name.startswith("usr.") or name.startswith("inference.") or name.startswith("tasks.")):
            continue
        for attr in ("GaussianDiffusion", "OfflineGaussianDiffusion"):
            cur = getattr(mod, attr, None)
            if cur is not None and id(cur) in swap:
                setattr(mod, attr, swap[id(cur)])
        reg = getattr(mod, "DIFF_DECODERS", None)
        if isinstance(reg, dict) and "wavenet" in reg:
            reg["wavenet"] = wavenet
    return _installed["new_cls"]


def uninstall():
    if not _installed:
        return
    back = {id(_installed[n]): _installed[r] for r, n in (("ref_cls", "new_cls"), ("ref_off", "new_off"), ("ref_old", "new_old"))
            if _installed[n] is not None}
    importlib.import_module("usr.diff.net").DiffNet = _installed["ref_net"]
    for name, mod in list(sys.modules.items()):
        if mod is None:
            continue
        for attr in ("GaussianDiffusion", "OfflineGaussianDiffusion"):
            cur = getattr(mod, attr, None)
            if cur is not None and id(cur) in back:
                setattr(mod, attr, back[id(cur)])
