"""Drop-in installation inside the reference tree.

    import diffsinger_b200.dropin as dropin; dropin.install()      # after utils.hparams.set_hparams(...)

replaces, without editing any reference file,
  * ``usr.diff.shallow_diffusion_tts.GaussianDiffusion`` (built by usr/diffspeech_task.py:25, usr/diffsinger_task.py:40),
  * ``usr.diff.shallow_diffusion_tts.OfflineGaussianDiffusion`` (usr/diffsinger_task.py:128) and
  * ``usr.diff.diffusion.GaussianDiffusion`` (the older full-T sampler, usr/task.py:18)
-- and the names bound from them in ``usr.*`` / ``tasks.*`` / ``inference.*`` modules already imported -- by subclasses
whose ``forward(infer=True)`` runs the sm_90a sampler, and the ``'wavenet'`` entry of every ``DIFF_DECODERS`` registry by
``diffsinger_b200.DiffNet``.  Construction arguments, parameter / buffer names, ``p_losses`` and the returned ``ret`` dict
are the reference's own, so the task files run unchanged.  With ``diff_decoder_type: 'fft'`` the reference's own ``FFT``
(usr/diff/candidate_decoder.py) stays the ``denoise_fn``: ``DsxSampler`` recognises it and runs its evaluations on dsx
(``dsx_load_fft``).  Only when hparams set ``dsx_train`` does the ``'fft'`` entry of every ``DIFF_DECODERS`` registry
build ``diffsinger_b200.FFT`` instead, so that training (``p_losses``) runs the sm_90a training step; ``uninstall()``
restores the entry.

    dropin.install_vocoder()

replaces ``modules.hifigan.hifigan.HifiGanGenerator`` -- and the name bound from it in ``vocoders.*`` modules already
imported -- by ``diffsinger_b200.HifiGanGenerator``, so ``vocoders/hifigan.py:load_model`` (strict ``load_state_dict``,
``remove_weight_norm``, ``.to(device)``) and ``spec2wav`` run the vocoder on dsx unchanged.

    dropin.install_pwg()

replaces ``ParallelWaveGANGenerator`` in ``modules.parallel_wavegan.models`` and
``modules.parallel_wavegan.models.parallel_wavegan`` -- and the name bound from them in ``vocoders.*`` modules already
imported (vocoders/pwg.py binds it at import) -- by ``diffsinger_b200.ParallelWaveGANGenerator``, so
``vocoders/pwg.py:load_pwg_model`` (``load_state_dict``, ``remove_weight_norm``, ``.eval().to(device)``) and ``spec2wav``
run the PWG vocoder on dsx unchanged.  ``uninstall_pwg()`` restores the reference's class.

    dropin.install_pitch_extractor()

replaces ``modules.fastspeech.pe.PitchExtractor`` -- and the name bound from it in ``inference.*`` / ``tasks.*`` /
``usr.*`` modules already imported (inference/svs/ds_e2e.py binds it at import) -- by ``diffsinger_b200.PitchExtractor``,
so the e2e inference's ``self.pe(mel_out)['f0_denorm_pred']`` runs on dsx after a strict ``load_ckpt``.

    dropin.install_fs2_decoder()      # before the model is built

rebinds ``FastspeechDecoder`` in ``modules.fastspeech.fs2`` and ``modules.diffsinger_midi.fs2`` to
``diffsinger_b200.FastspeechDecoder``.  Their ``FS_DECODERS['fft']`` looks the name up when it is called, so the next
``FastSpeech2`` / ``FastSpeech2MIDI`` gets the dsx decoder; ``mel_out`` stays the reference's ``nn.Linear``.
``modules.fastspeech.tts_modules`` keeps the reference's class, so subclasses of it (usr/diff/candidate_decoder.py) are
untouched.

    dropin.install_fs2_encoder()      # before the model is built

rebinds ``FastspeechEncoder``, ``FastspeechMIDIEncoder``, ``DurationPredictor`` and ``LengthRegulator`` in
``modules.fastspeech.fs2`` and ``modules.diffsinger_midi.fs2`` (where the module defines or imports the name) to the
classes of ``diffsinger_b200.fs2enc``.  ``FS_ENCODERS['fft']`` looks the encoder up when it is called and
``FastSpeech2.__init__`` the other two, so the next ``FastSpeech2`` / ``FastSpeech2MIDI`` runs its encoder, duration
predictor and length regulator on dsx; ``FastSpeech2.forward`` itself (the MIDI embeddings, the ``decoder_inp`` gather)
stays the reference's.  ``modules.fastspeech.tts_modules`` keeps the reference's classes.  Under ``dsx_train`` the
encoders and the duration predictor run their sm_90a training steps; ``FastSpeech2.add_dur``'s ``predictor_grad``
scaling of the predictor's input stays in the reference's graph.  ``install_fs2_encoder(duration_predictor=False)``
leaves the reference's ``DurationPredictor`` in place, so it trains in eager PyTorch.  ``uninstall_fs2_encoder()``
restores whatever was swapped.

    dropin.install_fs2_predictors()   # before the model is built

rebinds ``PitchPredictor`` and ``EnergyPredictor`` in ``modules.fastspeech.fs2`` and ``modules.diffsinger_midi.fs2``
(where the module has the name) to the classes of ``diffsinger_b200.pitchpred``, so the next ``FastSpeech2`` /
``FastSpeech2MIDI`` builds its pitch predictor -- the one inside ``cwt_predictor``'s ``Sequential(Linear,
PitchPredictor)`` included, whose ``Linear`` stays eager -- and its energy predictor on dsx.  Under ``dsx_train`` they run
their sm_90a training steps.  ``modules.fastspeech.tts_modules`` and ``modules.fastspeech.pe`` keep the reference's
classes, so the reference's ``PitchExtractor`` keeps its own predictor.  ``uninstall_fs2_predictors()`` restores
whatever was swapped.

    dropin.install_ssim()

rebinds ``ssim`` in ``modules.commons.ssim`` -- and the name bound from it in ``tasks.*`` / ``usr.*`` modules already
imported (tasks/tts/fs2.py binds it at import) -- to ``diffsinger_b200.ssim``, so ``FastSpeech2Task.ssim_loss`` and
``cwt_loss`` run the SSIM loss, forward and backward, on dsx unchanged.  The ``l1`` half of ``mel_loss``, the
nonzero-speech weights and the reference's ``SSIM`` module class stay eager.  ``uninstall_ssim()`` restores the
reference's function.
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
        if isinstance(reg, dict) and "fft" in reg and name not in _fft_entries:
            _fft_entries[name] = ref_fft = reg["fft"]
            reg["fft"] = _fft_builder(ref_fft)
    return _installed["new_cls"]


_fft_entries = {}   # module name -> the DIFF_DECODERS['fft'] entry install() replaced


def _fft_builder(ref_fft):
    """DIFF_DECODERS['fft']: diffsinger_b200.FFT under dsx_train, else the reference's entry (its own FFT)."""
    def build(hp):
        if not hp.get('dsx_train', False):
            return ref_fft(hp)
        from .fftdiff import FFT
        return FFT(hp['hidden_size'], hp['dec_layers'], hp['dec_ffn_kernel_size'], hp['num_heads'], hparams=hp)
    return build


def uninstall():
    if not _installed:
        return
    back = {id(_installed[n]): _installed[r] for r, n in (("ref_cls", "new_cls"), ("ref_off", "new_off"), ("ref_old", "new_old"))
            if _installed[n] is not None}
    importlib.import_module("usr.diff.net").DiffNet = _installed["ref_net"]
    for name, ref_fft in list(_fft_entries.items()):
        reg = getattr(sys.modules.get(name), "DIFF_DECODERS", None)
        if isinstance(reg, dict):
            reg["fft"] = ref_fft
        del _fft_entries[name]
    for name, mod in list(sys.modules.items()):
        if mod is None:
            continue
        for attr in ("GaussianDiffusion", "OfflineGaussianDiffusion"):
            cur = getattr(mod, attr, None)
            if cur is not None and id(cur) in back:
                setattr(mod, attr, back[id(cur)])


_vocoder = {}


def install_vocoder():
    from .vocoder import HifiGanGenerator
    mod = importlib.import_module("modules.hifigan.hifigan")
    _vocoder.setdefault("ref", mod.HifiGanGenerator)
    _swap_vocoder(_vocoder["ref"], HifiGanGenerator)
    return HifiGanGenerator


def uninstall_vocoder():
    if _vocoder:
        from .vocoder import HifiGanGenerator
        _swap_vocoder(HifiGanGenerator, _vocoder["ref"])


def _swap_vocoder(old, new):
    for name, mod in list(sys.modules.items()):
        if mod is None or not (name == "modules.hifigan.hifigan" or name.startswith("vocoders.")):
            continue
        if getattr(mod, "HifiGanGenerator", None) is old:
            mod.HifiGanGenerator = new


_pwg = {}
_PWG_MODULES = ("modules.parallel_wavegan.models", "modules.parallel_wavegan.models.parallel_wavegan")


def install_pwg():
    from .pwg import ParallelWaveGANGenerator
    mod = importlib.import_module("modules.parallel_wavegan.models.parallel_wavegan")
    if mod.ParallelWaveGANGenerator is not ParallelWaveGANGenerator:
        _pwg["ref"] = mod.ParallelWaveGANGenerator
    _swap_pwg(_pwg["ref"], ParallelWaveGANGenerator)
    return ParallelWaveGANGenerator


def uninstall_pwg():
    if _pwg:
        from .pwg import ParallelWaveGANGenerator
        _swap_pwg(ParallelWaveGANGenerator, _pwg["ref"])


def _swap_pwg(old, new):
    for name, mod in list(sys.modules.items()):
        if mod is None or not (name in _PWG_MODULES or name.startswith("vocoders.")):
            continue
        if getattr(mod, "ParallelWaveGANGenerator", None) is old:
            mod.ParallelWaveGANGenerator = new


_pe = {}


def install_pitch_extractor():
    from .pitch import PitchExtractor
    mod = importlib.import_module("modules.fastspeech.pe")
    _pe.setdefault("ref", mod.PitchExtractor)
    _swap_pitch_extractor(_pe["ref"], PitchExtractor)
    return PitchExtractor


def uninstall_pitch_extractor():
    if _pe:
        from .pitch import PitchExtractor
        _swap_pitch_extractor(PitchExtractor, _pe["ref"])


def _swap_pitch_extractor(old, new):
    for name, mod in list(sys.modules.items()):
        if mod is None or not (name == "modules.fastspeech.pe" or name.startswith(("inference.", "tasks.", "usr."))):
            continue
        if getattr(mod, "PitchExtractor", None) is old:
            mod.PitchExtractor = new


_fs2 = {}
_FS2_MODULES = ("modules.fastspeech.fs2", "modules.diffsinger_midi.fs2")


def install_fs2_decoder():
    from .fs2dec import FastspeechDecoder
    for name in _FS2_MODULES:
        try:
            mod = importlib.import_module(name)
        except ModuleNotFoundError as e:
            if e.name is None or not name.startswith(e.name):      # a missing dependency, not a missing module
                raise
            continue
        cur = mod.FastspeechDecoder
        _fs2.setdefault(name, cur)
        mod.FastspeechDecoder = FastspeechDecoder
    return FastspeechDecoder


def uninstall_fs2_decoder():
    for name, ref in list(_fs2.items()):
        mod = sys.modules.get(name)
        if mod is not None:
            mod.FastspeechDecoder = ref
        del _fs2[name]


_fs2enc = {}
_FS2ENC_NAMES = ("FastspeechEncoder", "FastspeechMIDIEncoder", "DurationPredictor", "LengthRegulator")


def install_fs2_encoder(duration_predictor=True):
    from . import fs2enc
    names = _FS2ENC_NAMES if duration_predictor else tuple(n for n in _FS2ENC_NAMES if n != "DurationPredictor")
    for name in _FS2_MODULES:
        try:
            mod = importlib.import_module(name)
        except ModuleNotFoundError as e:
            if e.name is None or not name.startswith(e.name):      # a missing dependency, not a missing module
                raise
            continue
        for attr in names:
            if not hasattr(mod, attr):
                continue
            _fs2enc.setdefault((name, attr), getattr(mod, attr))
            setattr(mod, attr, getattr(fs2enc, attr))
    return fs2enc.FastspeechMIDIEncoder


def uninstall_fs2_encoder():
    for (name, attr), ref in list(_fs2enc.items()):
        mod = sys.modules.get(name)
        if mod is not None:
            setattr(mod, attr, ref)
        del _fs2enc[(name, attr)]


_fs2pred = {}
_FS2PRED_NAMES = ("PitchPredictor", "EnergyPredictor")


def install_fs2_predictors():
    from . import pitchpred
    for name in _FS2_MODULES:
        try:
            mod = importlib.import_module(name)
        except ModuleNotFoundError as e:
            if e.name is None or not name.startswith(e.name):      # a missing dependency, not a missing module
                raise
            continue
        for attr in _FS2PRED_NAMES:
            if not hasattr(mod, attr):
                continue
            _fs2pred.setdefault((name, attr), getattr(mod, attr))
            setattr(mod, attr, getattr(pitchpred, attr))
    return pitchpred.PitchPredictor


def uninstall_fs2_predictors():
    for (name, attr), ref in list(_fs2pred.items()):
        mod = sys.modules.get(name)
        if mod is not None:
            setattr(mod, attr, ref)
        del _fs2pred[(name, attr)]


_ssim = {}


def install_ssim():
    from .ssim import ssim
    mod = importlib.import_module("modules.commons.ssim")
    if mod.ssim is not ssim:
        _ssim["ref"] = mod.ssim
    _swap_ssim(_ssim["ref"], ssim)
    return ssim


def uninstall_ssim():
    if _ssim:
        from .ssim import ssim
        _swap_ssim(ssim, _ssim["ref"])


def _swap_ssim(old, new):
    for name, mod in list(sys.modules.items()):
        if mod is None or not (name == "modules.commons.ssim" or name.startswith(("tasks.", "usr."))):
            continue
        if getattr(mod, "ssim", None) is old:
            mod.ssim = new
