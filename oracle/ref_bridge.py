"""TEST INFRASTRUCTURE ONLY -- imports the *live* reference from the checkout named by DSX_REFERENCE_ROOT.

Used by ``oracle/gen_golden.py`` to pin the oracle and write the fixtures under ``tests/golden``.  Recipe: stub ``librosa`` / ``pycwt``, ``set_hparams`` before importing ``usr.diff.shallow_diffusion_tts``
because ``max_beta`` binds at import time (usr/diff/shallow_diffusion_tts.py:44).
"""
import os
import sys
import types

REF_ROOT = os.environ.get("DSX_REFERENCE_ROOT", "")


def available():
    return bool(REF_ROOT) and os.path.isdir(os.path.join(REF_ROOT, "usr", "diff"))


_loaded = {}


def load(config="usr/configs/lj_ds_beta6.yaml", overrides=""):
    """Returns a namespace with the reference's hparams, DiffNet, GaussianDiffusion, module sdt.

    The reference keeps its configuration in a process-global dict and binds schedule
    defaults at import time, so one process can hold ONE configuration family; callers that
    need another ``max_beta`` pass explicit ``betas=`` to GaussianDiffusion instead.
    """
    key = (config, overrides)
    if _loaded:
        if key not in _loaded:
            ns = next(iter(_loaded.values()))
            return ns
        return _loaded[key]
    sys.dont_write_bytecode = True
    for n in ("librosa", "librosa.filters", "pycwt"):
        sys.modules.setdefault(n, types.ModuleType(n))
    sys.modules["pycwt"].wavelet = None
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    cwd = os.getcwd()
    os.chdir(REF_ROOT)          # configs use repo-relative base_config paths
    try:
        from utils.hparams import hparams, set_hparams
        set_hparams(config=config, exp_name="", hparams_str=overrides, print_hparams=False)
        from utils.text_encoder import TokenTextEncoder
        from usr.diff.net import DiffNet
        import usr.diff.shallow_diffusion_tts as sdt
    finally:
        os.chdir(cwd)
    ns = types.SimpleNamespace(hparams=hparams, DiffNet=DiffNet, sdt=sdt,
                               GaussianDiffusion=sdt.GaussianDiffusion,
                               TokenTextEncoder=TokenTextEncoder)
    _loaded[key] = ns
    return ns
