"""TEST INFRASTRUCTURE ONLY -- pins oracle/pe_oracle.py to the LIVE reference pitch extractor (needs a checkout of the
reference: DSX_REFERENCE_ROOT) and writes tests/golden/pitch_extractor.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_pe.py

The reference's PitchExtractor (modules/fastspeech/pe.py) is imported unmodified (stubs only for librosa / pycwt) and
built under the e2e opencpop config (usr/configs/midi/e2e/opencpop/ds100_adj_rel.yaml) with hidden_size=32.  Its
convolution and linear weights are the constructor's initialisation under a fixed seed; the normalisation parameters,
pos_embed_alpha and the head bias are then overwritten with seeded values (oracle.pe_oracle.random_state_dict), so that
none of them is an identity.  Input: B = 2, T = 48 seeded mel frames, the second utterance with a zero-padded tail."""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pe_oracle as O  # noqa: E402

REF_ROOT = os.environ.get("DSX_REFERENCE_ROOT", "")
CONFIG = "usr/configs/midi/e2e/opencpop/ds100_adj_rel.yaml"
OVERRIDES = "hidden_size=32"
HP_KEYS = ("hidden_size", "predictor_hidden", "ffn_padding", "predictor_kernel", "pitch_type", "use_uv", "pitch_norm")


def load_reference():
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
        set_hparams(config=CONFIG, exp_name="", hparams_str=OVERRIDES, print_hparams=False)
        from modules.fastspeech.pe import PitchExtractor
    finally:
        os.chdir(cwd)
    return hparams, PitchExtractor


def main():
    assert REF_ROOT and os.path.isdir(REF_ROOT), "set DSX_REFERENCE_ROOT to a checkout of the reference"
    hparams, PitchExtractor = load_reference()
    hp = {k: hparams[k] for k in HP_KEYS}
    torch.manual_seed(0)
    pe = PitchExtractor().eval()
    sd = O.random_state_dict(pe.state_dict(), seed=1)
    pe.load_state_dict(sd, strict=True)
    B, T = 2, 48
    gen = torch.Generator().manual_seed(2)
    mel = torch.randn(B, T, 80, generator=gen) * 1.5 - 4.0
    mel[1, 37:] = 0                                   # a zero-padded tail: padding frames
    with torch.no_grad():
        ret = pe(mel)
        pitch, f0 = O.pitch_extractor(sd, mel, hp, conv_layers=2)
    d1 = (ret['pitch_pred'] - pitch).abs().max().item()
    d2 = (ret['f0_denorm_pred'] - f0).abs().max().item()
    print(f"oracle vs live reference: pitch_pred max |d| = {d1:.3e}, f0 max |d| = {d2:.3e}")
    assert d1 <= 1e-6 * ret['pitch_pred'].abs().max().item() and d2 <= 1e-6 * ret['f0_denorm_pred'].abs().max().item(), \
        "the oracle must reproduce the reference"
    uv = (ret['pitch_pred'][..., 1] > 0).float().mean().item()
    print(f"f0 range {f0[f0 > 0].min():.1f}..{f0.max():.1f} Hz, unvoiced share {uv:.2f}, "
          f"min |uv logit| {ret['pitch_pred'][..., 1].abs().min():.2e}")
    out = os.path.join(ROOT, "tests", "golden", "pitch_extractor.npz")
    np.savez_compressed(out, mel=mel.numpy(), pitch_pred=ret['pitch_pred'].numpy(), f0_denorm_pred=ret['f0_denorm_pred'].numpy(),
                        conv_layers=np.int64(2), weight_seed=np.int64(0),
                        **{"hp." + k: np.asarray(v) for k, v in hp.items()},
                        **{"sd." + k: v.numpy() for k, v in sd.items()})
    print("wrote", out, os.path.getsize(out) // 1024, "KB;", sum(v.numel() for v in sd.values()), "state-dict values")


if __name__ == "__main__":
    main()
