"""TEST INFRASTRUCTURE ONLY -- pins oracle/pwg_oracle.py to the LIVE reference (needs a checkout of the reference:
DSX_REFERENCE_ROOT) and writes tests/golden/pwg_plain.npz and pwg_pitch.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_pwg.py

The reference module is imported unmodified (stubs only for librosa / pycwt, scipy.signal.kaiser, which newer SciPy moved
to scipy.signal.windows, and np.int, which newer NumPy removed).  Weights are the constructor's random initialisation under a fixed seed, stored in weight-norm
form; inputs are seeded.  Both fixtures use the shipped widths and upsampling (hop 256, aux_context_window 2) at 4 layers,
so each stays under 1 MB: the plain path with 2 stacks, and the use_pitch_embed path with 1 stack and an edge-padded
coarse pitch (vocoders/pwg.py:91-97)."""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pwg_oracle as P  # noqa: E402

REF_ROOT = os.environ.get("DSX_REFERENCE_ROOT", "")


def load_reference():
    sys.dont_write_bytecode = True
    for n in ("librosa", "librosa.filters", "pycwt"):
        sys.modules.setdefault(n, types.ModuleType(n))
    import scipy.signal
    import scipy.signal.windows
    if not hasattr(scipy.signal, "kaiser"):
        scipy.signal.kaiser = scipy.signal.windows.kaiser
    if "int" not in np.__dict__:                     # f0_to_coarse's np.int, removed in NumPy 1.24
        np.int = int
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    from modules.parallel_wavegan.models.parallel_wavegan import ParallelWaveGANGenerator
    from utils.pitch_utils import f0_to_coarse
    return ParallelWaveGANGenerator, f0_to_coarse


CASES = {
    "pwg_plain.npz": dict(layers=4, stacks=2, use_pitch_embed=False, seed=0),
    "pwg_pitch.npz": dict(layers=4, stacks=1, use_pitch_embed=True, seed=1),
}


def config(layers, stacks, use_pitch_embed):
    return dict(P.CONFIG_SHIPPED, layers=layers, stacks=stacks, use_pitch_embed=use_pitch_embed,
                upsample_params={"upsample_scales": [4, 4, 4, 4]})


def write_case(name, layers, stacks, use_pitch_embed, seed, B=2, T=12):
    Gen, f0_to_coarse = load_reference()
    cfg = config(layers, stacks, use_pitch_embed)
    torch.manual_seed(seed)
    g = Gen(**{k: (dict(v) if isinstance(v, dict) else v) for k, v in cfg.items()}).eval()
    sd = {k: v.detach().clone() for k, v in g.state_dict().items()}
    w, hp = cfg["aux_context_window"], P.hop(cfg)
    gen = torch.Generator().manual_seed(seed + 10)
    z = torch.randn(B, 1, T * hp, generator=gen)
    mel = torch.randn(B, T, 80, generator=gen)
    c = torch.from_numpy(np.pad(mel.numpy(), ((0, 0), (w, w), (0, 0)), "edge")).transpose(1, 2)   # spec2wav's view
    pitch = None
    if use_pitch_embed:
        f0 = (torch.rand(B, T, generator=gen) * 300 + 80).numpy()
        f0[0, 3:6] = 0                                               # an unvoiced stretch
        coarse = np.stack([f0_to_coarse(f) for f in f0])
        pitch = torch.from_numpy(np.pad(coarse, ((0, 0), (w, w)), "edge")).long()
    with torch.no_grad():
        ref = g(z, c, pitch)
        ora = P.generator(sd, cfg, z, c, pitch)
    d = (ref - ora).abs().max().item()
    print(f"{name}: oracle vs live reference max |d| = {d:.3e}")
    assert torch.equal(ref, ora), "the oracle must be bit-exact against the reference"
    out = os.path.join(ROOT, "tests", "golden", name)
    extra = {"pitch": pitch.numpy()} if pitch is not None else {}
    np.savez_compressed(out, z=z.numpy(), c=c.contiguous().numpy(), wav=ref.numpy(), layers=np.int64(layers),
                        stacks=np.int64(stacks), use_pitch_embed=np.int64(use_pitch_embed), weight_seed=np.int64(seed),
                        **extra, **{"sd." + k: v.numpy() for k, v in sd.items()})
    print("wrote", out, os.path.getsize(out) // 1024, "KB")


def main():
    for name, kw in CASES.items():
        write_case(name, **kw)
    print("FLOPs per sample of the shipped generator:", P.flops_per_sample(P.CONFIG_SHIPPED))


if __name__ == "__main__":
    main()
