"""TEST INFRASTRUCTURE ONLY -- pins oracle/ssim_oracle.py to the LIVE reference (needs a checkout of the reference:
DSX_REFERENCE_ROOT) and writes tests/golden/ssim.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_ssim.py

modules/commons/ssim.py imports with torch and numpy only, so it is imported unmodified.  The task's losses
(tasks/tts/fs2.py:158-175) need the whole task stack, so ssim_oracle.ssim_loss restates them and runs here with the
reference's ssim.  Two cases, seeded, in fp32 on the CPU:
  mel  2 x 40 x 80, bias 6: a mel-like target whose second utterance is zero-padded from frame 28, and a decoder output
       near it (nonzero on the padding, as a model's is); the map, ssim(size_average=True), the weighted loss and its
       gradient with respect to decoder_output
  cwt  2 x 30 x 10, bias 20 (cwt_loss): the same quantities for a CWT-spectrogram-like pair"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ssim_oracle as O  # noqa: E402

REF_ROOT = os.environ.get("DSX_REFERENCE_ROOT", "")


def load_reference():
    sys.dont_write_bytecode = True
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    from modules.commons import ssim as S
    return S


def mel_like(gen, B, T, n, lo, hi):
    """smooth in time and frequency, in [lo, hi]"""
    z = torch.randn(B, 1, T + 8, n + 8, generator=gen)
    z = torch.nn.functional.avg_pool2d(z, 9, stride=1)[:, 0]
    z = (z - z.amin()) / (z.amax() - z.amin())
    return lo + (hi - lo) * z


def case(S, gen, B, T, n, lo, hi, bias, pad_from):
    target = mel_like(gen, B, T, n, lo, hi)
    if pad_from is not None:
        target[1, pad_from:] = 0
    out = (target + 0.3 * torch.randn(B, T, n, generator=gen)).requires_grad_(True)
    x, y = out.detach()[:, None] + bias, target[:, None] + bias
    ref_map = S.ssim(x, y, size_average=False)
    ref_mean = S.ssim(x, y)
    ref_loss = O.ssim_loss(out, target, bias, ssim_fn=S.ssim)
    ref_loss.backward()
    o = out.detach().clone().requires_grad_(True)
    ora_loss = O.ssim_loss(o, target, bias)
    ora_loss.backward()
    assert torch.equal(O.ssim(x, y, size_average=False), ref_map), "oracle map must be bit-exact against the reference"
    assert torch.equal(O.ssim(x, y), ref_mean)
    assert torch.equal(ora_loss, ref_loss) and torch.equal(o.grad, out.grad)
    print(f"{B}x{T}x{n} bias {bias}: ssim {ref_mean.item():.6f}, loss {ref_loss.item():.6f} (oracle bit-exact)")
    return dict(decoder_output=out.detach().numpy(), target=target.numpy(), bias=np.float32(bias),
                map=ref_map.numpy(), mean=ref_mean.detach().numpy(), loss=ref_loss.detach().numpy(),
                d_decoder_output=out.grad.numpy())


def main():
    S = load_reference()
    assert torch.equal(S.gaussian(11, 1.5), O.gaussian()) and torch.equal(S.create_window(11, 1), O.window())
    gen = torch.Generator().manual_seed(0)
    mel = case(S, gen, 2, 40, 80, -5.5, 1.5, 6.0, 28)
    cwt = case(S, gen, 2, 30, 10, -3.0, 3.0, 20.0, None)
    out = os.path.join(ROOT, "tests", "golden", "ssim.npz")
    np.savez_compressed(out, window=O.gaussian().numpy(), **{f"mel.{k}": v for k, v in mel.items()},
                        **{f"cwt.{k}": v for k, v in cwt.items()})
    print("wrote", out, os.path.getsize(out) // 1024, "KB")


if __name__ == "__main__":
    main()
