"""CPU: the HiFi-GAN (NSF) oracle -- groundwork for the next scope row; no kernel yet -- against two cases computed by the
unmodified reference (oracle/gen_golden_hifigan.py, which asserts the oracle bit-exact against the reference when it writes
them)."""
import numpy as np
import torch

from conftest import golden
from oracle import hifigan_oracle as H


def _case(name="hifigan_nsf.npz"):
    g = golden(name)
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    h = dict(H.HPARAMS_TTS, upsample_initial_channel=int(g["upsample_initial_channel"]))
    return g, sd, h, torch.from_numpy(g["mel"]), torch.from_numpy(g["f0"])


def test_generator_matches_reference_fixture():
    g, sd, h, mel, f0 = _case()
    with torch.no_grad():
        torch.manual_seed(int(g["rng_seed"]))
        wav = H.generator(sd, h, mel, f0)
        plain = H.generator(sd, h, mel)
    assert wav.shape == (mel.shape[0], 1, mel.shape[2] * int(np.prod(h["upsample_rates"])))
    # same ATen kernels and RNG stream, but other host CPUs pick other conv kernels: a few ulps (3e-8 on a 0.1 signal)
    for out, ref in ((wav, g["wav_nsf"]), (plain, g["wav_plain"])):
        assert np.abs(out.numpy() - ref).max() <= 1e-6 * np.abs(ref).max()
    assert np.abs(g["wav_nsf"] - g["wav_plain"]).max() > 1e-4   # the harmonic source does reach the output


def test_weight_norm_and_plain_weights_agree():
    """after remove_weight_norm() a checkpoint carries plain `.weight` tensors: both forms give the same output"""
    g, sd, h, mel, f0 = _case()
    plain_sd = dict(sd)
    for k in list(sd):
        if k.endswith(".weight_g"):
            name = k[:-len(".weight_g")]
            plain_sd[name + ".weight"] = H.conv_weight(sd, name)
            del plain_sd[name + ".weight_g"], plain_sd[name + ".weight_v"]
    with torch.no_grad():
        a, b = H.generator(sd, h, mel), H.generator(plain_sd, h, mel)
    assert torch.equal(a, b)


def test_flops_per_frame_of_the_shipped_config():
    assert H.flops_per_frame(H.HPARAMS_TTS) == 38510592.0


def test_oracle_is_bit_exact_against_the_live_reference():
    """The reference's HifiGanGenerator on other weights (seed 3) and one utterance of 9 frames with the NSF source
    (tests/golden/hifigan_nsf_b1t9.npz): bit-exact where the fixture was written, a few ulps on other host CPUs."""
    g, sd, h, mel, f0 = _case("hifigan_nsf_b1t9.npz")
    with torch.no_grad():
        torch.manual_seed(int(g["rng_seed"]))
        b = H.generator(sd, h, mel, f0)
    assert b.shape == g["wav_nsf"].shape
    assert np.abs(b.numpy() - g["wav_nsf"]).max() <= 1e-6 * np.abs(g["wav_nsf"]).max()
