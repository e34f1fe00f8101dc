"""CPU: the Parallel WaveGAN oracle against the two cases the unmodified reference computed (oracle/gen_golden_pwg.py,
which asserts the oracle bit-exact against the reference when it writes them)."""
import numpy as np
import pytest
import torch

from oracle import pwg_oracle as P
from pwg_cases import FIXTURES, fixture, plain


def _run(name, **kw):
    g, sd, cfg = fixture(name)
    pitch = torch.from_numpy(g["pitch"]) if "pitch" in g.files else None
    with torch.no_grad():
        return g, P.generator(sd, cfg, torch.from_numpy(g["z"]), torch.from_numpy(g["c"]), pitch, **kw)


@pytest.mark.parametrize("name", FIXTURES)
def test_generator_matches_reference_fixture_bit_for_bit(name):
    g, wav = _run(name)
    assert wav.shape == g["wav"].shape
    assert np.array_equal(wav.numpy(), g["wav"])


def test_pitch_reaches_the_output_only_with_a_pitch_embedding():
    g, sd, cfg = fixture("pwg_pitch.npz")
    z, c, pitch = torch.from_numpy(g["z"]), torch.from_numpy(g["c"]), torch.from_numpy(g["pitch"])
    with torch.no_grad():
        assert not torch.equal(P.generator(sd, cfg, z, c, pitch), P.generator(sd, cfg, z, c, pitch.flip(1)))
        g0, sd0, cfg0 = fixture("pwg_plain.npz")
        z0, c0 = torch.from_numpy(g0["z"]), torch.from_numpy(g0["c"])
        assert torch.equal(P.generator(sd0, cfg0, z0, c0, pitch), P.generator(sd0, cfg0, z0, c0))


def test_weight_norm_and_plain_weights_agree():
    g, sd, cfg = fixture("pwg_plain.npz")
    z, c = torch.from_numpy(g["z"]), torch.from_numpy(g["c"])
    with torch.no_grad():
        assert torch.equal(P.generator(sd, cfg, z, c), P.generator(plain(sd), cfg, z, c))


def test_flops_per_sample_of_the_shipped_generator():
    """30 layers x 86,016 + the head 8,320 + first_conv 128 + conv_in and the four upsampling stages per sample"""
    assert P.flops_per_sample(P.CONFIG_SHIPPED) == 30 * 86016 + 8320 + 128 + (2 * 80 * 80 * 5 + 2 * 9 * 80 * 340) / 256


@pytest.mark.parametrize("name", FIXTURES)
def test_fp16_option(name):
    """fp16=False is the fp32 path bit for bit; fp16=True rounds (it differs), by about the 8e-4 / 1.4e-4 of the peak
    (max / mean) that test_gpu_pwg.py quotes for the fixtures"""
    g, a = _run(name)
    _, b = _run(name, fp16=False)
    _, s = _run(name, fp16=True)
    assert torch.equal(a, b)
    d, peak = (s - a).abs(), a.abs().max()
    assert 0 < d.max() <= 1e-3 * peak and d.mean() <= 1.6e-4 * peak, (d.max() / peak, d.mean() / peak)
