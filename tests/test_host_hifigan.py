"""CPU: the HiFi-GAN generator mirror (diffsinger_b200.HifiGanGenerator) has the reference's state-dict surface, loads
the reference fixtures strictly in both weight forms, and has no CPU path."""
import pytest
import torch

from conftest import golden
from oracle import hifigan_oracle as H

FIXTURES = ["hifigan_nsf.npz", "hifigan_nsf_b1t9.npz"]


def _fixture(name):
    g = golden(name)
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    h = dict(H.HPARAMS_TTS, upsample_initial_channel=int(g["upsample_initial_channel"]))
    return g, sd, h


def _plain(sd):
    out = dict(sd)
    for k in list(sd):
        if k.endswith(".weight_g"):
            name = k[:-len(".weight_g")]
            out[name + ".weight"] = H.conv_weight(sd, name)
            del out[name + ".weight_g"], out[name + ".weight_v"]
    return out


@pytest.mark.parametrize("name", FIXTURES)
def test_state_dict_surface_matches_the_reference(lib_built, name):
    from diffsinger_b200 import HifiGanGenerator
    _, sd, h = _fixture(name)
    m = HifiGanGenerator(h)
    mine = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert mine == {k: tuple(v.shape) for k, v in sd.items()}


@pytest.mark.parametrize("name", FIXTURES)
def test_strict_loading_in_both_weight_forms(lib_built, name):
    from diffsinger_b200 import HifiGanGenerator
    _, sd, h = _fixture(name)
    m = HifiGanGenerator(h)
    m.load_state_dict(sd, strict=True)
    m.remove_weight_norm()
    plain = _plain(sd)
    assert set(m.state_dict()) == set(plain)
    assert not any(k.endswith((".weight_g", ".weight_v")) for k in m.state_dict())
    m2 = HifiGanGenerator(h)
    m2.remove_weight_norm()
    m2.load_state_dict(plain, strict=True)
    for k, v in m.state_dict().items():
        assert torch.allclose(v, m2.state_dict()[k], rtol=1e-6, atol=1e-7), k


def test_cpu_forward_raises(lib_built):
    from diffsinger_b200 import DsxError, HifiGanGenerator
    g, sd, h = _fixture("hifigan_nsf_b1t9.npz")
    m = HifiGanGenerator(h)
    m.load_state_dict(sd, strict=True)
    with pytest.raises(DsxError):
        m(torch.from_numpy(g["mel"]), torch.from_numpy(g["f0"]))


def test_untransposed_mel_is_rejected(lib_built):
    """dsx_infer returns [B, T, 80]: handing it over without .transpose(1, 2) must fail before any device read"""
    from diffsinger_b200 import DsxError, HifiGanGenerator
    _, sd, h = _fixture("hifigan_nsf_b1t9.npz")
    m = HifiGanGenerator(h)
    m.load_state_dict(sd, strict=True)
    for shape in ((1, 9, 80), (1, 200, 80), (80, 9)):
        with pytest.raises(DsxError, match=r"\[B, 80, T\]"):
            m(torch.zeros(shape))
