"""CPU: the pitch-extractor mirror (diffsinger_b200.PitchExtractor) has the reference's state-dict surface, loads the
reference fixture strictly, and refuses what it does not run (CPU tensors, training mode, a [B, 80, T] mel,
unsupported hparams) with DsxError."""
import pytest
import torch

from conftest import golden


def _fixture():
    g = golden("pitch_extractor.npz")
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    return g, sd, hp


def _model(hp, **kw):
    from diffsinger_b200 import PitchExtractor
    return PitchExtractor(80, kw.pop("conv_layers", 2), hparams=dict(hp, **kw))


def test_state_dict_surface_matches_the_reference(lib_built):
    _, sd, hp = _fixture()
    mine = {k: tuple(v.shape) for k, v in _model(hp).state_dict().items()}
    assert mine == {k: tuple(v.shape) for k, v in sd.items()}


def test_strict_loading(lib_built):
    _, sd, hp = _fixture()
    m = _model(hp)
    m.load_state_dict(sd, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_without_mel_encoder_the_surface_has_no_encoder(lib_built):
    _, _, hp = _fixture()
    assert not any(k.startswith("mel_encoder.") for k in _model(hp, conv_layers=0).state_dict())


def test_cpu_tensor_raises(lib_built):
    from diffsinger_b200 import DsxError
    g, sd, hp = _fixture()
    m = _model(hp)
    m.load_state_dict(sd, strict=True)
    with pytest.raises(DsxError, match="CPU"):
        m.eval()(torch.from_numpy(g["mel"]))


def test_training_mode_raises(lib_built):
    from diffsinger_b200 import DsxError
    g, sd, hp = _fixture()
    m = _model(hp)
    with pytest.raises(DsxError, match="eval"):
        m.train()(torch.from_numpy(g["mel"]))


def test_untransposed_mel_raises(lib_built):
    """the reference's PE takes [B, T, 80]; a vocoder-layout [B, 80, T] mel fails before any device read"""
    from diffsinger_b200 import DsxError
    _, _, hp = _fixture()
    m = _model(hp).eval()
    for shape in ((1, 80, 9), (2, 80, 200), (9, 80 + 1), (80,)):
        with pytest.raises(DsxError, match=r"\[B, T, 80\]"):
            m(torch.zeros(shape))


@pytest.mark.parametrize("bad", [dict(hidden_size=40), dict(hidden_size=384), dict(predictor_hidden=8),
                                 dict(predictor_kernel=4), dict(pitch_norm="none"), dict(conv_layers=17)])
def test_unsupported_config_raises(lib_built, bad):
    from diffsinger_b200 import DsxError
    _, _, hp = _fixture()
    with pytest.raises(DsxError, match="unsupported"):
        _model(hp, **bad)


def test_unsupported_mel_bins_raises(lib_built):
    from diffsinger_b200 import DsxError, PitchExtractor
    _, _, hp = _fixture()
    with pytest.raises(DsxError, match="n_mel_bins"):
        PitchExtractor(n_mel_bins=128, hparams=hp)
