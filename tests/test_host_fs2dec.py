"""CPU: the FastSpeech2-decoder mirror (diffsinger_b200.FastspeechDecoder) has the reference's state-dict surface, loads
the seeded reference parameters strictly, and refuses what it does not run (CPU tensors, training mode, a wrong last
dim, padding_mask / attn_mask / return_hiddens, unsupported hparams) with DsxError."""
import ctypes

import pytest
import torch

from conftest import golden
from oracle import fs2dec_oracle as O


def _fixture():
    g = golden("fs2_decoder.npz")
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    return g, hp, O.random_state_dict(int(g["seed"]), hp)


def _model(hp, **kw):
    from diffsinger_b200 import FastspeechDecoder
    return FastspeechDecoder(hparams=dict(hp, **kw))


def test_state_dict_surface_matches_the_reference(lib_built):
    _, hp, sd = _fixture()
    mine = {k: tuple(v.shape) for k, v in _model(hp).state_dict().items()}
    assert len(mine) == 44
    assert mine == {k: tuple(v.shape) for k, v in sd.items()}
    assert list(mine) == list(sd)


def test_left_padding_surface(lib_built):
    _, hp, _ = _fixture()
    hpl = dict(hp, ffn_padding='LEFT')
    mine = {k: tuple(v.shape) for k, v in _model(hpl).state_dict().items()}
    assert mine == {k: tuple(v) for k, v in O.state_dict_shapes(hpl).items()}
    assert "layers.0.op.ffn.ffn_1.1.weight" in mine


def test_strict_loading(lib_built):
    _, hp, sd = _fixture()
    m = _model(hp)
    m.load_state_dict(sd, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_constructor_arguments_override_hparams(lib_built):
    _, hp, _ = _fixture()
    from diffsinger_b200 import FastspeechDecoder
    m = FastspeechDecoder(128, 1, 3, 1, hparams=hp)
    assert (m.hidden_size, m.num_layers, m.kernel_size, m.num_heads) == (128, 1, 3, 1)
    assert m.state_dict()["layers.0.op.ffn.ffn_1.weight"].shape == (512, 128, 3)


def test_cpu_tensor_raises(lib_built):
    from diffsinger_b200 import DsxError
    g, hp, sd = _fixture()
    m = _model(hp)
    m.load_state_dict(sd, strict=True)
    with pytest.raises(DsxError, match="CPU"):
        m.eval()(torch.from_numpy(g["x"]))


def test_training_mode_raises(lib_built):
    from diffsinger_b200 import DsxError
    g, hp, _ = _fixture()
    with pytest.raises(DsxError, match="eval"):
        _model(hp).train()(torch.from_numpy(g["x"]))


def test_wrong_last_dim_raises(lib_built):
    from diffsinger_b200 import DsxError
    _, hp, _ = _fixture()
    m = _model(hp).eval()
    for shape in ((1, 9, 80), (2, 256, 9), (9, 256), (256,)):      # (2, 256, 9): a channels-first [B, H, T] input
        with pytest.raises(DsxError, match=r"\[B, T, 256\]"):
            m(torch.zeros(shape))


@pytest.mark.parametrize("kw", [dict(padding_mask=torch.zeros(1, 4, dtype=torch.bool)),
                                dict(attn_mask=torch.zeros(4, 4)), dict(return_hiddens=True)])
def test_unsupported_forward_arguments_raise(lib_built, kw):
    from diffsinger_b200 import DsxError
    _, hp, _ = _fixture()
    with pytest.raises(DsxError, match="not supported"):
        _model(hp).eval()(torch.zeros(1, 4, 256), **kw)


@pytest.mark.parametrize("bad", [dict(hidden_size=32), dict(hidden_size=96), dict(hidden_size=320),
                                 dict(num_heads=8), dict(num_heads=3), dict(ffn_act="swish"),
                                 dict(dec_ffn_kernel_size=8), dict(ffn_padding="CAUSAL"), dict(dec_layers=0)])
def test_unsupported_config_raises(lib_built, bad):
    from diffsinger_b200 import DsxError
    _, hp, _ = _fixture()
    with pytest.raises(DsxError, match="unsupported"):
        _model(hp, **bad)


def test_even_kernel_is_supported_with_left_padding(lib_built):
    _, hp, _ = _fixture()
    assert _model(hp, dec_ffn_kernel_size=8, ffn_padding="LEFT").kernel_size == 8


def test_c_abi_symbols_are_exported(lib_built):
    from diffsinger_b200 import _capi
    lib = ctypes.CDLL(_capi.LIB_PATH)
    for name in ("dsx_fs2dec_create", "dsx_fs2dec_destroy", "dsx_fs2dec_load", "dsx_fs2dec_forward"):
        assert hasattr(lib, name), name
        assert name in _capi.SYMBOLS
