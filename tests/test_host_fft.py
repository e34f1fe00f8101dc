"""CPU: the FFT-denoiser mirror (diffsinger_b200.FFT) has the reference's state-dict surface, loads the seeded reference
parameters strictly and refuses what it does not run (CPU tensors, training mode, unsupported hparams) with DsxError; the
sampler recognises an FFT module with the reference's layout and reads its configuration from the module."""
import ctypes

import pytest
import torch
import torch.nn as nn

from conftest import golden
from oracle import fft_oracle as O


def _fixture():
    g = golden("fft_denoiser.npz")
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    return g, hp, O.random_state_dict(int(g["seed"]), hp)


def _model(hp, **kw):
    from diffsinger_b200 import FFT
    return FFT(hparams=dict(hp, **kw))


def test_state_dict_surface_matches_the_reference(lib_built):
    _, hp, sd = _fixture()
    mine = {k: tuple(v.shape) for k, v in _model(hp).state_dict().items()}
    assert len(mine) == 54
    assert list(mine) == list(sd)
    assert mine == {k: tuple(v.shape) for k, v in sd.items()}


def test_strict_loading(lib_built):
    _, hp, sd = _fixture()
    m = _model(hp)
    m.load_state_dict(sd, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, sd[k]), k


def test_residual_channels_differ_from_hidden(lib_built):
    _, hp, _ = _fixture()
    sd = _model(hp, residual_channels=128).state_dict()
    assert sd["get_decode_inp.weight"].shape == (256, 256 + 2 * 128) and sd["input_projection.weight"].shape == (128, 80, 1)


def test_cpu_tensor_raises(lib_built):
    from diffsinger_b200 import DsxError
    g, hp, sd = _fixture()
    m = _model(hp)
    m.load_state_dict(sd, strict=True)
    with pytest.raises(DsxError, match="CPU"):
        m.eval()(torch.from_numpy(g["spec"]), torch.from_numpy(g["t"][0]), torch.from_numpy(g["cond"]))


def test_training_mode_raises(lib_built):
    from diffsinger_b200 import DsxError
    g, hp, _ = _fixture()
    with pytest.raises(DsxError, match="eval"):
        _model(hp).train()(torch.from_numpy(g["spec"]), torch.from_numpy(g["t"][0]), torch.from_numpy(g["cond"]))


@pytest.mark.parametrize("bad", [dict(residual_channels=24), dict(residual_channels=2048), dict(audio_num_mel_bins=128),
                                 dict(hidden_size=96), dict(num_heads=3), dict(ffn_act="swish"),
                                 dict(dec_ffn_kernel_size=8)])
def test_unsupported_config_raises(lib_built, bad):
    from diffsinger_b200 import DsxError
    _, hp, _ = _fixture()
    with pytest.raises(DsxError, match="unsupported"):
        _model(hp, **bad)


def test_c_abi_symbol_is_exported(lib_built):
    from diffsinger_b200 import _capi
    lib = ctypes.CDLL(_capi.LIB_PATH)
    assert hasattr(lib, "dsx_load_fft") and "dsx_load_fft" in _capi.SYMBOLS


# ---- the configuration of a module with the reference's layout ---------------------------------------------------------
class _FFN(nn.Module):          # common_layers.TransformerFFNLayer: kernel_size, act, ffn_1 (Conv1d or Sequential)
    def __init__(self, H, k, padding, act):
        super().__init__()
        self.kernel_size, self.act = k, act
        conv = nn.Conv1d(H, 4 * H, k, padding=k // 2 if padding == 'SAME' else 0)
        self.ffn_1 = conv if padding == 'SAME' else nn.Sequential(nn.ConstantPad1d((k - 1, 0), 0.0), conv)


class _Attn(nn.Module):
    def __init__(self, heads):
        super().__init__()
        self.num_heads = heads


class _Op(nn.Module):
    def __init__(self, H, heads, k, padding, act):
        super().__init__()
        self.self_attn, self.ffn = _Attn(heads), _FFN(H, k, padding, act)


class _Layer(nn.Module):
    def __init__(self, *a):
        super().__init__()
        self.op = _Op(*a)


class _RefLikeFFT(nn.Module):
    def __init__(self, H, L, heads, k, padding, act, dim):
        super().__init__()
        self.layers = nn.ModuleList([_Layer(H, heads, k, padding, act) for _ in range(L)])
        self.input_projection = nn.Conv1d(80, dim, 1)
        self.get_decode_inp = nn.Linear(H + 2 * dim, H)


@pytest.mark.parametrize("args", [(256, 4, 2, 9, 'SAME', 'gelu', 256), (128, 1, 1, 4, 'LEFT', 'relu', 64)])
def test_sampler_reads_the_configuration_of_a_reference_layout_module(lib_built, args):
    from diffsinger_b200.fftdiff import module_config
    H, L, heads, k, padding, act, dim = args
    net = _RefLikeFFT(*args)
    cfg, pad = module_config(net, net.state_dict())
    assert pad == padding
    assert (cfg.dec.hidden, cfg.dec.layers, cfg.dec.heads, cfg.dec.kernel) == (H, L, heads, k)
    assert (cfg.dec.padding, cfg.dec.act) == ({'SAME': 0, 'LEFT': 1}[padding], {'gelu': 0, 'relu': 1}[act])
    assert (cfg.residual_channels, cfg.mel_bins) == (dim, 80)


def test_mirror_module_reads_the_same_way(lib_built):
    from diffsinger_b200.fftdiff import module_config
    _, hp, _ = _fixture()
    m = _model(hp, ffn_padding='LEFT', dec_ffn_kernel_size=4, ffn_act='relu', residual_channels=128)
    cfg, pad = module_config(m, m.state_dict())
    assert pad == 'LEFT' and (cfg.dec.kernel, cfg.dec.act, cfg.residual_channels) == (4, 1, 128)
