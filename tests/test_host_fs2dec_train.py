"""CPU: the FastSpeech2 decoder training step's host side -- its C symbols, the tape size formula of include/dsx.h, the
refused configurations, the dsx_train opt-in (hparams key and keyword), that training without it still raises, and the
DsxError refusals of the opt-in path."""
import ctypes

import pytest
import torch

HP = dict(hidden_size=256, dec_layers=4, dec_ffn_kernel_size=9, num_heads=2, ffn_padding='SAME', ffn_act='gelu',
          dropout=0.1)
DSX_E_INVALID = -1   # include/dsx.h
NAMES = ("dsx_fs2dec_train_create", "dsx_fs2dec_train_destroy", "dsx_fs2dec_train_tape_bytes",
         "dsx_fs2dec_train_workspace_bytes", "dsx_fs2dec_train_forward", "dsx_fs2dec_train_backward",
         "dsx_fs2dec_train_masks")


def test_symbols(lib_built):
    from diffsinger_b200 import _capi
    for n in NAMES:
        assert hasattr(_capi.lib, n) and n in _capi.SYMBOLS


def _a256(n):
    return (n + 255) // 256 * 256


def documented_tape_bytes(H, L, heads, B, T):
    """include/dsx.h, dsx_fs2dec_train_tape_bytes."""
    F = B * T
    return (_a256(24) + _a256(F) + _a256(4 * F) + (2 * L + 1) * _a256(4 * F * H)
            + L * (6 * _a256(2 * F * H) + _a256(4 * F * heads) + 2 * _a256(8 * F * H)))


def _handle(cfg):
    from diffsinger_b200 import _capi
    if not torch.cuda.is_available():     # a handle belongs to a device; without one none can be made
        pytest.skip("dsx_fs2dec_train_create needs a CUDA device")
    h = ctypes.c_void_p()
    assert _capi.lib.dsx_fs2dec_train_create(0, ctypes.byref(cfg), ctypes.byref(h)) == 0, _capi.lib.dsx_last_error()
    return h


@pytest.mark.parametrize("H,L,heads,B,T", [(256, 4, 2, 32, 1000), (256, 4, 2, 1, 1), (192, 2, 3, 3, 37),
                                           (64, 3, 1, 4, 4500)])
def test_tape_bytes_formula(lib_built, H, L, heads, B, T):
    from diffsinger_b200 import _capi
    from diffsinger_b200.fs2dec import _fs2dec_config
    h = _handle(_fs2dec_config(H, L, 9 if H != 64 else 1, heads, 'SAME', 'gelu'))
    n = ctypes.c_size_t()
    assert _capi.lib.dsx_fs2dec_train_tape_bytes(h, B, T, ctypes.byref(n)) == 0
    _capi.lib.dsx_fs2dec_train_destroy(h)
    assert n.value == documented_tape_bytes(H, L, heads, B, T)


@pytest.mark.parametrize("cfg", [(320, 4, 5, 9, 0, 0), (256, 4, 3, 9, 0, 0), (256, 4, 2, 8, 0, 0),
                                 (256, 65, 2, 9, 0, 0), (256, 4, 2, 9, 2, 0), (256, 4, 2, 9, 0, 2)])
def test_refused_configurations(lib_built, cfg):
    from diffsinger_b200 import _capi
    c = _capi.Fs2DecConfig()
    c.hidden, c.layers, c.heads, c.kernel, c.padding, c.act = cfg
    h = ctypes.c_void_p()
    assert _capi.lib.dsx_fs2dec_train_create(0, ctypes.byref(c), ctypes.byref(h)) == DSX_E_INVALID
    assert b"unsupported" in _capi.lib.dsx_last_error()


def test_opt_in_routing(monkeypatch):
    from diffsinger_b200 import FastspeechDecoder, fs2train
    calls = []
    monkeypatch.setattr(fs2train, "fs2dec_train_forward", lambda dec, x: calls.append(dec) or x)
    x = torch.ones(1, 3, 256)
    for m in (FastspeechDecoder(hparams=dict(HP, dsx_train=True)), FastspeechDecoder(hparams=HP, train=True)):
        assert m._dsx_train
        m.train()(x)
    assert len(calls) == 2
    m = FastspeechDecoder(hparams=dict(HP, dsx_train=True), train=False)
    assert not m._dsx_train


def test_training_without_opt_in_raises():
    from diffsinger_b200 import DsxError, FastspeechDecoder
    m = FastspeechDecoder(hparams=HP).train()
    with pytest.raises(DsxError, match="eval mode only"):
        m(torch.ones(1, 3, 256))
    m = FastspeechDecoder(hparams=dict(HP, dsx_train=True)).train()
    with torch.no_grad(), pytest.raises(DsxError, match="eval mode only"):
        m(torch.ones(1, 3, 256))


def test_refusals():
    from diffsinger_b200 import DsxError, FastspeechDecoder
    m = FastspeechDecoder(hparams=dict(HP, dsx_train=True)).train()
    x = torch.ones(1, 3, 256)
    with pytest.raises(DsxError, match="CPU"):
        m(x)
    with pytest.raises(DsxError, match="padding_mask"):
        m(x, padding_mask=torch.zeros(1, 3, dtype=torch.bool))
    with pytest.raises(DsxError, match="padding_mask"):
        m(x, return_hiddens=True)
    if torch.cuda.is_available():
        m2 = FastspeechDecoder(hparams=dict(HP, dsx_train=True)).cuda().train().double()
        with pytest.raises(DsxError, match="fp32"):
            m2(x.cuda())
