"""CPU: the FastSpeech2 encoder training step's host side -- its C symbols, the tape size formula of include/dsx.h, the
refused configurations, the dsx_train opt-in (hparams key and keyword) of both encoder classes, that training without
it or under no_grad still raises, the DsxError refusals of the opt-in path, and install_fs2_encoder's
duration_predictor keyword."""
import ctypes
import sys
import types

import pytest
import torch

from test_host_fs2dec_train import DSX_E_INVALID, _a256, documented_tape_bytes

HP = dict(hidden_size=256, enc_layers=4, dec_layers=4, enc_ffn_kernel_size=9, num_heads=2, ffn_padding='SAME',
          ffn_act='gelu', dropout=0.1, use_pos_embed=True, rel_pos=True)
VOCAB = 61
NAMES = ("dsx_fs2enc_train_create", "dsx_fs2enc_train_destroy", "dsx_fs2enc_train_tape_bytes",
         "dsx_fs2enc_train_workspace_bytes", "dsx_fs2enc_train_forward", "dsx_fs2enc_train_backward")


def test_symbols(lib_built):
    from diffsinger_b200 import _capi
    for n in NAMES:
        assert hasattr(_capi.lib, n) and n in _capi.SYMBOLS


def _config(H, L, heads, vocab, pos):
    from diffsinger_b200 import _capi
    from diffsinger_b200.fs2dec import _fs2dec_config
    return _capi.Fs2EncConfig(stack=_fs2dec_config(H, L, 9 if H != 64 else 1, heads, 'SAME', 'gelu'), vocab=vocab,
                              pos=pos)


@pytest.mark.parametrize("H,L,heads,B,T", [(256, 4, 2, 16, 250), (256, 4, 2, 1, 1), (192, 2, 3, 3, 37),
                                           (64, 3, 1, 64, 60)])
def test_tape_bytes_formula(lib_built, H, L, heads, B, T):
    from diffsinger_b200 import _capi
    if not torch.cuda.is_available():     # a handle belongs to a device; without one none can be made
        pytest.skip("dsx_fs2enc_train_create needs a CUDA device")
    h = ctypes.c_void_p()
    assert _capi.lib.dsx_fs2enc_train_create(0, ctypes.byref(_config(H, L, heads, VOCAB, 1)), ctypes.byref(h)) == 0
    n = ctypes.c_size_t()
    assert _capi.lib.dsx_fs2enc_train_tape_bytes(h, B, T, ctypes.byref(n)) == 0
    _capi.lib.dsx_fs2enc_train_destroy(h)
    assert n.value == documented_tape_bytes(H, L, heads, B, T) + _a256(8 * B * T)


@pytest.mark.parametrize("cfg", [(320, 4, 5, 61, 1), (256, 4, 3, 61, 1), (256, 65, 2, 61, 0), (256, 4, 2, 0, 0),
                                 (256, 4, 2, 61, 2)])
def test_refused_configurations(lib_built, cfg):
    from diffsinger_b200 import _capi
    H, L, heads, vocab, pos = cfg
    c = _capi.Fs2EncConfig(stack=_capi.Fs2DecConfig(hidden=H, layers=L, kernel=9, heads=heads, padding=0, act=0),
                           vocab=vocab, pos=pos)
    h = ctypes.c_void_p()
    assert _capi.lib.dsx_fs2enc_train_create(0, ctypes.byref(c), ctypes.byref(h)) == DSX_E_INVALID
    assert b"unsupported" in _capi.lib.dsx_last_error()


def _encoders(**kw):
    from diffsinger_b200 import FastspeechEncoder, FastspeechMIDIEncoder
    emb = torch.nn.Embedding(VOCAB, 256, 0)
    hp, hp_sin = dict(HP, **kw.pop("hp", {})), dict(HP, **dict(dict(rel_pos=False), **kw.pop("hp_sin", {})))
    return (FastspeechMIDIEncoder(emb, 256, 4, 9, hparams=hp, **kw),
            FastspeechEncoder(emb, 256, 4, 9, hparams=hp_sin, **kw))


def test_opt_in_routing(monkeypatch):
    from diffsinger_b200 import fs2enctrain
    calls = []
    monkeypatch.setattr(fs2enctrain, "fs2enc_train_forward", lambda enc, tok, adds: calls.append((enc, adds)) or tok)
    monkeypatch.setattr("diffsinger_b200.fs2enc._need_cuda", lambda *t: None)
    tok = torch.ones(1, 3, dtype=torch.long)
    add = torch.zeros(1, 3, 256)
    for midi, sin in (_encoders(hp=dict(dsx_train=True), hp_sin=dict(dsx_train=True)), _encoders(train=True)):
        assert midi._dsx_train and sin._dsx_train
        midi.train()(tok, add, 0, add)
        sin.train()(tok)
    assert len(calls) == 4
    assert calls[0][1][0] is add and calls[0][1][1] is None and calls[1][1] == [None, None, None]
    midi, sin = _encoders(hp=dict(dsx_train=True), hp_sin=dict(dsx_train=True), train=False)
    assert not midi._dsx_train and not sin._dsx_train


def test_training_without_opt_in_raises():
    from diffsinger_b200 import DsxError
    tok = torch.ones(1, 3, dtype=torch.long)
    midi, sin = _encoders()
    for m, args in ((midi, (tok, 0, 0, 0)), (sin, (tok,))):
        with pytest.raises(DsxError, match="eval mode only"):
            m.train()(*args)
    midi, sin = _encoders(train=True)
    for m, args in ((midi, (tok, 0, 0, 0)), (sin, (tok,))):
        with torch.no_grad(), pytest.raises(DsxError, match="eval mode only"):
            m.train()(*args)


def test_refusals():
    from diffsinger_b200 import DsxError
    midi, sin = _encoders(train=True)
    midi.train()
    tok = torch.ones(1, 3, dtype=torch.long)
    with pytest.raises(DsxError, match="CPU"):
        midi(tok, 0, 0, 0)
    rel_sin = _encoders(train=True, hp_sin=dict(rel_pos=True))[1].train()
    with pytest.raises(DsxError, match="rel_pos"):
        rel_sin(tok)
    if not torch.cuda.is_available():
        return
    dev = torch.device("cuda", 0)
    midi = midi.to(dev)
    with pytest.raises(DsxError, match=r"txt_tokens must be in \[0, 61\)"):
        midi(torch.full((1, 3), VOCAB, dtype=torch.long, device=dev), 0, 0, 0)
    half = torch.zeros(1, 3, 256, device=dev, dtype=torch.float16, requires_grad=True)
    with pytest.raises(DsxError, match="fp32 embedding addends"):
        midi(tok.to(dev), half, 0, 0)
    m2 = _encoders(train=True)[0].to(dev).train().double()
    with pytest.raises(DsxError, match="fp32"):
        m2(tok.to(dev), 0, 0, 0)
    m3 = _encoders(train=True)[0].to(dev).train()
    w = m3.layers[0].op.self_attn.in_proj_weight
    w.data = w.data.t().contiguous().t()
    with pytest.raises(DsxError, match="contiguous"):
        m3(tok.to(dev), 0, 0, 0)


def test_dropin_duration_predictor_keyword(monkeypatch):
    """install_fs2_encoder(duration_predictor=False) swaps the encoders and the length regulator but leaves the
    reference's DurationPredictor in place; uninstall restores every name it swapped"""
    import diffsinger_b200.dropin as dropin
    from diffsinger_b200 import fs2enc
    refs = {n: type(n, (), {}) for n in ("FastspeechEncoder", "FastspeechMIDIEncoder", "DurationPredictor",
                                         "LengthRegulator")}
    mods = {}
    for name in ("modules", "modules.fastspeech", "modules.fastspeech.fs2", "modules.diffsinger_midi",
                 "modules.diffsinger_midi.fs2"):
        mods[name] = types.ModuleType(name)
        monkeypatch.setitem(sys.modules, name, mods[name])
    for name in ("modules.fastspeech.fs2", "modules.diffsinger_midi.fs2"):
        for attr, cls in refs.items():
            setattr(mods[name], attr, cls)
    dropin.install_fs2_encoder(duration_predictor=False)
    try:
        for name in ("modules.fastspeech.fs2", "modules.diffsinger_midi.fs2"):
            assert mods[name].DurationPredictor is refs["DurationPredictor"]
            for attr in ("FastspeechEncoder", "FastspeechMIDIEncoder", "LengthRegulator"):
                assert getattr(mods[name], attr) is getattr(fs2enc, attr)
    finally:
        dropin.uninstall_fs2_encoder()
    for name in ("modules.fastspeech.fs2", "modules.diffsinger_midi.fs2"):
        for attr, cls in refs.items():
            assert getattr(mods[name], attr) is cls
    dropin.install_fs2_encoder()
    try:
        assert mods["modules.diffsinger_midi.fs2"].DurationPredictor is fs2enc.DurationPredictor
    finally:
        dropin.uninstall_fs2_encoder()
    assert mods["modules.diffsinger_midi.fs2"].DurationPredictor is refs["DurationPredictor"]
