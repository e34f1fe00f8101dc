"""CPU: the pitch and energy predictors' host side -- the C symbols and argtypes, the parameter names against the
reference's module, the tape size formula of include/dsx.h, the refused configurations, the dsx_train opt-in (hparams key
and keyword) and that training without it raises, pickling without the trainer, and that
install_fs2_predictors() / uninstall_fs2_predictors() touch only the two FastSpeech2 modules."""
import copy
import ctypes
import pickle
import sys
import types

import pytest
import torch

from test_host_fs2dec_train import DSX_E_INVALID, _a256

HP = dict(dsx_train=False)
NAMES = ("dsx_pitchpred_create", "dsx_pitchpred_destroy", "dsx_pitchpred_load", "dsx_pitchpred_forward",
         "dsx_pitchpred_train_create", "dsx_pitchpred_train_destroy", "dsx_pitchpred_train_tape_bytes",
         "dsx_pitchpred_train_workspace_bytes", "dsx_pitchpred_train_forward", "dsx_pitchpred_train_backward",
         "dsx_pitchpred_train_masks")


def documented_tape_bytes(idim, P, L, B, T):
    """include/dsx.h: a256(24) + a256(4 F) + a256(2 F idim) + L a256(4 F P) + (L - 1) a256(2 F P) + a256(4 F P)"""
    F = B * T
    return (_a256(24) + _a256(4 * F) + _a256(2 * F * idim) + L * _a256(4 * F * P) + (L - 1) * _a256(2 * F * P) +
            _a256(4 * F * P))


def test_symbols_and_argtypes(lib_built):
    from diffsinger_b200 import _capi
    for n in NAMES:
        assert hasattr(_capi.lib, n) and n in _capi.SYMBOLS
    lib = _capi.lib
    assert lib.dsx_pitchpred_destroy.restype is None and lib.dsx_pitchpred_train_destroy.restype is None
    assert lib.dsx_pitchpred_create.argtypes[1]._type_ is _capi.PitchPredConfig
    assert lib.dsx_pitchpred_train_create.argtypes[1]._type_ is _capi.PitchPredConfig
    assert lib.dsx_pitchpred_load.argtypes[1]._type_ is _capi.PitchPredParams
    assert len(lib.dsx_pitchpred_forward.argtypes) == 6
    assert len(lib.dsx_pitchpred_train_forward.argtypes) == 13
    assert lib.dsx_pitchpred_train_forward.argtypes[5] is ctypes.c_float
    assert lib.dsx_pitchpred_train_forward.argtypes[6] is ctypes.c_uint64
    assert len(lib.dsx_pitchpred_train_backward.argtypes) == 11
    assert lib.dsx_pitchpred_train_backward.argtypes[4]._type_ is _capi.PitchPredParams
    assert len(lib.dsx_pitchpred_train_masks.argtypes) == 7
    assert [f for f, _ in _capi.PitchPredParams._fields_][-1] == "pos_embed_alpha"


@pytest.mark.parametrize("cfg", [(256, 5, 256, 2, 5, 'SAME'), (256, 2, 256, 1, 5, 'SAME'), (128, 2, 256, 11, 5, 'SAME')])
def test_state_dict_matches_the_reference(cfg):
    """The state dict has the names and shapes of gen_golden_pitchpred_train.random_state_dict, which the generator loads
    strictly into the reference's own PitchPredictor (frame, ph and CWT configurations), and loads it strictly too"""
    from diffsinger_b200 import EnergyPredictor, PitchPredictor
    from diffsinger_b200.pitchpred import param_names
    from oracle.gen_golden_pitchpred_train import random_state_dict
    idim, L, C, od, k, pad = cfg
    for cls in (PitchPredictor, EnergyPredictor):
        m = cls(idim, n_layers=L, n_chans=C, odim=od, kernel_size=k, dropout_rate=0.5, padding=pad, hparams=HP)
        ref = random_state_dict(0, idim, L, C, od, k)
        assert {n: tuple(v.shape) for n, v in m.state_dict().items()} == {n: tuple(v.shape) for n, v in ref.items()}
        assert sorted(param_names(L)) == sorted(n for n, _ in m.named_parameters())
        m.load_state_dict(ref, strict=True)


@pytest.mark.parametrize("idim,P,L,B,T", [(256, 256, 5, 16, 1000), (256, 256, 2, 1, 1), (128, 256, 2, 3, 37),
                                          (16, 48, 16, 64, 60)])
def test_tape_bytes_formula(lib_built, idim, P, L, B, T):
    from diffsinger_b200 import _capi
    if not torch.cuda.is_available():     # a handle belongs to a device; without one none can be made
        pytest.skip("dsx_pitchpred_train_create needs a CUDA device")
    h = ctypes.c_void_p()
    c = _capi.PitchPredConfig(idim=idim, chans=P, layers=L, kernel=5, padding=0, odim=2)
    assert _capi.lib.dsx_pitchpred_train_create(0, ctypes.byref(c), ctypes.byref(h)) == 0
    n = ctypes.c_size_t()
    assert _capi.lib.dsx_pitchpred_train_tape_bytes(h, B, T, ctypes.byref(n)) == 0
    _capi.lib.dsx_pitchpred_train_destroy(h)
    assert n.value == documented_tape_bytes(idim, P, L, B, T)


@pytest.mark.parametrize("cfg", [(8, 256, 5, 5, 0, 2), (256, 272, 5, 5, 0, 2), (256, 24, 5, 5, 0, 2),
                                 (256, 256, 0, 5, 0, 2), (256, 256, 17, 5, 0, 2), (256, 256, 5, 4, 0, 2),
                                 (256, 256, 5, 33, 1, 2), (256, 256, 5, 5, 2, 2), (256, 256, 5, 5, 0, 0),
                                 (256, 256, 5, 5, 0, 17)])
def test_refused_configurations(lib_built, cfg):
    from diffsinger_b200 import DsxError, PitchPredictor, _capi
    idim, P, L, k, pad, od = cfg
    c = _capi.PitchPredConfig(idim=idim, chans=P, layers=L, kernel=k, padding=pad, odim=od)
    for create in (_capi.lib.dsx_pitchpred_create, _capi.lib.dsx_pitchpred_train_create):
        h = ctypes.c_void_p()
        assert create(0, ctypes.byref(c), ctypes.byref(h)) == DSX_E_INVALID
        assert b"unsupported" in _capi.lib.dsx_last_error()
    with pytest.raises(DsxError, match="unsupported PitchPredictor configuration"):
        PitchPredictor(idim, L, P, od, k, 0.5, {0: 'SAME', 1: 'LEFT'}.get(pad, 'CAUSAL'), hparams=HP)


def _pp(cls=None, **kw):
    from diffsinger_b200 import PitchPredictor
    hp = dict(HP, **kw.pop("hp", {}))
    return (cls or PitchPredictor)(256, 5, 256, 2, 5, 0.5, 'SAME', hparams=hp, **kw)


def test_opt_in_routing(monkeypatch):
    from diffsinger_b200 import EnergyPredictor, pitchpred
    calls = []
    monkeypatch.setattr(pitchpred, "pitchpred_train_forward", lambda pp, xs: calls.append((pp, xs)) or xs[..., :2])
    monkeypatch.setattr(pitchpred, "_need_cuda", lambda *t: None)
    xs = torch.zeros(2, 3, 256)
    for pp in (_pp(hp=dict(dsx_train=True)), _pp(train=True), _pp(EnergyPredictor, train=True)):
        assert pp._dsx_train and pp.dropout_rate == 0.5
        assert pp.train()(xs).shape == (2, 3, 2)
    assert len(calls) == 3 and calls[0][1] is xs
    assert not _pp(hp=dict(dsx_train=True), train=False)._dsx_train


def test_training_without_opt_in_raises():
    from diffsinger_b200 import DsxError
    xs = torch.zeros(1, 3, 256)
    with pytest.raises(DsxError, match="eval mode only"):
        _pp().train()(xs)
    pp = _pp(train=True).train()
    with torch.no_grad(), pytest.raises(DsxError, match="eval mode only"):
        pp(xs)


def test_refusals():
    from diffsinger_b200 import DsxError
    pp = _pp(train=True).train()
    with pytest.raises(DsxError, match="CPU"):
        pp(torch.zeros(1, 3, 256))
    with pytest.raises(DsxError, match=r"xs must be \[B, T, 256\]"):
        pp(torch.zeros(1, 3, 128))
    with pytest.raises(DsxError, match="CPU"):
        _pp().eval()(torch.zeros(1, 3, 256))


def test_copies_drop_the_trainer():
    pp = _pp(train=True)
    pp._dsx_train_step()
    assert pp._dsx_trainer is not None
    for c in (copy.deepcopy(pp), pickle.loads(pickle.dumps(pp))):
        assert c._dsx_trainer is None and c._dsx_train
    _pp().load_state_dict(pp.state_dict(), strict=True)


def test_install_touches_only_the_fastspeech2_modules(monkeypatch):
    """install_fs2_predictors() rebinds PitchPredictor / EnergyPredictor where the two FastSpeech2 modules have them, and
    nowhere else: tts_modules and the pitch extractor's module keep the reference's classes"""
    import diffsinger_b200.dropin as dropin
    from diffsinger_b200 import pitchpred
    mods = {}
    for name in ("modules", "modules.fastspeech", "modules.fastspeech.fs2", "modules.fastspeech.tts_modules",
                 "modules.fastspeech.pe", "modules.diffsinger_midi", "modules.diffsinger_midi.fs2"):
        mods[name] = types.ModuleType(name)
        monkeypatch.setitem(sys.modules, name, mods[name])
    RefP = type("PitchPredictor", (), {})
    RefE = type("EnergyPredictor", (RefP,), {})
    for name in ("modules.fastspeech.fs2", "modules.fastspeech.tts_modules", "modules.diffsinger_midi.fs2"):
        mods[name].PitchPredictor, mods[name].EnergyPredictor = RefP, RefE
    mods["modules.fastspeech.pe"].PitchPredictor = RefP
    del mods["modules.diffsinger_midi.fs2"].EnergyPredictor      # a module without the name keeps not having it
    dropin.install_fs2_predictors()
    try:
        assert mods["modules.fastspeech.fs2"].PitchPredictor is pitchpred.PitchPredictor
        assert mods["modules.fastspeech.fs2"].EnergyPredictor is pitchpred.EnergyPredictor
        assert mods["modules.diffsinger_midi.fs2"].PitchPredictor is pitchpred.PitchPredictor
        assert not hasattr(mods["modules.diffsinger_midi.fs2"], "EnergyPredictor")
        assert mods["modules.fastspeech.tts_modules"].PitchPredictor is RefP
        assert mods["modules.fastspeech.tts_modules"].EnergyPredictor is RefE
        assert mods["modules.fastspeech.pe"].PitchPredictor is RefP
    finally:
        dropin.uninstall_fs2_predictors()
    assert mods["modules.fastspeech.fs2"].PitchPredictor is RefP and mods["modules.fastspeech.fs2"].EnergyPredictor is RefE
    assert mods["modules.diffsinger_midi.fs2"].PitchPredictor is RefP
