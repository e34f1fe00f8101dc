"""CPU: the duration predictor training step's host side -- its C symbols and argtypes, the tape size formula of
include/dsx.h, the refused configurations, the dsx_train opt-in (hparams key and keyword), that training without it,
under no_grad or through .inference() still raises, the DsxError refusals of the opt-in path, pickling without the
trainer, and the drop-in under dsx_train."""
import copy
import ctypes
import pickle
import sys
import types

import pytest
import torch

from test_host_fs2dec_train import DSX_E_INVALID, _a256

HP = dict(dur_loss='mse', dsx_train=False)
NAMES = ("dsx_durpred_train_create", "dsx_durpred_train_destroy", "dsx_durpred_train_tape_bytes",
         "dsx_durpred_train_workspace_bytes", "dsx_durpred_train_forward", "dsx_durpred_train_backward",
         "dsx_durpred_train_masks")


def documented_tape_bytes(idim, P, L, B, T):
    """include/dsx.h: a256(24) + a256(F) + a256(2 F idim) + L a256(4 F P) + (L - 1) a256(2 F P) + a256(4 F P)"""
    F = B * T
    return (_a256(24) + _a256(F) + _a256(2 * F * idim) + L * _a256(4 * F * P) + (L - 1) * _a256(2 * F * P) +
            _a256(4 * F * P))


def test_symbols_and_argtypes(lib_built):
    from diffsinger_b200 import _capi
    for n in NAMES:
        assert hasattr(_capi.lib, n) and n in _capi.SYMBOLS
    lib = _capi.lib
    assert lib.dsx_durpred_train_destroy.restype is None
    assert lib.dsx_durpred_train_create.argtypes[1]._type_ is _capi.DurPredConfig
    assert len(lib.dsx_durpred_train_forward.argtypes) == 15
    assert lib.dsx_durpred_train_forward.argtypes[7] is ctypes.c_float
    assert lib.dsx_durpred_train_forward.argtypes[8] is ctypes.c_uint64
    assert len(lib.dsx_durpred_train_backward.argtypes) == 11
    assert lib.dsx_durpred_train_backward.argtypes[4]._type_ is _capi.DurPredParams
    assert len(lib.dsx_durpred_train_masks.argtypes) == 7


def test_param_names_match_the_module():
    from diffsinger_b200 import DurationPredictor
    from diffsinger_b200.durtrain import param_names
    dp = DurationPredictor(256, 5, 256, 3, 0.5, hparams=HP)
    assert sorted(param_names(5)) == sorted(n for n, _ in dp.named_parameters())


@pytest.mark.parametrize("idim,P,L,B,T", [(256, 256, 5, 16, 250), (256, 256, 2, 1, 1), (48, 16, 1, 3, 37),
                                          (16, 256, 16, 64, 60)])
def test_tape_bytes_formula(lib_built, idim, P, L, B, T):
    from diffsinger_b200 import _capi
    if not torch.cuda.is_available():     # a handle belongs to a device; without one none can be made
        pytest.skip("dsx_durpred_train_create needs a CUDA device")
    h = ctypes.c_void_p()
    c = _capi.DurPredConfig(idim=idim, chans=P, layers=L, kernel=3, padding=0, offset=1.0)
    assert _capi.lib.dsx_durpred_train_create(0, ctypes.byref(c), ctypes.byref(h)) == 0
    n = ctypes.c_size_t()
    assert _capi.lib.dsx_durpred_train_tape_bytes(h, B, T, ctypes.byref(n)) == 0
    _capi.lib.dsx_durpred_train_destroy(h)
    assert n.value == documented_tape_bytes(idim, P, L, B, T)


@pytest.mark.parametrize("cfg", [(8, 256, 5, 3, 0), (256, 272, 5, 3, 0), (256, 24, 5, 3, 0), (256, 256, 0, 3, 0),
                                 (256, 256, 17, 3, 0), (256, 256, 5, 4, 0), (256, 256, 5, 33, 1),
                                 (256, 256, 5, 0, 1), (256, 256, 5, 3, 2), (256, 256, 5, 3, float("inf"))])
def test_refused_configurations(lib_built, cfg):
    from diffsinger_b200 import _capi
    idim, P, L, k, pad = cfg
    c = _capi.DurPredConfig(idim=idim, chans=P, layers=L, kernel=k, padding=pad if pad in (0, 1, 2) else 0,
                            offset=1.0 if pad in (0, 1, 2) else pad)
    h = ctypes.c_void_p()
    assert _capi.lib.dsx_durpred_train_create(0, ctypes.byref(c), ctypes.byref(h)) == DSX_E_INVALID
    assert b"unsupported" in _capi.lib.dsx_last_error()


def _dp(**kw):
    from diffsinger_b200 import DurationPredictor
    hp = dict(HP, **kw.pop("hp", {}))
    return DurationPredictor(256, 5, 256, 3, 0.5, hparams=hp, **kw)


def test_opt_in_routing(monkeypatch):
    from diffsinger_b200 import durtrain
    calls = []
    monkeypatch.setattr(durtrain, "durpred_train_forward", lambda dp, xs, m: calls.append((dp, xs, m)) or xs[..., 0])
    monkeypatch.setattr("diffsinger_b200.fs2enc._need_cuda", lambda *t: None)
    xs, mask = torch.zeros(2, 3, 256), torch.zeros(2, 3, dtype=torch.bool)
    for dp in (_dp(hp=dict(dsx_train=True)), _dp(train=True)):
        assert dp._dsx_train and dp.dropout_rate == 0.5
        assert dp.train()(xs, mask).shape == (2, 3)
    assert len(calls) == 2 and calls[0][1] is xs and calls[0][2] is mask
    assert not _dp(hp=dict(dsx_train=True), train=False)._dsx_train


def test_training_without_opt_in_raises():
    from diffsinger_b200 import DsxError
    xs, mask = torch.zeros(1, 3, 256), torch.zeros(1, 3, dtype=torch.bool)
    with pytest.raises(DsxError, match="eval mode only"):
        _dp().train()(xs, mask)
    dp = _dp(train=True).train()
    with torch.no_grad(), pytest.raises(DsxError, match="eval mode only"):
        dp(xs, mask)
    with pytest.raises(DsxError, match="eval mode only"):
        dp.inference(xs, mask)


def test_refusals():
    from diffsinger_b200 import DsxError
    dp = _dp(train=True).train()
    xs = torch.zeros(1, 3, 256)
    with pytest.raises(DsxError, match="CPU"):
        dp(xs, torch.zeros(1, 3, dtype=torch.bool))
    with pytest.raises(DsxError, match="x_masks"):
        dp(xs)
    with pytest.raises(DsxError, match="x_masks"):
        dp(xs, torch.zeros(1, 4, dtype=torch.bool))
    with pytest.raises(DsxError, match=r"xs must be \[B, T, 256\]"):
        dp(torch.zeros(1, 3, 128), torch.zeros(1, 3, dtype=torch.bool))


def test_copies_drop_the_trainer():
    dp = _dp(train=True)
    dp._dsx_train_step()
    assert dp._dsx_trainer is not None
    for c in (copy.deepcopy(dp), pickle.loads(pickle.dumps(dp))):
        assert c._dsx_trainer is None and c._dsx_train
    assert set(dp.state_dict()) == set(_dp().state_dict())
    _dp().load_state_dict(dp.state_dict(), strict=True)


def test_dropin_trains_the_dsx_predictor_under_dsx_train(monkeypatch):
    """install_fs2_encoder() binds the dsx DurationPredictor where FastSpeech2.__init__ looks it up; under dsx_train the
    predictor it builds opts in to its training step, and training mode routes to it"""
    import diffsinger_b200.dropin as dropin
    from diffsinger_b200 import durtrain, fs2enc
    mods = {}
    for name in ("modules", "modules.fastspeech", "modules.fastspeech.fs2", "modules.diffsinger_midi",
                 "modules.diffsinger_midi.fs2"):
        mods[name] = types.ModuleType(name)
        monkeypatch.setitem(sys.modules, name, mods[name])
    for name in ("modules.fastspeech.fs2", "modules.diffsinger_midi.fs2"):
        mods[name].DurationPredictor = type("DurationPredictor", (), {})
    calls = []
    monkeypatch.setattr(durtrain, "durpred_train_forward", lambda dp, xs, m: calls.append(dp) or xs[..., 0])
    monkeypatch.setattr("diffsinger_b200.fs2enc._need_cuda", lambda *t: None)
    dropin.install_fs2_encoder()
    try:
        cls = mods["modules.diffsinger_midi.fs2"].DurationPredictor
        assert cls is fs2enc.DurationPredictor
        # fs2.py:45-50, with the global hparams of a dsx_train run
        dp = cls(256, n_chans=256, n_layers=5, dropout_rate=0.5, padding='SAME', kernel_size=3,
                 hparams=dict(HP, dsx_train=True))
        dur_input = torch.zeros(2, 4, 256, requires_grad=True)
        dp.train()(dur_input.detach() + 0.1 * (dur_input - dur_input.detach()), torch.zeros(2, 4, dtype=torch.bool))
        assert calls == [dp]
    finally:
        dropin.uninstall_fs2_encoder()
