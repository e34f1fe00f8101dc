"""CPU: the DiffNet training step's host side -- its C symbols, the tape size formula, the dsx_train opt-in, that
training without the opt-in never reaches libdsx, and the DsxError refusals of the opt-in path."""
import ctypes

import pytest
import torch

HP = dict(hidden_size=256, residual_layers=3, residual_channels=256, dilation_cycle_length=2)
NAMES = ("dsx_train_create", "dsx_train_destroy", "dsx_train_tape_bytes", "dsx_train_workspace_bytes",
         "dsx_train_forward", "dsx_train_backward")


def test_symbols(lib_built):
    from diffsinger_b200 import _capi
    for n in NAMES:
        assert hasattr(_capi.lib, n) and n in _capi.SYMBOLS


def _a256(n):
    return (n + 255) // 256 * 256


def documented_tape_bytes(L, B, T):
    """include/dsx.h, dsx_train_tape_bytes."""
    F = B * T
    return (_a256(160 * F) + 4 * _a256(512 * F) + _a256(1024 * B) + _a256(9216 * B)
            + L * (2 * _a256(512 * F) + _a256(1024 * F)))


@pytest.mark.parametrize("L,B,T", [(20, 4, 1024), (1, 1, 1), (3, 3, 37), (20, 16, 1000)])
def test_tape_bytes_formula(lib_built, L, B, T):
    from diffsinger_b200 import _capi
    h = ctypes.c_void_p()
    cfg = _capi.TrainConfig(80, 256, 256, L, 4)
    if not torch.cuda.is_available():     # a handle belongs to a device; without one none can be made
        pytest.skip("dsx_train_create needs a CUDA device")
    assert _capi.lib.dsx_train_create(0, ctypes.byref(cfg), ctypes.byref(h)) == 0, _capi.lib.dsx_last_error()
    n = ctypes.c_size_t()
    assert _capi.lib.dsx_train_tape_bytes(h, B, T, ctypes.byref(n)) == 0
    _capi.lib.dsx_train_destroy(h)
    assert n.value == documented_tape_bytes(L, B, T)


@pytest.mark.parametrize("cfg", [(80, 128, 256, 20, 4), (80, 256, 192, 20, 4), (64, 256, 256, 20, 4),
                                 (80, 256, 256, 0, 4), (80, 256, 256, 20, 0)])
def test_create_refuses_other_shapes(lib_built, cfg):
    from diffsinger_b200 import _capi
    h = ctypes.c_void_p()
    assert _capi.lib.dsx_train_create(0, ctypes.byref(_capi.TrainConfig(*cfg)), ctypes.byref(h)) == -1
    assert b"unsupported" in _capi.lib.dsx_last_error()


def test_opt_in_from_hparams_and_keyword(lib_built):
    from diffsinger_b200 import DiffNet
    assert not DiffNet(80, hparams=HP)._dsx_train
    assert DiffNet(80, hparams=dict(HP, dsx_train=True))._dsx_train
    assert DiffNet(80, hparams=HP, train=True)._dsx_train
    assert not DiffNet(80, hparams=dict(HP, dsx_train=True), train=False)._dsx_train


def _inputs(B=2, T=16, C=256):
    return torch.randn(B, 1, 80, T), torch.randint(0, 100, (B,)), torch.randn(B, C, T)


def test_without_opt_in_training_never_calls_libdsx(lib_built, monkeypatch):
    from diffsinger_b200 import DiffNet, _capi

    class Raising:
        def __getattr__(self, name):
            raise AssertionError(f"libdsx called: {name}")

    monkeypatch.setattr(_capi, "lib", Raising())
    import diffsinger_b200.sampler as sampler
    import diffsinger_b200.modules as modules
    monkeypatch.setattr(sampler, "lib", Raising())
    torch.manual_seed(0)
    net = DiffNet(80, hparams=HP).train()
    spec, t, cond = _inputs()
    eps = net(spec, t, cond)
    ref = net._forward_autograd(spec, t, cond)
    assert torch.equal(eps, ref)
    eps.abs().mean().backward()
    assert all(p.grad is not None for p in net.parameters())
    assert modules.DiffNet is DiffNet


def test_refusals(lib_built):
    from diffsinger_b200 import DiffNet, DsxError
    spec, t, cond = _inputs()
    net = DiffNet(80, hparams=HP, train=True).train()
    with pytest.raises(DsxError, match="CUDA"):
        net(spec, t, cond)                                           # CPU tensors
    with pytest.raises(DsxError, match="spec"):
        net(spec.clone().requires_grad_(True), t, cond)              # spec.requires_grad
    with pytest.raises(DsxError, match="cond"):
        net(spec, t, torch.randn(2, 256, 15))                        # cond of another length
    with pytest.raises(DsxError, match="spec"):
        net(torch.randn(2, 1, 64, 16), t, cond)                      # 64 mel bins
    small = DiffNet(80, hparams=dict(HP, residual_channels=128), train=True).train()
    with pytest.raises(DsxError, match="residual_channels"):
        small(*_inputs())
    # eval and no_grad are unchanged by the opt-in: inference (CPU tensors raise there as before)
    with torch.no_grad():
        eps = DiffNet(80, hparams=HP, train=True).train()(spec, t, cond)
    assert eps.shape == (2, 1, 80, 16)
