"""CPU: the SSIM loss mirror (diffsinger_b200.ssim) refuses what the kernels do not implement with DsxError, the C ABI
exports its two entries, and dropin.install_ssim() / uninstall_ssim() rebind and restore the name on a stand-in tree."""
import pytest
import torch

from ssim_standin import drop_tree, install_tree


def img(*shape, dtype=torch.float32):
    return torch.rand(*shape, dtype=dtype)


REFUSALS = [
    ("window_size", lambda: (img(2, 1, 16, 80), img(2, 1, 16, 80)), dict(window_size=7), "window_size"),
    ("dim3", lambda: (img(2, 16, 80), img(2, 16, 80)), {}, "dim 3"),
    ("dim5", lambda: (img(2, 1, 1, 16, 80), img(2, 1, 1, 16, 80)), {}, "dim 5"),
    ("shape", lambda: (img(2, 1, 16, 80), img(2, 1, 17, 80)), {}, "differ in shape"),
    ("channels", lambda: (img(2, 3, 16, 80), img(2, 3, 16, 80)), {}, "one channel"),
    ("float64", lambda: (img(2, 1, 16, 80, dtype=torch.float64),) * 2, {}, "float32"),
    ("float16", lambda: (img(2, 1, 16, 80), img(2, 1, 16, 80, dtype=torch.float16)), {}, "float32"),
    ("width", lambda: (img(1, 1, 16, 257), img(1, 1, 16, 257)), {}, "W <= 256"),
    ("empty", lambda: (img(0, 1, 16, 80), img(0, 1, 16, 80)), {}, "B >= 1"),
    ("cpu", lambda: (img(2, 1, 16, 80), img(2, 1, 16, 80)), {}, "CPU"),
]


@pytest.mark.parametrize("what,make,kw,match", REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals(lib_built, what, make, kw, match):
    from diffsinger_b200 import DsxError, ssim
    with pytest.raises(DsxError, match=match):
        ssim(*make(), **kw)


def test_abi_symbols(lib_built):
    from diffsinger_b200 import _capi
    for name in ("dsx_ssim_forward", "dsx_ssim_backward"):
        assert name in _capi.SYMBOLS
        assert getattr(_capi.lib, name).restype is not None


def test_abi_rejects_bad_sizes(lib_built):
    """checked before any device access, so the refusals need no GPU"""
    from diffsinger_b200._capi import lib
    p = torch.zeros(1).data_ptr()
    for B, H, W in ((0, 8, 80), (1, 0, 80), (1, 8, 0), (1, 8, 257), (-1, 8, 80)):
        assert lib.dsx_ssim_forward(p, p, B, H, W, p, None) == -1
        assert b"W <= 256" in lib.dsx_last_error()
        assert lib.dsx_ssim_backward(p, p, p, B, H, W, p, p, None) == -1
    assert lib.dsx_ssim_forward(None, p, 1, 8, 80, p, None) == -1
    assert lib.dsx_ssim_forward(p, p, 1, 8, 80, None, None) == -1
    assert lib.dsx_ssim_backward(p, p, None, 1, 8, 80, p, p, None) == -1
    assert lib.dsx_ssim_backward(p, p, p, 1, 8, 80, None, None, None) == 0      # nothing asked for: no launch


def test_install_and_uninstall(lib_built, tmp_path, monkeypatch):
    install_tree(tmp_path, monkeypatch)
    import modules.commons.ssim as ref_mod
    import tasks.tts.fs2 as fs2
    import usr.aux_task as aux
    import diffsinger_b200
    import diffsinger_b200.dropin as dropin
    ref = ref_mod.ssim
    assert fs2.ssim is ref and aux.ssim is ref
    new = dropin.install_ssim()
    try:
        assert new is diffsinger_b200.ssim
        assert ref_mod.ssim is new and fs2.ssim is new and aux.ssim is new
        assert dropin.install_ssim() is new and fs2.ssim is new          # a second install changes nothing
        with pytest.raises(diffsinger_b200.DsxError, match="CPU"):      # the task's loss now reaches dsx
            fs2.MelLossTask().mel_loss(torch.rand(1, 12, 80), torch.rand(1, 12, 80))
    finally:
        dropin.uninstall_ssim()
    assert ref_mod.ssim is ref and fs2.ssim is ref and aux.ssim is ref
    drop_tree()
