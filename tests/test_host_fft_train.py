"""CPU: the FFT denoiser training step's host side -- its C symbols, the tape size formula of include/dsx.h, the refused
configurations, the dsx_train opt-in (hparams key and keyword) and its loud failure without a GPU, that training without
it still raises, and the drop-in's rebinding of DIFF_DECODERS['fft'] on a stand-in reference tree."""
import ctypes
import sys

import pytest
import torch

HP = dict(hidden_size=256, dec_layers=4, dec_ffn_kernel_size=9, num_heads=2, ffn_padding='SAME', ffn_act='gelu',
          dropout=0.1, residual_channels=256, audio_num_mel_bins=80)
DSX_E_INVALID = -1   # include/dsx.h
NAMES = ("dsx_fft_train_create", "dsx_fft_train_destroy", "dsx_fft_train_tape_bytes", "dsx_fft_train_workspace_bytes",
         "dsx_fft_train_forward", "dsx_fft_train_backward")


def test_symbols(lib_built):
    from diffsinger_b200 import _capi
    for n in NAMES:
        assert hasattr(_capi.lib, n) and n in _capi.SYMBOLS
        assert n == "dsx_fft_train_destroy" or getattr(_capi.lib, n).argtypes


def _a256(n):
    return (n + 255) // 256 * 256


def documented_tape_bytes(H, L, heads, dim, B, T):
    """include/dsx.h, dsx_fft_train_tape_bytes (D: dsx_fs2dec_train_tape_bytes)."""
    F = B * T
    D = (_a256(24) + _a256(F) + _a256(4 * F) + (2 * L + 1) * _a256(4 * F * H)
         + L * (6 * _a256(2 * F * H) + _a256(4 * F * heads) + 2 * _a256(8 * F * H)))
    return D + _a256(4 * B * dim) + _a256(36 * B * dim) + _a256(480 * F) + _a256(6 * F * H) + _a256(2 * F * H)


def _config(H, L, heads, dim, k=9, padding='SAME', act='gelu', mel=80):
    from diffsinger_b200 import _capi
    from diffsinger_b200.fs2dec import _fs2dec_config
    c = _capi.FftConfig()
    c.dec, c.residual_channels, c.mel_bins = _fs2dec_config(H, L, k, heads, padding, act), dim, mel
    return c


@pytest.mark.parametrize("H,L,heads,dim,B,T", [(256, 4, 2, 256, 32, 1000), (256, 4, 2, 256, 1, 1),
                                               (192, 2, 3, 16, 3, 37), (64, 1, 1, 1024, 4, 4500)])
def test_tape_bytes_formula(lib_built, H, L, heads, dim, B, T):
    from diffsinger_b200 import _capi
    if not torch.cuda.is_available():     # a handle belongs to a device; without one none can be made
        pytest.skip("dsx_fft_train_create needs a CUDA device")
    h = ctypes.c_void_p()
    cfg = _config(H, L, heads, dim)
    assert _capi.lib.dsx_fft_train_create(0, ctypes.byref(cfg), ctypes.byref(h)) == 0, _capi.lib.dsx_last_error()
    n = ctypes.c_size_t()
    assert _capi.lib.dsx_fft_train_tape_bytes(h, B, T, ctypes.byref(n)) == 0
    _capi.lib.dsx_fft_train_destroy(h)
    assert n.value == documented_tape_bytes(H, L, heads, dim, B, T)


@pytest.mark.parametrize("dec,dim,mel", [((256, 4, 2, 9, 0, 0), 8, 80), ((256, 4, 2, 9, 0, 0), 1040, 80),
                                         ((256, 4, 2, 9, 0, 0), 24, 80), ((256, 4, 2, 9, 0, 0), 256, 128),
                                         ((320, 4, 5, 9, 0, 0), 256, 80), ((256, 4, 3, 9, 0, 0), 256, 80),
                                         ((256, 4, 2, 8, 0, 0), 256, 80), ((256, 65, 2, 9, 0, 0), 256, 80)])
def test_refused_configurations(lib_built, dec, dim, mel):
    from diffsinger_b200 import _capi
    c = _capi.FftConfig()
    c.dec.hidden, c.dec.layers, c.dec.heads, c.dec.kernel, c.dec.padding, c.dec.act = dec
    c.residual_channels, c.mel_bins = dim, mel
    h = ctypes.c_void_p()
    assert _capi.lib.dsx_fft_train_create(0, ctypes.byref(c), ctypes.byref(h)) == DSX_E_INVALID
    assert b"unsupported" in _capi.lib.dsx_last_error()


def _args():
    return torch.ones(1, 1, 80, 3), torch.zeros(1, dtype=torch.long), torch.ones(1, 256, 3)


def test_opt_in_routing(monkeypatch):
    from diffsinger_b200 import FFT, ffttrain
    calls = []
    monkeypatch.setattr(ffttrain, "fft_train_forward", lambda net, s, t, c: calls.append(net) or s)
    for m in (FFT(hparams=dict(HP, dsx_train=True)), FFT(hparams=HP, train=True)):
        assert m._dsx_train
        m.train()(*_args())
    assert len(calls) == 2
    assert not FFT(hparams=dict(HP, dsx_train=True), train=False)._dsx_train
    assert len(list(FFT(hparams=HP).parameters())) == 53


def test_training_without_opt_in_raises():
    from diffsinger_b200 import FFT, DsxError
    with pytest.raises(DsxError, match="eval mode only"):
        FFT(hparams=HP).train()(*_args())
    with torch.no_grad(), pytest.raises(DsxError, match="eval mode only"):
        FFT(hparams=dict(HP, dsx_train=True)).train()(*_args())


def test_opt_in_fails_loudly_without_a_gpu():
    from diffsinger_b200 import FFT, DsxError
    m = FFT(hparams=dict(HP, dsx_train=True)).train()
    with pytest.raises(DsxError, match="CPU"):
        m(*_args())
    spec, t, cond = _args()
    with pytest.raises(DsxError, match="spec.requires_grad"):
        m(spec.requires_grad_(True), t, cond)
    with pytest.raises(DsxError, match="cond must be"):
        m(torch.ones(1, 1, 80, 3), t, torch.ones(1, 256, 4))


FFT_SRC = '''
import torch.nn as nn


class FFT(nn.Module):
    def __init__(self, hidden_size=None, num_layers=None, kernel_size=None, num_heads=None):
        super().__init__()
        self.args = (hidden_size, num_layers, kernel_size, num_heads)
'''


def test_dropin_rebinds_the_fft_entry(tmp_path, monkeypatch):
    """install() on the stand-in tree with an 'fft' entry: the reference's FFT without dsx_train, diffsinger_b200.FFT
    with it; uninstall() restores the entry"""
    from standin_ref import write_tree
    write_tree(tmp_path)
    (tmp_path / "usr" / "diff" / "candidate_decoder.py").write_text(FFT_SRC)
    task = tmp_path / "usr" / "diffsinger_task.py"
    task.write_text(task.read_text() + "\nfrom usr.diff.candidate_decoder import FFT\n"
                    "DIFF_DECODERS['fft'] = lambda hp: FFT(hp['hidden_size'], hp['dec_layers'], "
                    "hp['dec_ffn_kernel_size'], hp['num_heads'])\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    for n in [n for n in sys.modules if n.split(".")[0] in ("usr", "utils", "modules", "tasks", "inference")]:
        monkeypatch.delitem(sys.modules, n)
    import usr.diffsinger_task as task_mod
    import diffsinger_b200
    import diffsinger_b200.dropin as dropin
    ref_entry = task_mod.DIFF_DECODERS['fft']
    dropin.install()
    try:
        built = task_mod.DIFF_DECODERS['fft'](dict(HP))
        assert type(built).__name__ == "FFT" and built.args == (256, 4, 9, 2)
        assert not isinstance(built, diffsinger_b200.FFT)
        built = task_mod.DIFF_DECODERS['fft'](dict(HP, dsx_train=True))
        assert isinstance(built, diffsinger_b200.FFT) and built._dsx_train
        assert (built.hidden_size, built.num_layers, built.kernel_size, built.num_heads) == (256, 4, 9, 2)
        dropin.install()
        assert isinstance(task_mod.DIFF_DECODERS['fft'](dict(HP, dsx_train=True)), diffsinger_b200.FFT)
    finally:
        dropin.uninstall()
    assert task_mod.DIFF_DECODERS['fft'] is ref_entry
