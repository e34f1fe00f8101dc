"""GPU: the FastSpeech2 decoder of libdsx.so against the reference's output (tests/golden/fs2_decoder.npz) and the
oracle (oracle/fs2dec_oracle.py, run here in fp32 with TF32 off).

The kernels round every GEMM operand to fp16 (weights, LayerNorm outputs, Q scaled in fp32 first, K, V, the softmax
numerators P, the attention output, the FFN activations) and keep accumulation, the residual stream, LayerNorm
statistics and the softmax state in fp32.  oracle.decoder_fp16_sim simulates that rounding on the CPU: against fp32 it
gives max 1.2e-3 / mean 1.6e-4 on the committed fixture (H 256, L 4, B 2, T 100) and max 1.1e-3 / mean 1.4e-4 at H 256,
B 4, T 1000 (outputs up to 5.8 in magnitude).  The bounds below are max 6e-3 and mean 6e-4; padding frames must be
exactly 0."""
import sys
import textwrap

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import fs2dec_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
MAX, MEAN = 6e-3, 6e-4


def fixture():
    g = golden("fs2_decoder.npz")
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    return g, hp, O.random_state_dict(int(g["seed"]), hp)


def model(hp, sd):
    from diffsinger_b200 import FastspeechDecoder
    m = FastspeechDecoder(hparams=hp)
    m.load_state_dict(sd, strict=True)
    return m.eval().to(DEV)


def run(m, x):
    with torch.no_grad():
        return m(x.to(DEV))


def oracle_gpu(sd, x, hp):
    """the oracle on the GPU in fp32 (TF32 off): the CPU takes minutes at T = 3000"""
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            return O.decoder({k: v.to(DEV) for k, v in sd.items()}, x.to(DEV), hp).cpu()
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu


def check(out, ref, x):
    out, ref = np.asarray(out.cpu(), np.float64), np.asarray(ref, np.float64)
    d = np.abs(out - ref)
    assert np.isfinite(out).all()
    assert d.max() <= MAX and d.mean() <= MEAN, (d.max(), d.mean())
    pad = (np.abs(np.asarray(x)).sum(-1) == 0)
    assert (out[pad] == 0).all()


def test_reference_fixture(lib_built):
    g, hp, sd = fixture()
    check(run(model(hp, sd), torch.from_numpy(g["x"])), g["out"], g["x"])


# ---- the oracle ---------------------------------------------------------------------------------------------------
CASES = {
    "T1": dict(T=1),
    "T37": dict(T=37),
    "T1000": dict(T=1000),
    "T3000_regrows_the_table": dict(T=3000),
    "left_padding": dict(T=200, hp=dict(ffn_padding='LEFT', dec_ffn_kernel_size=4)),
    "relu": dict(T=200, hp=dict(ffn_act='relu')),
    "heads4_D64": dict(T=300, hp=dict(num_heads=4)),
    "H128": dict(T=300, hp=dict(hidden_size=128, num_heads=1)),
    "H128_heads2_D64": dict(T=130, hp=dict(hidden_size=128)),
    "L1": dict(T=200, hp=dict(dec_layers=1)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_against_the_oracle(lib_built, case):
    c = CASES[case]
    hp = dict(O.HPARAMS_POPCS, **c.get("hp", {}))
    sd = O.random_state_dict(21, hp)
    T = c["T"]
    x = O.fixture_input(22, 4, T, hp["hidden_size"], tail=T - T // 4)
    check(run(model(hp, sd), x), oracle_gpu(sd, x, hp), x)


# ---- bit identity ---------------------------------------------------------------------------------------------------
def test_batch_matches_each_utterance_alone(lib_built):
    g, hp, sd = fixture()
    m = model(hp, sd)
    x = O.fixture_input(23, 3, 300, 256, tail=190).to(DEV)
    with torch.no_grad():
        out = m(x)
        for b in range(3):
            assert torch.equal(out[b:b + 1], m(x[b:b + 1])), b


def test_strided_input_is_bit_identical(lib_built):
    g, hp, sd = fixture()
    m = model(hp, sd)
    x_bht = torch.randn(2, 256, 150, generator=torch.Generator().manual_seed(24)).to(DEV)   # cond-like [B, H, T]
    with torch.no_grad():
        a = m(x_bht.transpose(1, 2))
        b = m(x_bht.transpose(1, 2).contiguous())
    assert torch.equal(a, b)


def test_two_calls_are_identical(lib_built):
    g, hp, sd = fixture()
    m = model(hp, sd)
    x = O.fixture_input(25, 4, 700, 256, tail=500).to(DEV)
    with torch.no_grad():
        a, b = m(x), m(x)
    assert torch.equal(a, b)


def test_all_padding_utterance_gives_zeros(lib_built):
    """the reference returns NaN for it (softmax over no key); dsx returns 0 and leaves the other utterances alone"""
    g, hp, sd = fixture()
    m = model(hp, sd)
    x = O.fixture_input(26, 3, 120, 256, tail=90).to(DEV)
    x[1] = 0
    with torch.no_grad():
        out = m(x)
        assert torch.equal(out[1], torch.zeros_like(out[1]))
        assert torch.equal(out[0:1], m(x[0:1])) and torch.equal(out[2:3], m(x[2:3]))


def test_repacks_after_load_state_dict(lib_built):
    g, hp, sd = fixture()
    m = model(hp, sd)
    x = torch.from_numpy(g["x"]).to(DEV)
    with torch.no_grad():
        a = m(x).clone()
        sd2 = dict(sd)
        sd2["layer_norm.bias"] = sd["layer_norm.bias"] + 1.0
        m.load_state_dict(sd2, strict=True)
        b = m(x)
    keep = ~O.padding_mask(x)
    assert torch.allclose((b - a)[keep], torch.ones_like(a[keep]), atol=1e-5)


# ---- drop-in ----------------------------------------------------------------------------------------------------------
STANDIN = {
    "modules/__init__.py": "",
    "modules/fastspeech/__init__.py": "",
    "modules/fastspeech/tts_modules.py": """
        import torch.nn as nn

        class FastspeechDecoder(nn.Module):   # the reference class: must stay bound here
            def __init__(self, hidden_size=None, num_layers=None, kernel_size=None, num_heads=None):
                super().__init__()
                raise RuntimeError("stand-in FastspeechDecoder: install_fs2_decoder() should have replaced it in fs2")
    """,
    "modules/fastspeech/fs2.py": """
        import torch.nn as nn
        from modules.fastspeech.tts_modules import FastspeechDecoder
        from utils.hparams import hparams

        FS_DECODERS = {                       # modules/fastspeech/fs2.py:15-18
            'fft': lambda hp: FastspeechDecoder(
                hp['hidden_size'], hp['dec_layers'], hp['dec_ffn_kernel_size'], hp['num_heads']),
        }

        class FastSpeech2(nn.Module):         # the decoder part of :21-40
            def __init__(self):
                super().__init__()
                self.decoder = FS_DECODERS['fft'](hparams)
                self.mel_out = nn.Linear(hparams['hidden_size'], 80, bias=True)
    """,
    "utils/__init__.py": "",
    "utils/hparams.py": "hparams = {}\n",
}


def test_dropin_fs2_decoder(lib_built, tmp_path, monkeypatch):
    for rel, body in STANDIN.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(body).lstrip("\n"))
    monkeypatch.syspath_prepend(str(tmp_path))
    roots = ("modules", "utils")
    drop = lambda: [n for n in sys.modules if n in roots or n.startswith(tuple(r + "." for r in roots))]
    for n in drop():
        monkeypatch.delitem(sys.modules, n)
    g, hp, sd = fixture()
    import utils.hparams
    utils.hparams.hparams.update(hp)
    import modules.fastspeech.fs2 as fs2
    import modules.fastspeech.tts_modules as tts
    import diffsinger_b200.dropin as dropin
    ref_cls = fs2.FastspeechDecoder
    new_cls = dropin.install_fs2_decoder()
    try:
        assert fs2.FastspeechDecoder is new_cls and tts.FastspeechDecoder is ref_cls
        net = fs2.FastSpeech2()
        assert type(net.decoder) is new_cls and isinstance(net.mel_out, torch.nn.Linear)
        net.decoder.load_state_dict(sd, strict=True)
        net = net.to(DEV).eval()
        x = torch.from_numpy(g["x"]).to(DEV)
        with torch.no_grad():
            out = net.decoder(x)
            assert torch.equal(out, model(hp, sd)(x))
        check(out, g["out"], g["x"])
    finally:
        dropin.uninstall_fs2_decoder()
    assert fs2.FastspeechDecoder is ref_cls and tts.FastspeechDecoder is ref_cls
    for n in drop():
        del sys.modules[n]
