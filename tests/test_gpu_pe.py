"""GPU: the pitch extractor of libdsx.so against the reference's output (tests/golden/pitch_extractor.npz) and the CPU
oracle (oracle/pe_oracle.py).

The kernels run every conv and linear with fp16 operands and fp32 accumulation.  A CPU simulation of that rounding
(pe_oracle.pitch_extractor(fp16=True); the norms, the position term and the Linear(P, 2) head stay fp32) on
the committed fixture (H = 32, B = 2, T = 48) gives, against fp32, max 5.5e-3 / mean 1.3e-3 on channel 0 (log2 Hz) and
max 3.5e-3 / mean 1.0e-3 on channel 1 (uv logit), with no uv flips; the reference's smallest |uv logit| there is 4.7e-3.
At H = 256, B = 4, T = 400 the same simulation gave max 5.2e-3 / 4.4e-3 and mean 1.0e-3 / 9.6e-4.  The bounds below are
max 2e-2 and mean 4e-3 in those units; uv must agree wherever the reference's |logit| exceeds the max bound."""
import ctypes
import sys
import textwrap

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import hifigan_oracle as HG
from oracle import pe_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
MAX, MEAN = 2e-2, 4e-3


def pe_fixture():
    g = golden("pitch_extractor.npz")
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    return g, sd, hp


def model(hp, sd, conv_layers=2):
    from diffsinger_b200 import PitchExtractor
    m = PitchExtractor(80, conv_layers, hparams=hp)
    m.load_state_dict(sd, strict=True)
    return m.eval().to(DEV)


def run(m, mel):
    with torch.no_grad():
        r = m(mel.to(DEV))
    return r['pitch_pred'].cpu(), r['f0_denorm_pred'].cpu()


def check(pitch, f0, ref_pitch, ref_f0, mel, hp):
    pitch, ref_pitch = np.asarray(pitch, np.float64), np.asarray(ref_pitch, np.float64)
    f0, ref_f0 = np.asarray(f0, np.float64), np.asarray(ref_f0, np.float64)
    for ch in range(2):
        d = np.abs(pitch[..., ch] - ref_pitch[..., ch])
        assert d.max() <= MAX and d.mean() <= MEAN, (ch, d.max(), d.mean())
    pad = np.abs(np.asarray(mel)).sum(-1) == 0
    assert (f0[pad] == 0).all()
    use_uv = hp['pitch_type'] == 'frame' and hp['use_uv']
    if use_uv:
        sure = np.abs(ref_pitch[..., 1]) > MAX
        assert ((pitch[..., 1] > 0) == (ref_pitch[..., 1] > 0))[sure].all()
    both = (f0 > 0) & (ref_f0 > 0)
    assert both.sum() > 0
    if hp['pitch_norm'] == 'log':
        d = np.abs(np.log2(f0[both]) - np.log2(ref_f0[both]))
        assert d.max() <= MAX and d.mean() <= MEAN, (d.max(), d.mean())
    else:
        d = np.abs(f0 - ref_f0)[~pad] / hp['f0_std']
        assert d.max() <= MAX and d.mean() <= MEAN, (d.max(), d.mean())


def test_reference_fixture(lib_built):
    g, sd, hp = pe_fixture()
    pitch, f0 = run(model(hp, sd, int(g["conv_layers"])), torch.from_numpy(g["mel"]))
    check(pitch, f0, g["pitch_pred"], g["f0_denorm_pred"], g["mel"], hp)


# ---- the oracle at the shipped size (H = 256) ---------------------------------------------------------------------
CASES = {
    "T1": dict(T=1),
    "T37": dict(T=37),
    "T1000": dict(T=1000),
    "no_mel_encoder": dict(T=200, conv_layers=0),
    "predictor_hidden128_kernel3": dict(T=200, hp=dict(predictor_hidden=128, predictor_kernel=3)),
    "left_standard_no_uv": dict(T=200, hp=dict(ffn_padding='LEFT', pitch_norm='standard', f0_mean=7.5, f0_std=1.3,
                                              use_uv=False)),
}


def shipped(seed, conv_layers=2, **over):
    """a PitchExtractor at hidden_size 256 with seeded normalisation parameters: (hp, state dict)"""
    from diffsinger_b200 import PitchExtractor
    hp = dict(O.HPARAMS_E2E, **over)
    torch.manual_seed(seed)
    m = PitchExtractor(80, conv_layers, hparams=hp)
    return hp, O.random_state_dict(m.state_dict(), seed + 1)


def mel_batch(B, T, seed, tail=True):
    mel = torch.randn(B, T, 80, generator=torch.Generator().manual_seed(seed)) * 1.5 - 4.0
    if tail and T > 4:
        mel[1, T - T // 4:] = 0             # one utterance with a zero-padded tail
    return mel


@pytest.mark.parametrize("case", list(CASES))
def test_against_the_oracle(lib_built, case):
    c = CASES[case]
    L = c.get("conv_layers", 2)
    hp, sd = shipped(3, L, **c.get("hp", {}))
    mel = mel_batch(4, c["T"], 4)
    with torch.no_grad():
        ref_pitch, ref_f0 = O.pitch_extractor(sd, mel, hp, L)
    pitch, f0 = run(model(hp, sd, L), mel)
    check(pitch, f0, ref_pitch, ref_f0, mel, hp)


# ---- bit identity ---------------------------------------------------------------------------------------------------
def test_batch_at_equal_T_matches_each_utterance_alone(lib_built):
    hp, sd = shipped(5)
    m = model(hp, sd)
    mel = mel_batch(3, 300, 6).to(DEV)
    with torch.no_grad():
        r = m(mel)
        for b in range(3):
            alone = m(mel[b:b + 1])
            assert torch.equal(r['pitch_pred'][b:b + 1], alone['pitch_pred']), b
            assert torch.equal(r['f0_denorm_pred'][b:b + 1], alone['f0_denorm_pred']), b


def test_strided_mel_is_bit_identical(lib_built):
    hp, sd = shipped(7)
    m = model(hp, sd)
    mel_bct = torch.randn(2, 80, 150, generator=torch.Generator().manual_seed(8)).to(DEV)   # vocoder layout
    with torch.no_grad():
        a = m(mel_bct.transpose(1, 2))
        b = m(mel_bct.transpose(1, 2).contiguous())
    assert torch.equal(a['pitch_pred'], b['pitch_pred']) and torch.equal(a['f0_denorm_pred'], b['f0_denorm_pred'])


def test_two_calls_are_identical(lib_built):
    hp, sd = shipped(9)
    m = model(hp, sd)
    mel = mel_batch(4, 700, 10).to(DEV)
    with torch.no_grad():
        a, b = m(mel), m(mel)
    assert torch.equal(a['pitch_pred'], b['pitch_pred']) and torch.equal(a['f0_denorm_pred'], b['f0_denorm_pred'])


def test_repacks_after_load_state_dict(lib_built):
    g, sd, hp = pe_fixture()
    m = model(hp, sd)
    mel = torch.from_numpy(g["mel"]).to(DEV)
    with torch.no_grad():
        a = m(mel)['pitch_pred'].clone()
        sd2 = dict(sd)
        sd2["pitch_predictor.linear.bias"] = sd["pitch_predictor.linear.bias"] + torch.tensor([1.0, 0.0])
        m.load_state_dict(sd2, strict=True)
        b = m(mel)['pitch_pred']
    assert torch.allclose(b[..., 0] - a[..., 0], torch.ones_like(a[..., 0]), atol=1e-5)


# ---- invalid configs and shapes ------------------------------------------------------------------------------------
def _config(**kw):
    from diffsinger_b200 import _capi
    c = _capi.PeConfig()
    c.n_mel_bins, c.hidden, c.predictor_hidden, c.predictor_kernel = kw.get("bins", 80), kw.get("H", 256), kw.get("P", 256), kw.get("k", 5)
    c.conv_layers, c.causal, c.pitch_norm = kw.get("L", 2), kw.get("causal", 0), kw.get("norm", 0)
    c.f0_mean, c.f0_std, c.use_uv = 0.0, 1.0, kw.get("uv", 1)
    return c


@pytest.mark.parametrize("bad", [dict(bins=128), dict(H=0), dict(H=40), dict(H=272), dict(P=8), dict(k=4), dict(k=33),
                                 dict(L=-1), dict(L=17), dict(causal=2), dict(norm=2), dict(uv=3)])
def test_invalid_configs(lib_built, bad):
    from diffsinger_b200 import _capi
    out = ctypes.c_void_p()
    assert _capi.lib.dsx_pe_create(0, ctypes.byref(_config(**bad)), ctypes.byref(out)) == -1
    assert not out.value


def test_invalid_shapes(lib_built):
    from diffsinger_b200 import DsxError, _capi
    g, sd, hp = pe_fixture()
    m = model(hp, sd)
    mel = torch.from_numpy(g["mel"]).to(DEV)
    run(m, mel)
    hnd, s = m._dsx[0], torch.cuda.current_stream().cuda_stream
    out = torch.empty(2, 48, 2, device=DEV)
    st = _capi.Strides(mel.stride(0), mel.stride(2), mel.stride(1))
    for B, T in ((0, 48), (2, 0), (-1, 48), (70000, 1)):
        assert _capi.lib.dsx_pe_forward(hnd, mel.data_ptr(), st, B, T, out.data_ptr(), None, s) == -1
    with pytest.raises(DsxError, match=r"\[B, T, 80\]"):
        m(mel.transpose(1, 2))


# ---- end to end: mel -> PE -> vocoder -------------------------------------------------------------------------------
def test_pe_f0_drives_the_vocoder(lib_built):
    """The e2e recipe: mel -> dsx PE -> f0 -> dsx HifiGanGenerator.  The wav matches the oracle vocoder fed the same f0
    within the vocoder's bound, and that f0 is within the PE's bound of the reference's.  (Wavs from the PE's f0 and from
    the reference's f0 are not compared sample by sample: the NSF phase integrates f0, so a 1e-3 log2-Hz difference
    already moves the wav by about 15 % of its peak.)"""
    from diffsinger_b200 import HifiGanGenerator
    g, sd, hp = pe_fixture()
    vg = golden("hifigan_nsf.npz")
    vsd = {k[3:]: torch.from_numpy(vg[k]) for k in vg.files if k.startswith("sd.")}
    h = dict(HG.HPARAMS_TTS, upsample_initial_channel=int(vg["upsample_initial_channel"]))
    voc = HifiGanGenerator(h)
    voc.load_state_dict(vsd, strict=True)
    voc = voc.to(DEV)
    mel = torch.from_numpy(g["mel"]).to(DEV)
    B, T, _ = mel.shape
    hop = int(np.prod(h["upsample_rates"]))
    torch.manual_seed(13)
    ph = torch.rand(B, 9)
    ph[:, 0] = 0
    nz = torch.randn(B, T * hop, 9)
    with torch.no_grad():
        f0 = model(hp, sd)(mel)['f0_denorm_pred']
        wav = voc(mel.transpose(1, 2), f0, phase0=ph.to(DEV), src_noise=nz.to(DEV)).cpu().numpy()
        torch.manual_seed(13)
        ref = HG.generator(vsd, h, mel.transpose(1, 2).cpu(), f0.cpu()).numpy()
    both = (f0.cpu().numpy() > 0) & (g["f0_denorm_pred"] > 0)
    assert np.abs(np.log2(f0.cpu().numpy()[both]) - np.log2(g["f0_denorm_pred"][both])).max() <= MAX
    d, peak = np.abs(wav - ref), np.abs(ref).max()
    assert d.max() <= 4e-3 * peak and d.mean() <= 1e-3 * peak, (d.max(), d.mean(), peak)


# ---- drop-in ----------------------------------------------------------------------------------------------------------
STANDIN = {
    "modules/__init__.py": "",
    "modules/fastspeech/__init__.py": "",
    "modules/fastspeech/pe.py": """
        import torch.nn as nn

        class PitchExtractor(nn.Module):     # replaced by diffsinger_b200.PitchExtractor at install time
            def __init__(self, n_mel_bins=80, conv_layers=2):
                super().__init__()
                raise RuntimeError("stand-in PitchExtractor: dropin.install_pitch_extractor() should have replaced this")
    """,
    "utils/__init__.py": "",
    "utils/hparams.py": "hparams = {}\n",
    "inference/__init__.py": "",
    "inference/svs/__init__.py": "",
    "inference/svs/ds_e2e.py": """
        import torch
        from modules.fastspeech.pe import PitchExtractor

        class E2eInfer:                       # inference/svs/ds_e2e.py:11-45: the PE part
            def __init__(self, state, device):
                self.pe = PitchExtractor().to(device)
                self.pe.load_state_dict(state, strict=True)
                self.pe.eval()

            def f0(self, mel_out):
                with torch.no_grad():
                    return self.pe(mel_out)['f0_denorm_pred']
    """,
}


def test_dropin_pitch_extractor(lib_built, tmp_path, monkeypatch):
    for rel, body in STANDIN.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(body).lstrip("\n"))
    monkeypatch.syspath_prepend(str(tmp_path))
    roots = ("modules", "utils", "inference")
    drop = lambda: [n for n in sys.modules if n in roots or n.startswith(tuple(r + "." for r in roots))]
    for n in drop():
        monkeypatch.delitem(sys.modules, n)
    g, sd, hp = pe_fixture()
    import utils.hparams
    utils.hparams.hparams.update(hp)
    import modules.fastspeech.pe as ref_mod
    import inference.svs.ds_e2e as e2e
    import diffsinger_b200.dropin as dropin
    ref_cls = ref_mod.PitchExtractor
    new_cls = dropin.install_pitch_extractor()
    try:
        assert e2e.PitchExtractor is new_cls is ref_mod.PitchExtractor
        f0 = e2e.E2eInfer(sd, DEV).f0(torch.from_numpy(g["mel"]).to(DEV)).cpu().numpy()
        both = (f0 > 0) & (g["f0_denorm_pred"] > 0)
        assert both.sum() > 0
        assert np.abs(np.log2(f0[both]) - np.log2(g["f0_denorm_pred"][both])).max() <= MAX
    finally:
        dropin.uninstall_pitch_extractor()
    assert e2e.PitchExtractor is ref_cls and ref_mod.PitchExtractor is ref_cls
    for n in drop():
        del sys.modules[n]
