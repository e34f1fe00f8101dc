"""GPU: the HiFi-GAN (NSF) vocoder of libdsx.so against the reference's output (tests/golden/hifigan_*.npz) and the
CPU oracle (oracle/hifigan_oracle.py).  The kernels use fp16 conv operands with fp32 accumulation; a CPU simulation of
that arithmetic (hifigan_oracle.generator(fp16=True): the input and weight of conv_pre, every ups and every ResBlock conv
rounded to fp16) puts the error at max 9e-5 / mean 2e-5 on a 0.1 signal, and the bound below is 2.5-4x that."""
import ctypes
import sys
import textwrap

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import hifigan_oracle as H

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def within_bound(out, ref):
    out, ref = np.asarray(out, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    peak, d = np.abs(ref).max(), np.abs(out - ref)
    assert d.max() <= 4e-3 * peak and d.mean() <= 1e-3 * peak, (d.max(), d.mean(), peak)


def fixture(name):
    g = golden(name)
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    h = dict(H.HPARAMS_TTS, upsample_initial_channel=int(g["upsample_initial_channel"]))
    return g, sd, h


def generator(h, sd):
    from diffsinger_b200 import HifiGanGenerator
    m = HifiGanGenerator(h)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV)


def draws(seed, B, L):
    """the NSF source's draws in the reference's order (source.py: torch.rand(B, 9) with column 0 zeroed, then randn)"""
    torch.manual_seed(seed)
    ph = torch.rand(B, 9)
    ph[:, 0] = 0
    return ph, torch.randn(B, L, 9)


def hop(h):
    return int(np.prod(h["upsample_rates"]))


@pytest.mark.parametrize("name", ["hifigan_nsf.npz", "hifigan_nsf_b1t9.npz"])
def test_reference_fixtures(lib_built, name):
    g, sd, h = fixture(name)
    m = generator(h, sd)
    mel, f0 = torch.from_numpy(g["mel"]), torch.from_numpy(g["f0"])
    B, _, T = mel.shape
    ph, nz = draws(int(g["rng_seed"]), B, T * hop(h))
    with torch.no_grad():
        wav = m(mel.to(DEV), f0.to(DEV), phase0=ph.to(DEV), src_noise=nz.to(DEV)).cpu()
        plain = m(mel.to(DEV)).cpu()
        ref_plain = g["wav_plain"] if "wav_plain" in g.files else H.generator(sd, h, mel).numpy()
    within_bound(wav, g["wav_nsf"])
    within_bound(plain, ref_plain)


TOPOLOGIES = {
    "tts128_resblock1": dict(H.HPARAMS_TTS),
    "resblock2": dict(H.HPARAMS_TTS, resblock="2", upsample_initial_channel=64, resblock_kernel_sizes=[3, 5, 7],
                      resblock_dilation_sizes=[[1, 2], [2, 6], [3, 12]]),
    "hop128": dict(H.HPARAMS_TTS, upsample_rates=[8, 4, 2, 2], upsample_kernel_sizes=[16, 8, 4, 4]),
    # 256- and 128-channel stages run one launch per conv, the 64- and 32-channel stages the chained ResBlock kernel
    "wide512": dict(H.HPARAMS_TTS, upsample_initial_channel=512),
}


@pytest.mark.parametrize("topo", list(TOPOLOGIES))
def test_against_the_oracle(lib_built, topo):
    from diffsinger_b200 import HifiGanGenerator
    h = TOPOLOGIES[topo]
    torch.manual_seed(1)
    m = HifiGanGenerator(h)                         # the reference's own initialisation
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    B, T = (2, 16) if topo == "wide512" else (2, 64)
    gen = torch.Generator().manual_seed(2)
    mel = torch.randn(B, 80, T, generator=gen)
    f0 = torch.rand(B, T, generator=gen) * 300 + 100
    f0[1, 10:20] = 0
    with torch.no_grad():
        torch.manual_seed(3)
        ref = H.generator(sd, h, mel, f0)
        ph, nz = draws(3, B, T * hop(h))
        wav = m.to(DEV)(mel.to(DEV), f0.to(DEV), phase0=ph.to(DEV), src_noise=nz.to(DEV)).cpu()
    within_bound(wav, ref)


def test_weight_norm_and_plain_checkpoints_agree(lib_built):
    g, sd, h = fixture("hifigan_nsf.npz")
    m = generator(h, sd)
    mel = torch.from_numpy(g["mel"]).to(DEV)
    with torch.no_grad():
        a = m(mel).cpu()
        m.remove_weight_norm()                      # new parameters: the next call repacks
        b = m(mel).cpu()
    within_bound(b, a)
    assert not torch.equal(a, torch.zeros_like(a))


def test_lengths_match_each_utterance_alone(lib_built):
    _, sd, h = fixture("hifigan_nsf.npz")
    m = generator(h, sd)
    B, T, hp = 3, 40, hop(h)
    gen = torch.Generator().manual_seed(4)
    mel = torch.randn(B, 80, T, generator=gen).to(DEV)
    f0 = (torch.rand(B, T, generator=gen) * 300 + 100).to(DEV)
    f0[2, 3:5] = 0
    ph, nz = (t.to(DEV) for t in draws(5, B, T * hp))
    lens = [T, T - 5, 9]
    with torch.no_grad():
        wav = m(mel, f0, lengths=torch.tensor(lens, dtype=torch.int32, device=DEV), phase0=ph, src_noise=nz)
        for b, L in enumerate(lens):
            alone = m(mel[b:b + 1, :, :L], f0[b:b + 1, :L], phase0=ph[b:b + 1], src_noise=nz[b:b + 1, :L * hp].contiguous())
            assert torch.equal(wav[b:b + 1, :, :L * hp], alone), b
            assert torch.count_nonzero(wav[b, :, L * hp:]) == 0


def test_strided_mel_is_bit_identical(lib_built):
    g, sd, h = fixture("hifigan_nsf.npz")
    m = generator(h, sd)
    mel_btc = torch.randn(2, 16, 80, generator=torch.Generator().manual_seed(6)).to(DEV)   # dsx_infer's [B, T, 80]
    f0 = torch.from_numpy(g["f0"]).to(DEV)
    with torch.no_grad():
        a = m(mel_btc.transpose(1, 2), f0, seed=3)
        b = m(mel_btc.transpose(1, 2).contiguous(), f0, seed=3)
    assert torch.equal(a, b)


def test_philox_draws(lib_built):
    g, sd, h = fixture("hifigan_nsf.npz")
    m = generator(h, sd)
    mel, f0 = torch.from_numpy(g["mel"]).to(DEV), torch.from_numpy(g["f0"]).to(DEV)
    with torch.no_grad():
        a, b, c = m(mel, f0, seed=7), m(mel, f0, seed=7), m(mel, f0, seed=8)
    assert torch.equal(a, b)
    assert not torch.equal(a, c)
    assert torch.isfinite(a).all()


def test_philox_draws_have_the_reference_distribution(lib_built):
    """In-kernel noise against torch.randn noise on an unvoiced stretch (the source is then noise only), and in-kernel
    initial phases: uniform per utterance, so identical utterances come out different."""
    g, sd, h = fixture("hifigan_nsf.npz")
    m = generator(h, sd)
    B, T, hp = 4, 128, hop(h)
    mel = torch.from_numpy(g["mel"][:1]).repeat(B, 1, 8).to(DEV)
    zero_ph = torch.zeros(B, 9, device=DEV)
    with torch.no_grad():
        plain = m(mel)
        unvoiced = torch.zeros(B, T, device=DEV)
        philox = m(mel, unvoiced, phase0=zero_ph, seed=11) - plain
        torch.manual_seed(12)
        torch_noise = m(mel, unvoiced, phase0=zero_ph, src_noise=torch.randn(B, T * hp, 9, device=DEV)) - plain
        ratio = (philox.std() / torch_noise.std()).item()
        assert 0.9 < ratio < 1.1, ratio
        assert abs(philox.mean().item() - torch_noise.mean().item()) < 0.1 * torch_noise.std().item()
        voiced = torch.full((B, T), 220.0, device=DEV)
        no_noise = torch.zeros(B, T * hp, 9, device=DEV)
        fixed = m(mel, voiced, phase0=zero_ph, src_noise=no_noise)
        drawn = m(mel, voiced, src_noise=no_noise, seed=11)
    assert all(torch.equal(fixed[0], fixed[b]) for b in range(1, B))
    assert all(not torch.equal(drawn[0], drawn[b]) for b in range(1, B))


def _config(**kw):
    from diffsinger_b200 import _capi
    c = _capi.HifiganConfig()
    c.num_upsamples = kw.get("nu", 4)
    for i, (u, k) in enumerate(zip(kw.get("rates", [8, 8, 2, 2]), kw.get("ks", [16, 16, 4, 4]))):
        c.upsample_rates[i], c.upsample_kernel_sizes[i] = u, k
    c.upsample_initial_channel = kw.get("c0", 128)
    c.resblock = kw.get("resblock", 1)
    c.num_kernels = 3
    for j, k in enumerate(kw.get("rk", [3, 7, 11])):
        c.resblock_kernel_sizes[j] = k
        for q, d in enumerate((1, 3, 5)):
            c.resblock_dilation_sizes[j][q] = d
    c.audio_sample_rate = kw.get("sr", 24000)
    c.use_pitch_embed = kw.get("pitch", 1)
    return c


@pytest.mark.parametrize("bad", [dict(nu=0), dict(nu=5), dict(ks=[15, 16, 4, 4]), dict(ks=[16, 16, 4, 5]),
                                 dict(rates=[8, 8, 2, 2], ks=[18, 16, 4, 4]), dict(c0=100), dict(resblock=3),
                                 dict(rk=[3, 4, 11]), dict(sr=0), dict(rates=[2, 2, 2, 3], ks=[4, 4, 4, 9])])
def test_invalid_configs(lib_built, bad):
    from diffsinger_b200 import _capi
    out = ctypes.c_void_p()
    assert _capi.lib.dsx_hifigan_create(0, ctypes.byref(_config(**bad)), ctypes.byref(out)) == -1
    assert not out.value


def test_invalid_shapes(lib_built):
    from diffsinger_b200 import _capi
    g, sd, h = fixture("hifigan_nsf.npz")
    m = generator(h, sd)
    mel = torch.from_numpy(g["mel"]).to(DEV)
    with torch.no_grad():
        m(mel)
    hnd, s = m._dsx[0], torch.cuda.current_stream().cuda_stream
    wav = torch.empty(2, 1, 16 * 256, device=DEV)
    st = _capi.Strides(*mel.stride())
    for B, T in ((0, 16), (2, 0), (-1, 16)):
        assert _capi.lib.dsx_hifigan_forward(hnd, mel.data_ptr(), st, None, None, None, None, 0, B, T, wav.data_ptr(), s) == -1
    h_plain = dict(h, use_pitch_embed=False)
    from diffsinger_b200 import DsxError, HifiGanGenerator
    plain = HifiGanGenerator(h_plain)
    plain.load_state_dict({k: v for k, v in sd.items() if not k.startswith(("noise_convs", "m_source"))}, strict=True)
    plain = plain.to(DEV)
    with pytest.raises(DsxError, match=r"\(-1\)"):
        plain(mel, torch.from_numpy(g["f0"]).to(DEV))


STANDIN = {
    "modules/__init__.py": "",
    "modules/hifigan/__init__.py": "",
    "modules/hifigan/hifigan.py": """
        import torch.nn as nn

        class HifiGanGenerator(nn.Module):     # replaced by diffsinger_b200.HifiGanGenerator at install time
            def __init__(self, h, c_out=1):
                super().__init__()
                raise RuntimeError("stand-in HifiGanGenerator: dropin.install_vocoder() should have replaced this class")
    """,
    "vocoders/__init__.py": "",
    "vocoders/hifigan.py": """
        import torch
        from modules.hifigan.hifigan import HifiGanGenerator

        def load_model(config, state, device):          # vocoders/hifigan.py:load_model after reading the checkpoint
            model = HifiGanGenerator(config)
            model.load_state_dict(state, strict=True)
            model.remove_weight_norm()
            model = model.eval().to(device)
            return model

        def spec2wav(model, mel, f0, device, **kw):    # HifiGAN.spec2wav: one utterance, mel [T, 80], f0 [T]
            with torch.no_grad():
                c = torch.FloatTensor(mel).unsqueeze(0).transpose(2, 1).to(device)
                f0 = torch.FloatTensor(f0[None, :]).to(device)
                return model(c, f0, **kw).view(-1).cpu().numpy()
    """,
}


def test_dropin_vocoder(lib_built, tmp_path, monkeypatch):
    for rel, body in STANDIN.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(body).lstrip("\n"))
    monkeypatch.syspath_prepend(str(tmp_path))
    for n in [n for n in sys.modules if n == "modules" or n.startswith(("modules.", "vocoders"))]:
        monkeypatch.delitem(sys.modules, n)
    import modules.hifigan.hifigan as ref_mod
    import vocoders.hifigan as voc
    import diffsinger_b200.dropin as dropin
    ref_cls = ref_mod.HifiGanGenerator
    new_cls = dropin.install_vocoder()
    try:
        assert voc.HifiGanGenerator is new_cls is ref_mod.HifiGanGenerator
        g, sd, h = fixture("hifigan_nsf_b1t9.npz")
        model = voc.load_model(h, sd, DEV)
        ph, nz = draws(int(g["rng_seed"]), 1, 9 * hop(h))
        wav = voc.spec2wav(model, g["mel"][0].T, g["f0"][0], DEV, phase0=ph.to(DEV), src_noise=nz.to(DEV))
        within_bound(wav, g["wav_nsf"].reshape(-1))
    finally:
        dropin.uninstall_vocoder()
    assert voc.HifiGanGenerator is ref_cls and ref_mod.HifiGanGenerator is ref_cls
    for n in [n for n in sys.modules if n == "modules" or n.startswith(("modules.", "vocoders"))]:
        del sys.modules[n]
