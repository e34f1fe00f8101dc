"""GPU: the Parallel WaveGAN vocoder of libdsx.so against the reference's output (tests/golden/pwg_*.npz) and the CPU
oracle (oracle/pwg_oracle.py), at the edges of what dsx_pwg_create accepts.

The residual layers use fp16 operands with fp32 accumulation.  A CPU simulation of that arithmetic
(pwg_oracle.generator(fp16=True): the x taps, the upsampled conditioning, the gate output and the layer weights rounded
to fp16) against fp32 gives, relative to the output's peak (max / mean):

    pwg_plain 8.1e-4 / 1.4e-4    pwg_pitch 7.5e-4 / 1.3e-4    shipped 6.9e-4 / 1.3e-4    hop300 1.1e-3 / 2.2e-4
    layers1 7.5e-4 / 1.4e-4      layers64 2.4e-3 / 5.7e-4     per_stack1 8.1e-4 / 1.6e-4 per_stack16 1.5e-3 / 2.4e-4
    one_frame 5.9e-4 / 1.4e-4    one_scale 6.4e-4 / 1.5e-4    hop1024 1.7e-3 / 2.3e-4    window16_pitch 9.6e-4 / 1.8e-4

Each case's bound is 3x its simulated max and mean (SIMULATED below, rounded up)."""
import ctypes
import sys
import textwrap

import numpy as np
import pytest
import torch

from oracle import pwg_oracle as P
from pwg_cases import FIXTURES, TOPOLOGIES, fixture, inputs, plain, random_sd, topology

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)

SIMULATED = {"pwg_plain.npz": (8.2e-4, 1.4e-4), "pwg_pitch.npz": (7.6e-4, 1.3e-4), "shipped": (7e-4, 1.3e-4),
             "hop300": (1.2e-3, 2.3e-4), "layers1": (7.6e-4, 1.5e-4), "layers64": (2.4e-3, 5.7e-4),
             "per_stack1": (8.2e-4, 1.6e-4), "per_stack16": (1.6e-3, 2.5e-4), "one_frame": (6e-4, 1.4e-4),
             "one_scale": (6.4e-4, 1.5e-4), "hop1024": (1.8e-3, 2.3e-4), "window16_pitch": (9.6e-4, 1.8e-4)}
FACTOR = 3.0


def within_bound(out, ref, case):
    out, ref = np.asarray(out, dtype=np.float64), np.asarray(ref, dtype=np.float64)
    peak, d = np.abs(ref).max(), np.abs(out - ref)
    smax, smean = SIMULATED[case]
    assert d.max() <= FACTOR * smax * peak and d.mean() <= FACTOR * smean * peak, (case, d.max() / peak, d.mean() / peak)


def generator(cfg, sd):
    from diffsinger_b200 import ParallelWaveGANGenerator
    m = ParallelWaveGANGenerator(**cfg)
    m.load_state_dict(sd, strict=True)
    return m.eval().to(DEV)


def fixture_inputs(g):
    pitch = torch.from_numpy(g["pitch"]).to(DEV) if "pitch" in g.files else None
    return torch.from_numpy(g["z"]).to(DEV), torch.from_numpy(g["c"]).to(DEV), pitch


@pytest.mark.parametrize("name", FIXTURES)
def test_reference_fixtures(lib_built, name):
    g, sd, cfg = fixture(name)
    m = generator(cfg, sd)
    with torch.no_grad():
        wav = m(*fixture_inputs(g)).cpu()
    within_bound(wav, g["wav"], name)


@pytest.mark.parametrize("topo", list(TOPOLOGIES))
def test_against_the_oracle(lib_built, topo):
    cfg, B, T = topology(topo)
    i = list(TOPOLOGIES).index(topo)
    sd = random_sd(cfg, 10 + i)
    z, c, pitch = inputs(cfg, B, T, 20 + i)
    with torch.no_grad():
        ref = P.generator(sd, cfg, z, c, pitch)
        wav = generator(cfg, sd)(z.to(DEV), c.to(DEV), pitch.to(DEV)).cpu()
    assert wav.shape == (B, 1, T * P.hop(cfg))
    within_bound(wav, ref, topo)


def test_weight_norm_and_plain_weights_agree(lib_built):
    g, sd, cfg = fixture("pwg_plain.npz")
    m = generator(cfg, sd)
    args = fixture_inputs(g)
    with torch.no_grad():
        a = m(*args).cpu()
        m.remove_weight_norm()                      # new parameters: the next call repacks
        b = m(*args).cpu()
        from diffsinger_b200 import ParallelWaveGANGenerator
        m2 = ParallelWaveGANGenerator(**cfg)
        m2.remove_weight_norm()
        m2.load_state_dict(plain(sd), strict=True)
        c = m2.eval().to(DEV)(*args).cpu()
    within_bound(b, a, "pwg_plain.npz")
    within_bound(c, a, "pwg_plain.npz")
    assert not torch.equal(a, torch.zeros_like(a))


def test_batch_is_each_utterance_alone_and_repeatable(lib_built):
    cfg, _, _ = topology("hop300")                  # hop 300: utterances do not start on a 64-row tile boundary
    sd = random_sd(cfg, 3)
    m = generator(cfg, sd)
    z, c, pitch = (t.to(DEV) for t in inputs(cfg, 3, 7, 4))
    with torch.no_grad():
        wav = m(z, c)
        assert torch.equal(wav, m(z, c))
        for b in range(3):
            assert torch.equal(wav[b:b + 1], m(z[b:b + 1], c[b:b + 1])), b


def test_strided_c_is_bit_identical(lib_built):
    g, sd, cfg = fixture("pwg_plain.npz")
    m = generator(cfg, sd)
    z, c, _ = fixture_inputs(g)
    view = c.transpose(1, 2).contiguous().transpose(1, 2)      # spec2wav's [B, T, 80] -> transposed view
    assert not view.is_contiguous()
    with torch.no_grad():
        assert torch.equal(m(z, view), m(z, c.contiguous()))


def test_pitch_is_ignored_without_a_pitch_embedding(lib_built):
    g, sd, cfg = fixture("pwg_plain.npz")
    m = generator(cfg, sd)
    z, c, _ = fixture_inputs(g)
    pitch = torch.randint(0, 300, (c.shape[0], c.shape[2]), device=DEV)
    with torch.no_grad():
        assert torch.equal(m(z, c), m(z, c, pitch))


def test_out_of_range_pitch_reads_a_zero_row(lib_built):
    g, sd, cfg = fixture("pwg_pitch.npz")
    m = generator(cfg, sd)
    z, c, pitch = fixture_inputs(g)
    sd0 = dict(sd)
    sd0["pitch_embed.weight"] = sd["pitch_embed.weight"].clone()
    sd0["pitch_embed.weight"][7] = 0
    bad = pitch.clone()
    bad[0, 2], bad[1, 5] = 300, -4
    ref = pitch.clone()
    ref[0, 2], ref[1, 5] = 7, 7
    with torch.no_grad():
        assert torch.equal(m(z, c, bad), generator(cfg, sd0)(z, c, ref))


def _config(**kw):
    from diffsinger_b200 import _capi
    c = _capi.PwgConfig(layers=30, stacks=3, kernel_size=3, residual_channels=64, gate_channels=128, skip_channels=64,
                        aux_channels=80, aux_context_window=2, num_scales=4, use_pitch_embed=0)
    for i, s in enumerate(kw.pop("scales", [4, 4, 4, 4])):
        c.upsample_scales[i] = s
    for k, v in kw.items():
        setattr(c, k, v)
    return c


@pytest.mark.parametrize("bad", [dict(residual_channels=128), dict(gate_channels=64), dict(skip_channels=128),
                                 dict(aux_channels=128), dict(kernel_size=5), dict(layers=0), dict(layers=65, stacks=5),
                                 dict(layers=30, stacks=4), dict(layers=34, stacks=2), dict(num_scales=0),
                                 dict(num_scales=5), dict(scales=[17, 1, 1, 1]), dict(scales=[0, 4, 4, 4]),
                                 dict(scales=[16, 16, 4, 2]), dict(aux_context_window=17), dict(aux_context_window=-1),
                                 dict(use_pitch_embed=2)])
def test_invalid_configs(lib_built, bad):
    from diffsinger_b200 import _capi
    out = ctypes.c_void_p()
    assert _capi.lib.dsx_pwg_create(0, ctypes.byref(_config(**bad)), ctypes.byref(out)) == -1
    assert b"unsupported" in _capi.lib.dsx_last_error()
    assert not out.value


def test_invalid_shapes(lib_built):
    from diffsinger_b200 import _capi
    g, sd, cfg = fixture("pwg_pitch.npz")
    m = generator(cfg, sd)
    z, c, pitch = fixture_inputs(g)
    with torch.no_grad():
        m(z, c, pitch)
    hnd, s = m._dsx[0], torch.cuda.current_stream().cuda_stream
    wav = torch.empty_like(z)
    st = _capi.Strides(*c.stride())
    f = _capi.lib.dsx_pwg_forward
    T = c.shape[2] - 4
    for B, TT in ((0, T), (2, 0), (-1, T), (1, (1 << 17) + 1), (1 << 12, 1 << 9)):      # the last two: above 2^25 samples
        assert f(hnd, z.data_ptr(), c.data_ptr(), st, pitch.data_ptr(), B, TT, wav.data_ptr(), s) == -1
    assert f(hnd, z.data_ptr(), c.data_ptr(), st, None, 2, T, wav.data_ptr(), s) == -1           # pitch is required
    torch.cuda.synchronize()


STANDIN = {
    "modules/__init__.py": "",
    "modules/parallel_wavegan/__init__.py": "",
    "modules/parallel_wavegan/models/__init__.py": "from .parallel_wavegan import *  # NOQA\n",
    "modules/parallel_wavegan/models/parallel_wavegan.py": """
        import torch

        class ParallelWaveGANGenerator(torch.nn.Module):     # replaced by diffsinger_b200's at install time
            def __init__(self, **kw):
                super().__init__()
                raise RuntimeError("stand-in ParallelWaveGANGenerator: dropin.install_pwg() should have replaced it")
    """,
    "vocoders/__init__.py": "",
    "vocoders/pwg.py": """
        import numpy as np
        import torch
        from torch import nn
        from modules.parallel_wavegan.models import ParallelWaveGANGenerator

        def load_pwg_model(config, state, device, official=True):    # vocoders/pwg.py:16-50 after reading the files
            model = ParallelWaveGANGenerator(**config["generator_params"])
            if official:
                model.load_state_dict(state)
            else:
                fake_task = nn.Module()
                fake_task.model_gen = model
                fake_task.load_state_dict({"model_gen." + k: v for k, v in state.items()}, strict=False)
            model.remove_weight_norm()
            model = model.eval().to(device)
            return model, None, config, device

        def spec2wav(model, config, device, mel, z, coarse=None):   # PWG.spec2wav (:82-103): z and f0_to_coarse(f0)
            pad_size = (config["generator_params"]["aux_context_window"],
                        config["generator_params"]["aux_context_window"])
            with torch.no_grad():
                c = np.pad(mel, (pad_size, (0, 0)), "edge")
                c = torch.FloatTensor(c).unsqueeze(0).transpose(2, 1).to(device)
                p = coarse                                           # from the caller
                if p is not None:
                    p = np.pad(p, (pad_size,), "edge")
                    p = torch.LongTensor(p[None, :]).to(device)
                y = model(z.to(device), c, p).view(-1)
            return y.cpu().numpy()
    """,
}


@pytest.mark.parametrize("name,official", [("pwg_plain.npz", True), ("pwg_pitch.npz", False)])
def test_dropin_pwg(lib_built, tmp_path, monkeypatch, name, official):
    for rel, body in STANDIN.items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(textwrap.dedent(body).lstrip("\n"))
    monkeypatch.syspath_prepend(str(tmp_path))
    for n in [n for n in sys.modules if n == "modules" or n.startswith(("modules.", "vocoders"))]:
        monkeypatch.delitem(sys.modules, n)
    import modules.parallel_wavegan.models as models_pkg
    import modules.parallel_wavegan.models.parallel_wavegan as ref_mod
    import vocoders.pwg as voc
    import diffsinger_b200.dropin as dropin
    ref_cls = ref_mod.ParallelWaveGANGenerator
    new_cls = dropin.install_pwg()
    try:
        assert voc.ParallelWaveGANGenerator is new_cls is ref_mod.ParallelWaveGANGenerator
        assert models_pkg.ParallelWaveGANGenerator is new_cls
        g, sd, cfg = fixture(name)
        model, _, config, _ = voc.load_pwg_model({"generator_params": cfg}, sd, DEV, official)
        w = cfg["aux_context_window"]
        for b in range(g["z"].shape[0]):
            mel = g["c"][b].T[w:len(g["c"][b].T) - w]                      # the unpadded [T, 80] mel
            f0 = g["pitch"][b][w:g["pitch"].shape[1] - w] if "pitch" in g.files else None
            wav = voc.spec2wav(model, config, DEV, mel, torch.from_numpy(g["z"][b:b + 1]), f0)
            within_bound(wav, g["wav"][b].reshape(-1), name)
    finally:
        dropin.uninstall_pwg()
    assert voc.ParallelWaveGANGenerator is ref_cls and ref_mod.ParallelWaveGANGenerator is ref_cls
    assert models_pkg.ParallelWaveGANGenerator is ref_cls
    for n in [n for n in sys.modules if n == "modules" or n.startswith(("modules.", "vocoders"))]:
        del sys.modules[n]
