"""CPU: the pitch-extractor oracle (oracle/pe_oracle.py) reproduces the reference's output stored in
tests/golden/pitch_extractor.npz (written by oracle/gen_golden_pe.py from the unmodified reference)."""
import numpy as np
import torch

from conftest import golden
from oracle import pe_oracle as O


def pe_fixture():
    g = golden("pitch_extractor.npz")
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    return g, sd, hp


def test_oracle_reproduces_the_reference_fixture():
    g, sd, hp = pe_fixture()
    with torch.no_grad():
        pitch, f0 = O.pitch_extractor(sd, torch.from_numpy(g["mel"]), hp, int(g["conv_layers"]))
    for out, ref in ((pitch.numpy(), g["pitch_pred"]), (f0.numpy(), g["f0_denorm_pred"])):
        assert np.abs(out - ref).max() <= 1e-6 * np.abs(ref).max()


def test_fixture_covers_padding_and_both_voicing_states():
    g, _, hp = pe_fixture()
    pad = np.abs(g["mel"]).sum(-1) == 0
    assert pad.any() and not pad.all()
    assert (g["f0_denorm_pred"][pad] == 0).all()
    uv = g["pitch_pred"][..., 1] > 0
    assert uv[~pad].any() and (~uv[~pad]).any()
    assert hp["pitch_type"] == "frame" and hp["use_uv"] and hp["pitch_norm"] == "log"


def test_position_table_matches_its_definition():
    t = O.sinusoidal_table(10, 16)
    assert torch.equal(t[0], torch.zeros(16))
    f = torch.exp(torch.arange(8, dtype=torch.float) * -(np.log(10000) / 7))
    assert torch.allclose(t[3], torch.cat([torch.sin(3 * f), torch.cos(3 * f)]))
    assert torch.equal(O.make_positions(torch.tensor([[1.0, 0.0, 2.0, 3.0]])), torch.tensor([[1, 0, 2, 3]]))


def test_fp16_option_leaves_the_fp32_path_bit_identical():
    g, sd, hp = pe_fixture()
    mel = torch.from_numpy(g["mel"])
    with torch.no_grad():
        a = O.pitch_extractor(sd, mel, hp, int(g["conv_layers"]))
        b = O.pitch_extractor(sd, mel, hp, int(g["conv_layers"]), fp16=False)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert torch.equal(O.sinusoidal_table(50, 16), O.sinusoidal_table(50, 16, dtype=torch.float))


def test_fp16_simulation_is_within_the_quoted_error():
    """pitch_extractor(fp16=True) on the fixture: within what test_gpu_pe.py quotes for the kernels' fp16 operands (max
    5.5e-3 / mean 1.3e-3 on log2 Hz, max 3.5e-3 / mean 1.0e-3 on the uv logit, no uv flips); padding frames stay 0"""
    g, sd, hp = pe_fixture()
    with torch.no_grad():
        pitch, f0 = O.pitch_extractor(sd, torch.from_numpy(g["mel"]), hp, int(g["conv_layers"]), fp16=True)
    pitch, f0 = pitch.numpy(), f0.numpy()
    for ch, (mx, mean) in enumerate(((5.5e-3, 1.3e-3), (3.5e-3, 1.0e-3))):
        d = np.abs(pitch[..., ch] - g["pitch_pred"][..., ch])
        assert 0 < d.max() <= 1.1 * mx and d.mean() <= 1.1 * mean, (ch, d.max(), d.mean())   # 10 %: other host CPUs
    assert ((pitch[..., 1] > 0) == (g["pitch_pred"][..., 1] > 0)).all()
    pad = np.abs(g["mel"]).sum(-1) == 0
    assert (f0[pad] == 0).all()
