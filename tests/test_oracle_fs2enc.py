"""CPU: oracle/fs2enc_oracle.py reproduces the live reference's outputs stored in tests/golden/fs2_encoder.npz (written
and pinned bit for bit by oracle/gen_golden_fs2enc.py on the machine that ran it), from the seeded parameters whose
checksums the fixture holds.  Another CPU's vector math may move the last bits of the float outputs (relative 1e-5 of
their peak); the integer outputs (durations, mel2ph) must match exactly: the fixture keeps every duration far from a
rounding boundary."""
import numpy as np
import torch

from conftest import golden
from oracle import fs2dec_oracle as D
from oracle import fs2enc_oracle as O


def _fixture(tag=""):
    g = golden("fs2_encoder.npz")
    hp = {k[len("hp" + tag + "."):]: g[k].item() for k in g.files if k.startswith("hp" + tag + ".")}
    return g, hp


def close(out, ref, what):
    assert np.abs(out - ref).max() <= 1e-5 * np.abs(ref).max(), what
    assert (out[ref == 0] == 0).all(), what


def _inputs(g):
    return tuple(torch.from_numpy(g[k]) for k in ("txt_tokens", "pitch_midi", "midi_dur", "is_slur"))


def test_seeded_parameters_match_the_checksums():
    for tag, midi in (("", True), ("_popcs", False)):
        g, hp = _fixture(tag)
        sd = O.random_state_dict(int(g["seed"]), hp, int(g["vocab"]), midi=midi)
        cks = {k[len("cks" + tag + "."):]: g[k] for k in g.files if k.startswith("cks" + tag + ".")}
        assert list(cks) == list(sd)
        for k, v in D.checksums(sd).items():
            np.testing.assert_allclose(v, cks[k], rtol=1e-12, atol=1e-9, err_msg=k)


def test_midi_forward_reproduces_the_reference():
    g, hp = _fixture()
    sd = O.random_state_dict(int(g["seed"]), hp, int(g["vocab"]))
    with torch.no_grad():
        ret = O.midi_forward(sd, *_inputs(g), hp)
    for k in ("encoder_out", "dur", "decoder_inp"):
        close(ret[k].numpy(), g[k], k)
    for k in ("dur_choice", "mel2ph"):
        assert np.array_equal(ret[k].numpy(), g[k]), k


def test_sinusoidal_encoder_and_duration_forward_reproduce_the_reference():
    g, hp = _fixture("_popcs")
    sd = O.random_state_dict(int(g["seed"]), hp, int(g["vocab"]), midi=False)
    tok = torch.from_numpy(g["txt_tokens"])
    with torch.no_grad():
        enc = O.encoder(O.sub(sd, "encoder."), tok, hp)
        xs = O.dur_predictor(O.sub(sd, "dur_predictor."), enc * (tok > 0).float()[:, :, None], tok == 0, hp)
    close(enc.numpy(), g["popcs_encoder_out"], "encoder_out")
    close(xs.squeeze(-1).numpy(), g["popcs_dur"], "xs")


def test_length_regulator_cases():
    g, _ = _fixture()
    dur, pad = torch.from_numpy(g["lr_dur"]), torch.from_numpy(g["lr_pad"])
    names = [k[3:] for k in g.files if k.startswith("lr.")]
    assert len(names) == 4
    for name in names:
        p = None if name == "no_padding" else pad
        out = O.length_regulator(dur, p, float(g["lr_alpha." + name]))
        assert np.array_equal(out.numpy(), g["lr." + name]), name


def test_fixture_has_the_margin_the_gpu_test_relies_on():
    g, _ = _fixture()
    dist, per = O.half_integer_margin(torch.from_numpy(g["dur"]), torch.from_numpy(g["dur_choice"]))
    valid = torch.from_numpy(g["txt_tokens"]) > 0
    assert (dist[valid] >= per[valid] * np.expm1(float(g["xs_bound"]))).all()
    d = g["dur_choice"][valid.numpy()]
    assert 3 <= d.min() and d.max() <= 25
