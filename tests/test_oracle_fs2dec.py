"""CPU: the FastSpeech2-decoder oracle (oracle/fs2dec_oracle.py) reproduces the reference's output stored in
tests/golden/fs2_decoder.npz (written by oracle/gen_golden_fs2dec.py from the unmodified reference), over the state dict
regenerated from the fixture's seed."""
import numpy as np
import torch

from conftest import golden
from oracle import fs2dec_oracle as O


def fixture():
    g = golden("fs2_decoder.npz")
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    return g, hp, O.random_state_dict(int(g["seed"]), hp)


def test_regenerated_state_dict_matches_the_checksums():
    g, hp, sd = fixture()
    stored = {k[4:]: g[k] for k in g.files if k.startswith("cks.")}
    assert set(stored) == set(sd) and len(sd) == 44
    for k, v in O.checksums(sd).items():
        np.testing.assert_allclose(v, stored[k], rtol=1e-12, atol=1e-12, err_msg=k)


def test_oracle_reproduces_the_reference_fixture():
    g, hp, sd = fixture()
    with torch.no_grad():
        out = O.decoder(sd, torch.from_numpy(g["x"]), hp).numpy()
    ref = g["out"]
    assert np.abs(out - ref).max() <= 1e-5 * np.abs(ref).max()


def test_fixture_covers_padding_and_the_position_skip():
    g, hp, _ = fixture()
    x = g["x"]
    pad = np.abs(x).sum(-1) == 0
    assert pad[0].sum() == 1 and pad[1, 73:].all() and not pad[1, :73].any()
    assert ((x[0, :, 0] == 0) & ~pad[0]).sum() == 1          # a frame the position scan skips without being padding
    assert (g["out"][pad] == 0).all() and np.isfinite(g["out"]).all()
    assert (hp["hidden_size"], hp["dec_layers"], hp["num_heads"], hp["dec_ffn_kernel_size"]) == (256, 4, 2, 9)
    assert hp["ffn_padding"] == "SAME" and hp["ffn_act"] == "gelu"


def test_random_state_dict_is_not_trivial():
    _, hp, sd = fixture()
    assert sd["layers.0.op.layer_norm2.bias"].abs().min() > 0          # beta2 != 0: padded rows feed the FFN conv
    assert sd["pos_embed_alpha"].item() != 1.0
