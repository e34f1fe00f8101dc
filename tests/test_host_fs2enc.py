"""CPU: the encoder / duration-path mirrors (diffsinger_b200.FastspeechEncoder, FastspeechMIDIEncoder, DurationPredictor,
LengthRegulator) have the reference's state-dict surface, load the seeded reference parameters strictly, and refuse what
they do not run (CPU tensors, training mode, unsupported hparams) with DsxError."""
import ctypes

import pytest
import torch

from conftest import golden
from oracle import fs2enc_oracle as O


def _fixture(tag=""):
    g = golden("fs2_encoder.npz")
    hp = {k[len("hp" + tag + "."):]: g[k].item() for k in g.files if k.startswith("hp" + tag + ".")}
    return g, hp


def _encoder(hp, vocab, midi=True, **kw):
    import diffsinger_b200 as dsx
    hp = dict(hp, **kw)
    cls = dsx.FastspeechMIDIEncoder if midi else dsx.FastspeechEncoder
    return cls(torch.nn.Embedding(vocab, hp['hidden_size'], 0), hp['hidden_size'], hp['enc_layers'],
               hp['enc_ffn_kernel_size'], num_heads=hp['num_heads'], hparams=hp)


def _dur_predictor(hp, **kw):
    import diffsinger_b200 as dsx
    hp = dict(hp, **kw)
    return dsx.DurationPredictor(hp['hidden_size'], n_chans=O.predictor_hidden(hp), n_layers=hp['dur_predictor_layers'],
                                 dropout_rate=hp['predictor_dropout'], padding=hp['ffn_padding'],
                                 kernel_size=hp['dur_predictor_kernel'], hparams=hp)


@pytest.mark.parametrize("tag", ["", "_popcs"])
def test_state_dict_surface_matches_the_reference(lib_built, tag):
    g, hp = _fixture(tag)
    midi = tag == ""
    V = int(g["vocab"])
    ref = O.state_dict_shapes(hp, V, midi)
    enc = _encoder(hp, V, midi)
    mine = [(k, tuple(v.shape)) for k, v in enc.state_dict().items()]
    assert mine == [(k[8:], s) for k, s in ref.items() if k.startswith("encoder.")]
    assert ("embed_positions._float_tensor" in dict(mine)) == (not midi)
    assert not any("pos_embed_alpha" in k for k, _ in mine)
    dp = [(k, tuple(v.shape)) for k, v in _dur_predictor(hp).state_dict().items()]
    assert dp == [(k[14:], s) for k, s in ref.items() if k.startswith("dur_predictor.")]


def test_strict_loading(lib_built):
    g, hp = _fixture()
    sd = O.random_state_dict(int(g["seed"]), hp, int(g["vocab"]))
    enc, dp = _encoder(hp, int(g["vocab"])), _dur_predictor(hp)
    enc.load_state_dict(O.sub(sd, "encoder."), strict=True)
    dp.load_state_dict(O.sub(sd, "dur_predictor."), strict=True)
    for k, v in enc.state_dict().items():
        assert torch.equal(v, sd["encoder." + k]), k
    import diffsinger_b200 as dsx
    assert dsx.LengthRegulator().state_dict() == {}


@pytest.mark.parametrize("bad", [dict(use_pos_embed=False), dict(hidden_size=96), dict(num_heads=3),
                                 dict(enc_ffn_kernel_size=8), dict(ffn_act="swish"), dict(enc_layers=0)])
def test_unsupported_encoder_config_raises(lib_built, bad):
    from diffsinger_b200 import DsxError
    g, hp = _fixture()
    with pytest.raises(DsxError, match="unsupported"):
        _encoder(hp, int(g["vocab"]), **bad)


def test_rel_pos_without_midi_raises_at_forward_only(lib_built):
    """FastSpeech2MIDI.__init__ builds (and deletes) a FastspeechEncoder under rel_pos: construction must work"""
    from diffsinger_b200 import DsxError
    g, hp = _fixture()
    enc = _encoder(hp, int(g["vocab"]), midi=False).eval()
    with pytest.raises(DsxError, match="rel_pos"):
        enc(torch.ones(1, 4, dtype=torch.long))


@pytest.mark.parametrize("bad", [dict(dur_loss="huber"), dict(dur_loss="mog"), dict(dur_predictor_kernel=4),
                                 dict(dur_predictor_layers=0), dict(predictor_hidden=300)])
def test_unsupported_duration_predictor_config_raises(lib_built, bad):
    from diffsinger_b200 import DsxError
    _, hp = _fixture()
    with pytest.raises(DsxError, match="unsupported"):
        _dur_predictor(hp, **bad)


def test_cpu_tensors_raise(lib_built):
    import diffsinger_b200 as dsx
    g, hp = _fixture()
    tok = torch.from_numpy(g["txt_tokens"])
    z = torch.zeros(*tok.shape, hp['hidden_size'])
    with pytest.raises(dsx.DsxError, match="CPU"):
        _encoder(hp, int(g["vocab"])).eval()(tok, z, z, z)
    with pytest.raises(dsx.DsxError, match="CPU"):
        _dur_predictor(hp).eval()(z, tok == 0)
    with pytest.raises(dsx.DsxError, match="CPU"):
        dsx.LengthRegulator()(torch.ones_like(tok), tok == 0)


def test_training_mode_raises(lib_built):
    from diffsinger_b200 import DsxError
    g, hp = _fixture()
    tok = torch.from_numpy(g["txt_tokens"])
    z = torch.zeros(*tok.shape, hp['hidden_size'])
    with pytest.raises(DsxError, match="eval"):
        _encoder(hp, int(g["vocab"])).train()(tok, z, z, z)
    with pytest.raises(DsxError, match="eval"):
        _dur_predictor(hp).train().inference(z, tok == 0)


def test_length_regulator_rejects_bad_arguments(lib_built):
    import diffsinger_b200 as dsx
    with pytest.raises(dsx.DsxError, match="alpha"):
        dsx.LengthRegulator()(torch.ones(1, 3, dtype=torch.long), alpha=0.0)
    with pytest.raises(dsx.DsxError, match="integer"):
        dsx.LengthRegulator()(torch.ones(1, 3))


def test_c_abi_symbols_are_exported(lib_built):
    from diffsinger_b200 import _capi
    lib = ctypes.CDLL(_capi.LIB_PATH)
    for name in ("dsx_fs2enc_create", "dsx_fs2enc_destroy", "dsx_fs2enc_load", "dsx_fs2enc_forward",
                 "dsx_durpred_create", "dsx_durpred_destroy", "dsx_durpred_load", "dsx_durpred_forward",
                 "dsx_length_totals", "dsx_length_regulate"):
        assert hasattr(lib, name), name
        assert name in _capi.SYMBOLS
