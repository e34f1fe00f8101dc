"""TEST INFRASTRUCTURE ONLY -- pins oracle/fs2enc_oracle.py to the LIVE reference FastSpeech2 encoder and duration path
(needs a checkout of the reference: DSX_REFERENCE_ROOT) and writes tests/golden/fs2_encoder.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_fs2enc.py

The reference modules are imported unmodified (stubs only for librosa / pycwt) and loaded strictly (FastSpeech2MIDI: all
but its decoder and mel_out, which skip_decoder=True does not run) with oracle.fs2enc_oracle.random_state_dict(SEED); the
oracle must reproduce, bit for bit:
  * FastSpeech2MIDI.forward(infer=True, skip_decoder=True) under usr/configs/midi/e2e/opencpop/ds100_adj_rel.yaml
    (rel_pos, a 5-layer duration predictor with k = 3): encoder_out, ret['dur'], ret['dur_choice'], mel2ph, decoder_inp;
  * the sinusoidal FastspeechEncoder and DurationPredictor.forward under usr/configs/popcs_ds_beta6.yaml;
  * LengthRegulator on zero durations, padding, alpha 0.5 and 1.3 with exact x.5 products, and unequal totals.
Inputs: B = 2, T_txt = 40, utterance 1 padded from token 29 (oracle.fixture_inputs).  fp16 operands move xs a little;
the input seed is the first from INPUT_SEED0 on for which every valid token's exp(xs) - 1 lies at least
2 (dur + 1.5) (e^XS_BOUND - 1) from a half-integer, so that the GPU, whose xs is within XS_BOUND of the reference's, must
give the same dur and mel2ph.  Weights are not stored, only per-tensor float64 checksums; the tests regenerate them."""
import math
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import fs2dec_oracle as D  # noqa: E402
from oracle import fs2enc_oracle as O  # noqa: E402

REF_ROOT = os.environ.get("DSX_REFERENCE_ROOT", "")
MIDI_CONFIG = "usr/configs/midi/e2e/opencpop/ds100_adj_rel.yaml"
POPCS_CONFIG = "usr/configs/popcs_ds_beta6.yaml"
HP_KEYS = tuple(O.HPARAMS_MIDI)
SEED, INPUT_SEED0, VOCAB, B, T, TAILS = 31, 100, 61, 2, 40, (None, 29)
XS_BOUND = 2e-3          # the GPU test's bound on |xs_dsx - xs| (tests/test_gpu_fs2enc.py)


class Dictionary:
    """the two members FastSpeech2.__init__ reads of its TokenTextEncoder"""

    def __init__(self, n):
        self.n = n

    def pad(self):
        return 0

    def __len__(self):
        return self.n


def load_reference():
    sys.dont_write_bytecode = True
    for n in ("librosa", "librosa.filters", "pycwt"):
        sys.modules.setdefault(n, types.ModuleType(n))
    sys.modules["pycwt"].wavelet = None
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    from utils.hparams import hparams, set_hparams

    def configure(config):
        cwd = os.getcwd()
        os.chdir(REF_ROOT)          # configs use repo-relative base_config paths
        try:
            set_hparams(config=config, exp_name="", print_hparams=False)
        finally:
            os.chdir(cwd)
        return {k: bool(hparams.get(k)) if k == 'rel_pos' else hparams[k] for k in HP_KEYS}   # rel_pos may be unset

    return hparams, configure


def ordered_shapes(sd):
    return [(k, tuple(v.shape)) for k, v in sd.items()]


def midi_case(hparams, configure):
    hp = configure(MIDI_CONFIG)
    assert hp == O.HPARAMS_MIDI, hp
    assert not (hparams['use_pitch_embed'] or hparams['use_energy_embed'] or hparams['use_spk_embed'] or
                hparams['use_spk_id']), "the MIDI forward here has no pitch, energy or speaker embedding"
    from modules.diffsinger_midi.fs2 import FastSpeech2MIDI
    model = FastSpeech2MIDI(Dictionary(VOCAB)).eval()
    sd = O.random_state_dict(SEED, hp, VOCAB)
    ref_sd = model.state_dict()
    assert [(k, s) for k, s in ordered_shapes(ref_sd) if k in sd] == ordered_shapes(sd)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    assert not unexpected and all(k.startswith(("decoder.", "mel_out.")) for k in missing), (missing, unexpected)
    # an xs error of XS_BOUND moves exp(xs) - 1 by at most (dur + 1.5) (e^XS_BOUND - 1); twice that is the margin
    for input_seed in range(INPUT_SEED0, INPUT_SEED0 + 5000):
        tok, midi, mdur, slur = O.fixture_inputs(input_seed, B, T, TAILS, VOCAB)
        with torch.no_grad():
            mine = O.midi_forward(sd, tok, midi, mdur, slur, hp)
        dist, per = O.half_integer_margin(mine['dur'], mine['dur_choice'])
        valid = tok > 0
        if (dist[valid] >= per[valid] * math.expm1(XS_BOUND)).all():
            break
    else:
        raise AssertionError("no input seed with the margin")
    with torch.no_grad():
        ret = model(tok, infer=True, skip_decoder=True, pitch_midi=midi, midi_dur=mdur, is_slur=slur)
        enc_ref = model.encoder(tok, *O.midi_addends(sd, midi, mdur, slur))
        sim = O.midi_forward(sd, tok, midi, mdur, slur, hp, fp16=True)
    assert torch.equal(enc_ref, mine['encoder_out']), (enc_ref - mine['encoder_out']).abs().max()
    for k in ('dur', 'dur_choice', 'mel2ph', 'decoder_inp'):
        assert torch.equal(ret[k], mine[k]), (k, (ret[k].double() - mine[k].double()).abs().max())
    d_enc = (sim['encoder_out'] - mine['encoder_out']).abs()
    d_xs = (sim['dur'] - mine['dur']).abs()
    print(f"MIDI: input seed {input_seed}; durations {ret['dur_choice'][valid].min().item()}.."
          f"{ret['dur_choice'][valid].max().item()}, T_mel {ret['mel2ph'].shape[1]}; fp16 simulation vs fp32: "
          f"encoder_out max {d_enc.max():.2e} mean {d_enc.mean():.2e}, xs max {d_xs.max():.2e}; "
          f"dur equal {torch.equal(sim['dur_choice'], mine['dur_choice'])}")
    return hp, sd, input_seed, (tok, midi, mdur, slur), ret, enc_ref


def popcs_case(hparams, configure, tok):
    hp = configure(POPCS_CONFIG)
    assert hp == O.HPARAMS_POPCS, hp
    from modules.fastspeech.tts_modules import DurationPredictor, FastspeechEncoder
    sd = O.random_state_dict(SEED, hp, VOCAB, midi=False)
    H = hp['hidden_size']
    emb = torch.nn.Embedding(VOCAB, H, 0)
    enc = FastspeechEncoder(emb, H, hp['enc_layers'], hp['enc_ffn_kernel_size'], num_heads=hp['num_heads']).eval()
    dp = DurationPredictor(H, n_chans=O.predictor_hidden(hp), n_layers=hp['dur_predictor_layers'],
                           dropout_rate=hp['predictor_dropout'], padding=hp['ffn_padding'],
                           kernel_size=hp['dur_predictor_kernel']).eval()
    enc_sd, dp_sd = O.sub(sd, "encoder."), O.sub(sd, "dur_predictor.")
    assert ordered_shapes(enc.state_dict()) == ordered_shapes(enc_sd)
    assert ordered_shapes(dp.state_dict()) == ordered_shapes(dp_sd)
    enc.load_state_dict(enc_sd, strict=True)
    dp.load_state_dict(dp_sd, strict=True)
    with torch.no_grad():
        enc_out = enc(tok)
        dur_inp = enc_out * (tok > 0).float()[:, :, None]
        xs = dp(dur_inp, tok == 0)
        mine_enc = O.encoder(enc_sd, tok, hp)
        mine_xs = O.dur_predictor(dp_sd, dur_inp, tok == 0, hp).squeeze(-1)
    assert torch.equal(enc_out, mine_enc), (enc_out - mine_enc).abs().max()
    assert torch.equal(xs, mine_xs), (xs - mine_xs).abs().max()
    print("popcs: sinusoidal encoder and DurationPredictor.forward bit-exact")
    return hp, sd, enc_out, xs


def lr_cases():
    from modules.fastspeech.tts_modules import LengthRegulator
    lr = LengthRegulator()
    dur = torch.tensor([[3, 0, 5, 1, 7, 0, 2, 9], [1, 3, 5, 7, 9, 11, 4, 4]])
    pad = torch.tensor([[0, 0, 0, 0, 0, 0, 1, 1], [0, 0, 0, 0, 0, 0, 0, 0]], dtype=torch.bool)
    cases = {"plain": (dur, pad, 1.0), "alpha_0.5_half_even": (dur, pad, 0.5), "alpha_1.3": (dur, pad, 1.3),
             "no_padding": (dur, None, 1.0)}
    out = {}
    for name, (d, p, a) in cases.items():
        ref = lr(d, p, a)
        assert torch.equal(ref, O.length_regulator(d, p, a)), name
        out[name] = ref
    x5 = (dur.float() * 0.5)[pad.logical_not()]
    assert (x5 - x5.floor() == 0.5).any(), "alpha 0.5 must hit exact .5 products"
    return dur, pad, {k: (v, c[2]) for (k, v), c in zip(out.items(), cases.values())}


def main():
    assert REF_ROOT and os.path.isdir(REF_ROOT), "set DSX_REFERENCE_ROOT to a checkout of the reference"
    hparams, configure = load_reference()
    hp, sd, input_seed, (tok, midi, mdur, slur), ret, enc_out = midi_case(hparams, configure)
    hp_p, sd_p, enc_out_p, xs_p = popcs_case(hparams, configure, tok)
    lr_dur, lr_pad, lr = lr_cases()
    out = os.path.join(ROOT, "tests", "golden", "fs2_encoder.npz")
    np.savez_compressed(
        out, seed=np.int64(SEED), input_seed=np.int64(input_seed), vocab=np.int64(VOCAB), xs_bound=np.float64(XS_BOUND),
        txt_tokens=tok.numpy(), pitch_midi=midi.numpy(), midi_dur=mdur.numpy(), is_slur=slur.numpy(),
        encoder_out=enc_out.numpy(), dur=ret['dur'].numpy(), dur_choice=ret['dur_choice'].numpy(),
        mel2ph=ret['mel2ph'].numpy(), decoder_inp=ret['decoder_inp'].numpy(),
        popcs_encoder_out=enc_out_p.numpy(), popcs_dur=xs_p.numpy(),
        lr_dur=lr_dur.numpy(), lr_pad=lr_pad.numpy(),
        **{f"lr.{k}": v.numpy() for k, (v, a) in lr.items()}, **{f"lr_alpha.{k}": np.float64(a) for k, (v, a) in lr.items()},
        **{"hp." + k: np.asarray(v) for k, v in hp.items()}, **{"hp_popcs." + k: np.asarray(v) for k, v in hp_p.items()},
        **{"cks." + k: v for k, v in D.checksums(sd).items()},
        **{"cks_popcs." + k: v for k, v in D.checksums(sd_p).items()})
    print("wrote", out, os.path.getsize(out) // 1024, "KB")


if __name__ == "__main__":
    main()
