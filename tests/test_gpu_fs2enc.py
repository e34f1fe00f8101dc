"""GPU: the FastSpeech2 encoder, duration predictor and length regulator of libdsx.so against the reference's outputs
(tests/golden/fs2_encoder.npz) and the oracle (oracle/fs2enc_oracle.py, run here in fp32 with TF32 off).

Bounds.  The encoder's layers are the FastSpeech2 decoder's kernels: fp16 GEMM operands (weights, LayerNorm outputs, Q,
K, V, the softmax numerators, the attention output, the FFN activations), fp32 accumulation, residual stream and
LayerNorm statistics; the entry (embedding, addends, position term) is fp32.  The duration predictor's convolutions read
fp16 operands; its LayerNorms, the Linear(C, 1) head and out2dur are fp32.  oracle.fs2enc_oracle.midi_forward(fp16=True)
simulates that rounding on the CPU: on the committed fixture (H 256, 4 layers, B 2, T 40) it moves encoder_out by at
most 8.7e-5 (mean 1.1e-5) and xs by at most 1.13e-3 from fp32; fs2dec_oracle.decoder_fp16_sim, the same stack, gives
at most 1.2e-3 at T 1000.  The bounds below are encoder_out max 6e-3 / mean 6e-4 (the decoder's), xs 2e-3 (XS_BOUND,
the fixture's xs_bound).  The LayerNorms of the duration predictor divide by the spread of ReLU outputs, which is small
on some tokens: there the fp16 rounding of the convolutions' inputs is amplified (the simulation moves xs by up to
1.4e-2 at T 1550 with the oracle cases' seeded weights, mean 6e-4; on the GPU one token of the T 5200 case moves by
0.3 from fp32 but by 7e-3 from the simulation).  So the oracle cases compare xs with dur_predictor(fp16=True) on the
same input, where the remaining differences (summation order, and LayerNorm outputs rounded to fp16 on the other side
of a tie) are amplified the same way -- up to 7e-3 measured, bound 2e-2 -- and bound the mean distance to fp32 over
the valid tokens by 2e-3.  The fixture's input seed was chosen (oracle/gen_golden_fs2enc.py) so that every valid token's
exp(xs) - 1 lies at least 2 (dur + 1.5) (e^XS_BOUND - 1) from a half-integer: within the xs bound, dur, dur_choice and
mel2ph must then be exactly the reference's.  Padding rows must be exactly 0."""
import sys
import textwrap

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import fs2enc_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
MAX, MEAN = 6e-3, 6e-4
XS_BOUND = 2e-3
SIM_BOUND = 2e-2


def fixture():
    g = golden("fs2_encoder.npz")
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    assert float(g["xs_bound"]) == XS_BOUND
    return g, hp, O.random_state_dict(int(g["seed"]), hp, int(g["vocab"]))


def inputs(g):
    return tuple(torch.from_numpy(g[k]).to(DEV) for k in ("txt_tokens", "pitch_midi", "midi_dur", "is_slur"))


def models(hp, sd, vocab, midi=True):
    import diffsinger_b200 as dsx
    H = hp['hidden_size']
    cls = dsx.FastspeechMIDIEncoder if midi else dsx.FastspeechEncoder
    enc = cls(torch.nn.Embedding(vocab, H, 0), H, hp['enc_layers'], hp['enc_ffn_kernel_size'], num_heads=hp['num_heads'],
              hparams=hp)
    enc.load_state_dict(O.sub(sd, "encoder."), strict=True)
    dp = dsx.DurationPredictor(H, n_chans=O.predictor_hidden(hp), n_layers=hp['dur_predictor_layers'],
                               dropout_rate=hp['predictor_dropout'], padding=hp['ffn_padding'],
                               kernel_size=hp['dur_predictor_kernel'], hparams=hp)
    dp.load_state_dict(O.sub(sd, "dur_predictor."), strict=True)
    return enc.eval().to(DEV), dp.eval().to(DEV)


def addends(sd, midi, mdur, slur):
    return O.midi_addends({k: v.to(DEV) for k, v in sd.items()}, midi, mdur, slur)


def no_tf32(fn):
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            return fn()
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu


def check(out, ref, tok):
    out, ref = np.asarray(out.cpu(), np.float64), np.asarray(ref.cpu() if torch.is_tensor(ref) else ref, np.float64)
    d = np.abs(out - ref)
    assert np.isfinite(out).all()
    assert d.max() <= MAX and d.mean() <= MEAN, (d.max(), d.mean())
    pad = np.asarray(tok.cpu()) == 0
    assert (out[pad] == 0).all()


# ---- the reference fixture ------------------------------------------------------------------------------------------
def test_reference_fixture(lib_built):
    import diffsinger_b200 as dsx
    g, hp, sd = fixture()
    enc, dp = models(hp, sd, int(g["vocab"]))
    tok, midi, mdur, slur = inputs(g)
    with torch.no_grad():
        out = enc(tok, *addends(sd, midi, mdur, slur))
        check(out, g["encoder_out"], tok)
        dur, xs = dp.inference(out * (tok > 0).float()[:, :, None], tok == 0)
        mel2ph = dsx.LengthRegulator()(dur, tok == 0)
    d = (xs.cpu() - torch.from_numpy(g["dur"])).abs()
    assert d.max() <= XS_BOUND, d.max()
    assert (xs.cpu()[tok.cpu() == 0] == 0).all()
    assert np.array_equal(dur.cpu().numpy(), g["dur_choice"])
    assert np.array_equal(mel2ph.cpu().numpy(), g["mel2ph"])


def test_sinusoidal_encoder_and_duration_forward_fixture(lib_built):
    g = golden("fs2_encoder.npz")
    hp = {k[9:]: g[k].item() for k in g.files if k.startswith("hp_popcs.")}
    sd = O.random_state_dict(int(g["seed"]), hp, int(g["vocab"]), midi=False)
    enc, dp = models(hp, sd, int(g["vocab"]), midi=False)
    tok = torch.from_numpy(g["txt_tokens"]).to(DEV)
    with torch.no_grad():
        out = enc(tok)
        xs = dp(out * (tok > 0).float()[:, :, None], tok == 0)
    check(out, g["popcs_encoder_out"], tok)
    assert (xs.cpu() - torch.from_numpy(g["popcs_dur"])).abs().max() <= XS_BOUND


# ---- the oracle ---------------------------------------------------------------------------------------------------
CASES = {
    "T1": dict(T=1),
    "T63": dict(T=63),
    "T64": dict(T=64),
    "T65": dict(T=65),
    "T1550": dict(T=1550),
    "rel_T5200_longer_than_the_table": dict(T=5200, B=1),
    "sinusoidal_T300": dict(T=300, hp=dict(rel_pos=False)),
    "H128_heads1": dict(T=200, hp=dict(hidden_size=128, num_heads=1)),
    "H128_heads2": dict(T=130, hp=dict(hidden_size=128)),
    "L1": dict(T=200, hp=dict(enc_layers=1)),
    "relu": dict(T=200, hp=dict(ffn_act='relu')),
    "left_padding": dict(T=200, hp=dict(ffn_padding='LEFT', enc_ffn_kernel_size=4)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_against_the_oracle(lib_built, case):
    c = CASES[case]
    hp = dict(O.HPARAMS_MIDI, **c.get("hp", {}))
    T, B, V = c["T"], c.get("B", 3), 61
    sd = O.random_state_dict(41, hp, V, midi=hp['rel_pos'])
    tails = [None] + [T - T // 4 if T > 4 else None] * (B - 1)
    tok, midi, mdur, slur = (t.to(DEV) for t in O.fixture_inputs(42, B, T, tails, V))
    enc, dp = models(hp, sd, V, midi=hp['rel_pos'])
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    add = addends(sd, midi, mdur, slur) if hp['rel_pos'] else ()
    with torch.no_grad():
        out = enc(tok, *add)
    if hp['rel_pos']:
        assert enc._rel_len == max(5000, T)
    ref = no_tf32(lambda: O.encoder(O.sub(sdd, "encoder."), tok, hp, add, rel_len=max(5000, T)))
    check(out, ref, tok)
    # the duration predictor on the dsx encoder output: against the oracle with the kernels' fp16 operand rounding, and
    # on average against fp32
    x = out * (tok > 0).float()[:, :, None]
    with torch.no_grad():
        xs = dp(x, tok == 0)
    dps = O.sub(sdd, "dur_predictor.")
    xs_sim = no_tf32(lambda: O.dur_predictor(dps, x, tok == 0, hp, fp16=True)).squeeze(-1)
    xs_ref = no_tf32(lambda: O.dur_predictor(dps, x, tok == 0, hp)).squeeze(-1)
    assert (xs - xs_sim).abs().max().item() <= SIM_BOUND
    assert (xs - xs_ref).abs()[tok > 0].mean().item() <= XS_BOUND
    assert (xs[tok == 0] == 0).all()


def test_duration_rounding_is_out2dur_of_the_kernels_own_xs(lib_built):
    g, hp, sd = fixture()
    enc, dp = models(hp, sd, int(g["vocab"]))
    B, T = 8, 300
    tok, midi, mdur, slur = (t.to(DEV) for t in O.fixture_inputs(43, B, T, [None] + [250] * (B - 1), int(g["vocab"])))
    with torch.no_grad():
        x = enc(tok, *addends(sd, midi, mdur, slur)) * (tok > 0).float()[:, :, None]
        x = x + 0.3 * torch.randn(x.shape, generator=torch.Generator(device=DEV).manual_seed(1), device=DEV)
        dur, xs = dp.inference(x, tok == 0)
    y = xs.squeeze(-1).float().exp() - 1
    away = ((y - torch.floor(y) - 0.5).abs() > 1e-5) | (tok == 0)
    want = torch.clamp(torch.round(y), min=0).long()
    assert away.float().mean() > 0.99
    assert torch.equal(dur[away], want[away])
    assert (dur[tok == 0] == 0).all() and dur.dtype == torch.int64 and xs.shape == (B, T, 1)


# ---- length regulator ------------------------------------------------------------------------------------------------
def lr_check(dur, pad, alpha):
    import diffsinger_b200 as dsx
    with torch.no_grad():
        out = dsx.LengthRegulator()(dur.to(DEV), None if pad is None else pad.to(DEV), alpha)
        ref = O.length_regulator(dur.to(DEV), None if pad is None else pad.to(DEV), alpha)
    assert out.dtype == torch.int64 and torch.equal(out, ref), (out.shape, ref.shape)
    return out


def test_length_regulator_fixture_cases(lib_built):
    import diffsinger_b200 as dsx
    g = golden("fs2_encoder.npz")
    dur, pad = torch.from_numpy(g["lr_dur"]).to(DEV), torch.from_numpy(g["lr_pad"]).to(DEV)
    for name in [k[3:] for k in g.files if k.startswith("lr.")]:
        out = dsx.LengthRegulator()(dur, None if name == "no_padding" else pad, float(g["lr_alpha." + name]))
        assert np.array_equal(out.cpu().numpy(), g["lr." + name]), name


@pytest.mark.parametrize("alpha", [1.0, 0.5, 1.3])
def test_length_regulator_against_the_oracle(lib_built, alpha):
    gen = torch.Generator().manual_seed(7)
    dur = torch.randint(0, 12, (5, 90), generator=gen)
    dur[0, ::3] = 0
    dur[2, 40:] = 0                                             # unequal totals
    pad = torch.zeros(5, 90, dtype=torch.bool)
    pad[1, 60:] = True
    pad[3, :] = True                                            # an all-padding utterance: total 0
    lr_check(dur, pad, alpha)
    lr_check(dur, None, alpha)


def test_length_regulator_zero_total_and_large(lib_built):
    out = lr_check(torch.zeros(3, 7, dtype=torch.long), None, 1.0)
    assert out.shape == (3, 0)
    gen = torch.Generator().manual_seed(8)
    dur = torch.randint(0, 11, (16, 1550), generator=gen)
    pad = torch.zeros(16, 1550, dtype=torch.bool)
    pad[5:, 1400:] = True
    out = lr_check(dur, pad, 1.0)
    assert 7000 < out.shape[1] < 9000


def test_length_regulator_negative_durations_raise(lib_built):
    import diffsinger_b200 as dsx
    dur = torch.tensor([[3, -1, 2], [1, 1, 1]], device=DEV)
    with pytest.raises(dsx.DsxError, match="negative"):
        dsx.LengthRegulator()(dur)
    pad = torch.tensor([[0, 1, 0], [0, 0, 0]], dtype=torch.bool, device=DEV)
    assert dsx.LengthRegulator()(dur, pad).shape == (2, 5)   # a negative duration under padding is masked to 0


# ---- bit identity ---------------------------------------------------------------------------------------------------
def test_batch_matches_each_utterance_alone(lib_built):
    g, hp, sd = fixture()
    enc, dp = models(hp, sd, int(g["vocab"]))
    tok, midi, mdur, slur = (t.to(DEV) for t in O.fixture_inputs(44, 3, 150, [None, 120, 77], int(g["vocab"])))
    add = addends(sd, midi, mdur, slur)
    with torch.no_grad():
        out = enc(tok, *add)
        x = out * (tok > 0).float()[:, :, None]
        dur, xs = dp.inference(x, tok == 0)
        for b in range(3):
            one = enc(tok[b:b + 1], *(a[b:b + 1] for a in add))
            assert torch.equal(out[b:b + 1], one), b
            d1, x1 = dp.inference(x[b:b + 1], tok[b:b + 1] == 0)
            assert torch.equal(xs[b:b + 1], x1) and torch.equal(dur[b:b + 1], d1), b


def test_strided_addends_are_bit_identical(lib_built):
    g, hp, sd = fixture()
    enc, dp = models(hp, sd, int(g["vocab"]))
    tok, midi, mdur, slur = inputs(g)
    add = addends(sd, midi, mdur, slur)
    strided = [a.transpose(1, 2).contiguous().transpose(1, 2) for a in add]
    assert not strided[0].is_contiguous()
    with torch.no_grad():
        a = enc(tok, *add)
        b = enc(tok, *strided)
        c = enc(tok, add[0], 0, add[2])          # FastSpeech2MIDI passes 0 for a missing midi_dur
        d = enc(tok, add[0], torch.zeros_like(add[1]), add[2])
        x = a * (tok > 0).float()[:, :, None]
        assert torch.equal(dp(x, tok == 0), dp(x.transpose(1, 2).contiguous().transpose(1, 2), tok == 0))
    assert torch.equal(a, b) and torch.equal(c, d)


def test_two_calls_are_identical(lib_built):
    g, hp, sd = fixture()
    enc, dp = models(hp, sd, int(g["vocab"]))
    tok, midi, mdur, slur = inputs(g)
    add = addends(sd, midi, mdur, slur)
    with torch.no_grad():
        a, b = enc(tok, *add), enc(tok, *add)
        x = a * (tok > 0).float()[:, :, None]
        (d1, x1), (d2, x2) = dp.inference(x, tok == 0), dp.inference(x, tok == 0)
    assert torch.equal(a, b) and torch.equal(x1, x2) and torch.equal(d1, d2)


def test_all_padding_utterance_gives_zeros(lib_built):
    g, hp, sd = fixture()
    enc, dp = models(hp, sd, int(g["vocab"]))
    tok, midi, mdur, slur = (t.to(DEV) for t in O.fixture_inputs(45, 3, 80, [None, 60, None], int(g["vocab"])))
    tok[1] = 0
    add = addends(sd, midi, mdur, slur)
    with torch.no_grad():
        out = enc(tok, *add)
        assert torch.equal(out[1], torch.zeros_like(out[1]))
        for b in (0, 2):
            assert torch.equal(out[b:b + 1], enc(tok[b:b + 1], *(a[b:b + 1] for a in add)))
        dur, xs = dp.inference(out * (tok > 0).float()[:, :, None], tok == 0)
    assert (dur[1] == 0).all() and (xs[1] == 0).all()


def test_out_of_range_tokens_raise(lib_built):
    import diffsinger_b200 as dsx
    g, hp, sd = fixture()
    enc, _ = models(hp, sd, int(g["vocab"]))
    tok, midi, mdur, slur = inputs(g)
    add = addends(sd, midi, mdur, slur)
    for bad in (int(g["vocab"]), -1):
        t = tok.clone()
        t[0, 3] = bad
        with pytest.raises(dsx.DsxError, match="txt_tokens"):
            enc(t, *add)


def test_repacks_after_load_state_dict(lib_built):
    g, hp, sd = fixture()
    enc, dp = models(hp, sd, int(g["vocab"]))
    tok, midi, mdur, slur = inputs(g)
    add = addends(sd, midi, mdur, slur)
    keep = tok > 0
    with torch.no_grad():
        a = enc(tok, *add).clone()
        x = a * keep.float()[:, :, None]
        xa = dp(x, tok == 0).clone()
        esd = O.sub(sd, "encoder.")
        esd["layer_norm.bias"] = esd["layer_norm.bias"] + 1.0
        enc.load_state_dict(esd, strict=True)
        psd = O.sub(sd, "dur_predictor.")
        psd["linear.bias"] = psd["linear.bias"] + 0.5
        dp.load_state_dict(psd, strict=True)
        b = enc(tok, *add)
        xb = dp(x, tok == 0)
    assert torch.allclose((b - a)[keep], torch.ones_like(a[keep]), atol=1e-5)
    assert torch.allclose((xb - xa)[keep], torch.full_like(xa[keep], 0.5), atol=1e-6)


# ---- drop-in ----------------------------------------------------------------------------------------------------------
# Stand-ins for the reference modules install_fs2_encoder() touches.  Their classes raise: a passing test ran dsx.  The
# FastSpeech2MIDI stand-in's forward is the infer + skip_decoder path without pitch, energy or speaker embeddings.
STANDIN = {
    "modules/__init__.py": "",
    "modules/fastspeech/__init__.py": "",
    "modules/fastspeech/tts_modules.py": """
        import torch.nn as nn

        class _Ref(nn.Module):
            def __init__(self, *a, **k):
                super().__init__()
                raise RuntimeError(f"stand-in {type(self).__name__}: install_fs2_encoder() should have replaced it")

        class FastspeechEncoder(_Ref):
            pass

        class DurationPredictor(_Ref):
            pass

        class LengthRegulator(_Ref):
            pass
    """,
    "modules/fastspeech/fs2.py": """
        import torch
        import torch.nn as nn
        import torch.nn.functional as F
        from modules.fastspeech.tts_modules import FastspeechEncoder, DurationPredictor, LengthRegulator
        from utils.hparams import hparams

        FS_ENCODERS = {
            'fft': lambda hp, embed_tokens, d: FastspeechEncoder(
                embed_tokens, hp['hidden_size'], hp['enc_layers'], hp['enc_ffn_kernel_size'], num_heads=hp['num_heads']),
        }

        class FastSpeech2(nn.Module):
            def __init__(self, dictionary):
                super().__init__()
                self.hidden_size = hparams['hidden_size']
                self.encoder_embed_tokens = nn.Embedding(len(dictionary), self.hidden_size, 0)
                self.encoder = FS_ENCODERS['fft'](hparams, self.encoder_embed_tokens, dictionary)
                ph = hparams['predictor_hidden'] if hparams['predictor_hidden'] > 0 else self.hidden_size
                self.dur_predictor = DurationPredictor(
                    self.hidden_size, n_chans=ph, n_layers=hparams['dur_predictor_layers'],
                    dropout_rate=hparams['predictor_dropout'], padding=hparams['ffn_padding'],
                    kernel_size=hparams['dur_predictor_kernel'])
                self.length_regulator = LengthRegulator()

            def add_dur(self, dur_input, mel2ph, txt_tokens, ret):
                src_padding = txt_tokens == 0
                dur_input = dur_input.detach() + hparams['predictor_grad'] * (dur_input - dur_input.detach())
                dur, xs = self.dur_predictor.inference(dur_input, src_padding)
                ret['dur'], ret['dur_choice'] = xs, dur
                ret['mel2ph'] = mel2ph = self.length_regulator(dur, src_padding).detach()
                return mel2ph
    """,
    "modules/diffsinger_midi/__init__.py": "",
    "modules/diffsinger_midi/fs2.py": """
        import torch
        import torch.nn as nn
        import torch.nn.functional as F
        from modules.fastspeech.tts_modules import FastspeechEncoder
        from modules.fastspeech.fs2 import FastSpeech2
        from utils.hparams import hparams

        class FastspeechMIDIEncoder(FastspeechEncoder):
            pass

        FS_ENCODERS = {
            'fft': lambda hp, embed_tokens, d: FastspeechMIDIEncoder(
                embed_tokens, hp['hidden_size'], hp['enc_layers'], hp['enc_ffn_kernel_size'], num_heads=hp['num_heads']),
        }

        class FastSpeech2MIDI(FastSpeech2):
            def __init__(self, dictionary):
                super().__init__(dictionary)
                del self.encoder
                self.encoder = FS_ENCODERS['fft'](hparams, self.encoder_embed_tokens, dictionary)
                self.midi_embed = nn.Embedding(300, self.hidden_size, 0)
                self.midi_dur_layer = nn.Linear(1, self.hidden_size)
                self.is_slur_embed = nn.Embedding(2, self.hidden_size)

            def forward(self, txt_tokens, infer=True, skip_decoder=True, **kwargs):
                ret = {}
                midi = self.midi_embed(kwargs['pitch_midi'])
                midi_dur = self.midi_dur_layer(kwargs['midi_dur'][:, :, None])
                slur = self.is_slur_embed(kwargs['is_slur'])
                encoder_out = self.encoder(txt_tokens, midi, midi_dur, slur)
                src_nonpadding = (txt_tokens > 0).float()[:, :, None]
                mel2ph = self.add_dur(encoder_out * src_nonpadding, None, txt_tokens, ret)
                decoder_inp = F.pad(encoder_out, [0, 0, 1, 0])
                decoder_inp = torch.gather(decoder_inp, 1, mel2ph[..., None].repeat([1, 1, encoder_out.shape[-1]]))
                ret['decoder_inp'] = decoder_inp * (mel2ph > 0).float()[:, :, None]
                return ret
    """,
    "utils/__init__.py": "",
    "utils/hparams.py": "hparams = {}\n",
}


class _Dictionary:
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n


def test_dropin_fs2_encoder(lib_built, tmp_path, monkeypatch):
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
    import modules.diffsinger_midi.fs2 as mfs2
    import modules.fastspeech.fs2 as fs2
    import modules.fastspeech.tts_modules as tts
    import diffsinger_b200 as dsx
    import diffsinger_b200.dropin as dropin
    names = ("FastspeechEncoder", "DurationPredictor", "LengthRegulator")
    before = {(m.__name__, n): getattr(m, n) for m in (fs2, mfs2, tts) for n in names + ("FastspeechMIDIEncoder",)
              if hasattr(m, n)}
    dropin.install_fs2_encoder()
    try:
        assert fs2.FastspeechEncoder is dsx.FastspeechEncoder and mfs2.FastspeechMIDIEncoder is dsx.FastspeechMIDIEncoder
        assert fs2.DurationPredictor is dsx.DurationPredictor and fs2.LengthRegulator is dsx.LengthRegulator
        assert all(getattr(tts, n) is before[("modules.fastspeech.tts_modules", n)] for n in names)
        with torch.cuda.device(DEV):
            used = torch.cuda.memory_allocated(DEV)
            net = mfs2.FastSpeech2MIDI(_Dictionary(int(g["vocab"])))
            assert torch.cuda.memory_allocated(DEV) == used      # construction does not touch the GPU
        assert type(net.encoder) is dsx.FastspeechMIDIEncoder and type(net.dur_predictor) is dsx.DurationPredictor
        net.load_state_dict(sd, strict=True)
        net = net.to(DEV).eval()
        tok, midi, mdur, slur = inputs(g)
        with torch.no_grad():
            ret = net(tok, infer=True, skip_decoder=True, pitch_midi=midi, midi_dur=mdur, is_slur=slur)
        assert np.array_equal(ret['mel2ph'].cpu().numpy(), g["mel2ph"])
        assert np.array_equal(ret['dur_choice'].cpu().numpy(), g["dur_choice"])
        assert (ret['dur'].cpu() - torch.from_numpy(g["dur"])).abs().max() <= XS_BOUND
        ref = torch.from_numpy(g["decoder_inp"])
        d = (ret['decoder_inp'].cpu() - ref).abs()
        assert d.max() <= MAX and d.mean() <= MEAN and (ret['decoder_inp'].cpu()[ref.abs().sum(-1) == 0] == 0).all()
    finally:
        dropin.uninstall_fs2_encoder()
    after = {(m.__name__, n): getattr(m, n) for m in (fs2, mfs2, tts) for n in names + ("FastspeechMIDIEncoder",)
             if hasattr(m, n)}
    assert after == before
    for n in drop():
        del sys.modules[n]
