"""TEST INFRASTRUCTURE ONLY -- functional torch-CPU fp32 restatement of the reference's FastSpeech2 encoder and duration
path in eval mode, over state dicts with the reference's names:
  * FastspeechEncoder / FastspeechMIDIEncoder (modules/fastspeech/tts_modules.py:310-347, modules/diffsinger_midi/fs2.py:
    11-36) with the sinusoidal (common_layers.py:88-143) or the relative (modules/commons/espnet_positional_embedding.py:
    14-113) position term;
  * DurationPredictor.forward / .inference with dur_loss 'mse' (tts_modules.py:59-151) and LengthRegulator (:154-189);
  * FastSpeech2MIDI.forward(infer=True, skip_decoder=True) (modules/diffsinger_midi/fs2.py:55-118 with add_dur of
    modules/fastspeech/fs2.py:151-174) under configs without pitch, energy or speaker embeddings.
The FFTBlocks layers are oracle.fs2dec_oracle.decoder's: the encoder's FFTBlocks (no position embedding, no
pos_embed_alpha, padding mask txt_tokens == 0) compute exactly what the decoder's compute with pos_embed_alpha = 0 on the
masked embedding, whose rows are all zero exactly on the padding tokens (checked)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import fs2dec_oracle as D
from oracle.pe_oracle import make_positions, sinusoidal_table

# the shipped MIDI singing configuration (usr/configs/midi/e2e/opencpop/ds100_adj_rel.yaml and its bases) and the
# non-MIDI one (usr/configs/popcs_ds_beta6.yaml), as far as the encoder and the duration path read them
HPARAMS_MIDI = dict(hidden_size=256, enc_layers=4, enc_ffn_kernel_size=9, num_heads=2, ffn_padding='SAME', ffn_act='gelu',
                    dropout=0.1, dur_predictor_layers=5, dur_predictor_kernel=3, predictor_hidden=-1, rel_pos=True,
                    use_pos_embed=True, dur_loss='mse', predictor_grad=0.1, predictor_dropout=0.5)
HPARAMS_POPCS = dict(HPARAMS_MIDI, dur_predictor_layers=2, rel_pos=False, predictor_grad=0.0)
REL_MAX_LEN = 5000
DUR_LN_EPS = 1e-12


def _param(w):
    """nn.Module weights require grad, and ATen's matmul folds a strided 3-d input by that flag (see fs2dec_oracle._ffn)"""
    return w if w.requires_grad else torch.nn.Parameter(w)


def stack_hp(hp):
    """the decoder-oracle hparams of the encoder's FFTBlocks"""
    return dict(hidden_size=hp['hidden_size'], dec_layers=hp['enc_layers'], dec_ffn_kernel_size=hp['enc_ffn_kernel_size'],
                num_heads=hp['num_heads'], ffn_padding=hp['ffn_padding'], ffn_act=hp['ffn_act'])


def rel_table(P, H, dtype=torch.float32):
    """RelPositionalEncoding's table of length P (extend_pe with reverse=True, :23-45) -> [P, H] (``dtype`` gives a
    reference-precision table)"""
    pe = torch.zeros(P, H, dtype=dtype)
    position = torch.arange(P - 1, -1, -1.0, dtype=dtype).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, H, 2, dtype=dtype) * -(math.log(10000.0) / H))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


def embedding(sd, tokens, hp, addends=(), rel_len=REL_MAX_LEN):
    """forward_embedding (tts_modules.py:339-347, diffsinger_midi/fs2.py:12-23): [B, T, H], padding rows not masked.
    ``addends``: midi_embedding, midi_dur_embedding, slur_embedding ([B, T, H] or 0) for the MIDI encoder.  The position
    tables are built in the embedding's dtype (float32 in the reference; float64 for the edge tests)."""
    H = int(hp['hidden_size'])
    x = math.sqrt(H) * F.embedding(tokens, sd["embed_tokens.weight"], 0)
    if addends:
        midi, dur, slur = addends
        x = x + midi + dur + slur
    if hp.get('rel_pos'):
        x = x * math.sqrt(H) + rel_table(max(rel_len, tokens.shape[1]), H, x.dtype).to(x)[None, :tokens.shape[1]]
    else:
        T = tokens.shape[1]
        table = sinusoidal_table(max(2000, 1 + T), H, dtype=x.dtype).to(x)
        x = x + table.index_select(0, make_positions(tokens).view(-1)).view(*tokens.shape, -1)
    return x


def _stack_input(sd, tokens, hp, addends, rel_len):
    pad = tokens.eq(0)
    x = embedding(sd, tokens, hp, addends, rel_len)
    x = x * (~pad).to(x.dtype)[..., None]
    assert torch.equal(D.padding_mask(x), pad), "a non-padding token embedded to an all-zero row"
    return dict(sd, pos_embed_alpha=torch.zeros(1, dtype=x.dtype, device=x.device)), x


def encoder(sd, tokens, hp, addends=(), rel_len=REL_MAX_LEN):
    """FastspeechEncoder.forward(txt_tokens) / FastspeechMIDIEncoder.forward(txt_tokens, *addends) -> [B, T, H]"""
    sd0, x = _stack_input(sd, tokens, hp, addends, rel_len)
    return D.decoder(sd0, x, stack_hp(hp))


def encoder_fp16_sim(sd, tokens, hp, addends=(), rel_len=REL_MAX_LEN):
    """the encoder as the dsx kernels round it: the entry in fp32, then fs2dec_oracle.decoder_fp16_sim's stack"""
    sd0, x = _stack_input(sd, tokens, hp, addends, rel_len)
    return D.decoder_fp16_sim(sd0, x, stack_hp(hp))


def _dp_pad(hp, k):
    return ((k - 1) // 2, (k - 1) // 2) if hp['ffn_padding'] == 'SAME' else (k - 1, 0)


def dur_predictor(sd, xs, mask, hp, fp16=False):
    """DurationPredictor._forward(xs, x_masks) (tts_modules.py:113-129) -> the log-domain xs [B, T, 1].  fp16=True: each
    conv's input and weight rounded to fp16 as the dsx kernels round them (LayerNorm and the linear head in fp32)."""
    r = (lambda t: t.half().float()) if fp16 else (lambda t: t)
    k = int(hp['dur_predictor_kernel'])
    keep = (1 - mask.float()).to(xs.dtype)
    x = xs.transpose(1, -1)
    for i in range(int(hp['dur_predictor_layers'])):
        p = f"conv.{i}."
        x = F.conv1d(F.pad(r(x), _dp_pad(hp, k), value=0.0), r(sd[p + "1.weight"]), sd[p + "1.bias"])
        x = torch.relu(x)
        x = F.layer_norm(x.transpose(1, -1), (x.shape[1],), sd[p + "3.weight"], sd[p + "3.bias"], DUR_LN_EPS).transpose(1, -1)
        x = x * keep[:, None, :]
    x = F.linear(x.transpose(1, -1), _param(sd["linear.weight"]), sd["linear.bias"])
    return x * keep[:, :, None]


def out2dur(xs, offset=1.0):
    """tts_modules.py:119-124 (dur_loss 'mse'): xs [B, T, 1] -> int64 [B, T]"""
    return torch.clamp(torch.round(xs.squeeze(-1).exp() - offset), min=0).long()


def length_regulator(dur, dur_padding=None, alpha=1.0):
    """LengthRegulator.forward, tts_modules.py:159-189"""
    assert alpha > 0
    dur = torch.round(dur.float() * alpha).long()
    if dur_padding is not None:
        dur = dur * (1 - dur_padding.long())
    token_idx = torch.arange(1, dur.shape[1] + 1)[None, :, None].to(dur.device)
    dur_cumsum = torch.cumsum(dur, 1)
    dur_cumsum_prev = F.pad(dur_cumsum, [1, -1], mode='constant', value=0)
    pos_idx = torch.arange(dur.sum(-1).max())[None, None].to(dur.device)
    token_mask = (pos_idx >= dur_cumsum_prev[:, :, None]) & (pos_idx < dur_cumsum[:, :, None])
    return (token_idx * token_mask.long()).sum(1)


def sub(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def midi_addends(sd, pitch_midi, midi_dur, is_slur):
    """FastSpeech2MIDI.forward's three embeddings (diffsinger_midi/fs2.py:60-66)"""
    midi = F.embedding(pitch_midi, sd["midi_embed.weight"], 0)
    dur = F.linear(midi_dur[:, :, None], _param(sd["midi_dur_layer.weight"]), sd["midi_dur_layer.bias"])
    slur = F.embedding(is_slur, sd["is_slur_embed.weight"])
    return midi, dur, slur


def midi_forward(sd, tokens, pitch_midi, midi_dur, is_slur, hp, fp16=False):
    """FastSpeech2MIDI.forward(txt_tokens, infer=True, skip_decoder=True, pitch_midi=, midi_dur=, is_slur=) with
    mel2ph = None -> dict(encoder_out, dur, dur_choice, mel2ph, decoder_inp).  fp16=True: the encoder and the duration
    predictor as the dsx kernels round them."""
    ret = {}
    enc = encoder_fp16_sim if fp16 else encoder
    encoder_out = enc(sub(sd, "encoder."), tokens, hp, midi_addends(sd, pitch_midi, midi_dur, is_slur))
    ret['encoder_out'] = encoder_out
    src_nonpadding = (tokens > 0).float()[:, :, None]
    dur_inp = (encoder_out + 0 + 0) * src_nonpadding
    src_padding = tokens == 0                                        # add_dur, modules/fastspeech/fs2.py:160-166
    dur_inp = dur_inp.detach() + hp['predictor_grad'] * (dur_inp - dur_inp.detach())
    xs = dur_predictor(sub(sd, "dur_predictor."), dur_inp, src_padding, hp, fp16)
    ret['dur'] = xs
    ret['dur_choice'] = dur = out2dur(xs)
    ret['mel2ph'] = mel2ph = length_regulator(dur, src_padding)
    decoder_inp = F.pad(encoder_out, [0, 0, 1, 0])
    mel2ph_ = mel2ph[..., None].repeat([1, 1, encoder_out.shape[-1]])
    decoder_inp = torch.gather(decoder_inp, 1, mel2ph_)
    tgt_nonpadding = (mel2ph > 0).float()[:, :, None]
    ret['decoder_inp'] = (decoder_inp + 0) * tgt_nonpadding
    return ret


# ---- seeded parameters --------------------------------------------------------------------------------------------
def predictor_hidden(hp):
    return hp['predictor_hidden'] if hp['predictor_hidden'] > 0 else hp['hidden_size']


def state_dict_shapes(hp, vocab, midi=True):
    """name -> shape of the front end's state dict (the modules the encoder and duration path use), in the order of
    FastSpeech2MIDI's (midi=False: FastSpeech2's) state dict; encoder.embed_tokens.weight is encoder_embed_tokens.weight"""
    H, C, k = int(hp['hidden_size']), predictor_hidden(hp), int(hp['dur_predictor_kernel'])
    enc = {}
    for name, shape in D.state_dict_shapes(stack_hp(hp)).items():
        if name.startswith("layers.") or name.startswith("layer_norm."):
            enc["encoder." + name] = shape
    enc["encoder.embed_tokens.weight"] = (vocab, H)
    if not hp.get('rel_pos'):
        enc["encoder.embed_positions._float_tensor"] = (1,)
    dp = {}
    for i in range(int(hp['dur_predictor_layers'])):
        dp.update({f"dur_predictor.conv.{i}.1.weight": (C, H if i == 0 else C, k), f"dur_predictor.conv.{i}.1.bias": (C,),
                   f"dur_predictor.conv.{i}.3.weight": (C,), f"dur_predictor.conv.{i}.3.bias": (C,)})
    dp.update({"dur_predictor.linear.weight": (1, C), "dur_predictor.linear.bias": (1,)})
    out = {"encoder_embed_tokens.weight": (vocab, H)}
    if midi:    # FastSpeech2MIDI.__init__ deletes and re-adds the encoder after the duration predictor
        out.update(dp)
        out.update(enc)
        out.update({"midi_embed.weight": (300, H), "midi_dur_layer.weight": (H, 1), "midi_dur_layer.bias": (H,),
                    "is_slur_embed.weight": (2, H)})
    else:
        out.update(enc)
        out.update(dp)
    return out


def random_state_dict(seed, hp, vocab, midi=True, frames_per_token=10.0):
    """Seeded parameters from np.random.RandomState: the FFTBlocks of fs2dec_oracle.random_state_dict(seed), embeddings
    N(0, H^-1/2) with the padding rows 0 (nn.Embedding keeps them 0 in training), convolutions uniform in +-1/sqrt(fan_in),
    non-trivial LayerNorm affines, and a duration head whose bias is ln(frames_per_token) with small weights, so the
    predicted durations fall around 3-20 frames."""
    H = int(hp['hidden_size'])
    stack = D.random_state_dict(seed, stack_hp(hp))
    rs = np.random.RandomState(seed + 1000)
    out = {}
    for name, shape in state_dict_shapes(hp, vocab, midi).items():
        if name.startswith("encoder.layer"):
            out[name] = stack[name[len("encoder."):]]
            continue
        if name == "encoder.embed_tokens.weight":
            out[name] = out["encoder_embed_tokens.weight"]
            continue
        if name.endswith("_float_tensor"):
            v = np.zeros(shape)
        elif name.endswith("embed_tokens.weight") or name.endswith("embed.weight"):
            v = rs.standard_normal(shape) * H ** -0.5
            if name != "is_slur_embed.weight":
                v[0] = 0
        elif name == "dur_predictor.linear.weight":
            v = rs.uniform(-0.03, 0.03, shape)
        elif name == "dur_predictor.linear.bias":
            v = np.full(shape, math.log(frames_per_token))
        elif ".3." in name:
            v = 1.0 + 0.2 * rs.standard_normal(shape) if name.endswith("weight") else 0.1 * rs.standard_normal(shape)
        elif name.endswith("bias"):
            v = 0.05 * rs.standard_normal(shape)
        else:
            a = 1.0 / np.sqrt(int(np.prod(shape[1:])))
            v = rs.uniform(-a, a, shape)
        out[name] = torch.from_numpy(np.asarray(v, np.float32))
    return out


def fixture_inputs(seed, B, T, tails, vocab):
    """Realistic MIDI inputs: phoneme ids in [1, vocab), MIDI notes 48-76 held over runs of 1-3 tokens, note durations of
    0.1-0.8 s, about one slur in eight; utterance b is padding (all four 0) from tails[b] on."""
    rs = np.random.RandomState(seed)
    tok = rs.randint(1, vocab, (B, T))
    midi = np.zeros((B, T), np.int64)
    mdur = np.zeros((B, T), np.float32)
    for b in range(B):
        t = 0
        while t < T:
            n = rs.randint(1, 4)
            midi[b, t:t + n] = rs.randint(48, 77)
            mdur[b, t:t + n] = rs.uniform(0.1, 0.8)
            t += n
    slur = (rs.uniform(size=(B, T)) < 0.125).astype(np.int64)
    for b, tail in enumerate(tails):
        if tail is not None:
            tok[b, tail:] = midi[b, tail:] = slur[b, tail:] = 0
            mdur[b, tail:] = 0
    return (torch.from_numpy(tok), torch.from_numpy(midi), torch.from_numpy(mdur), torch.from_numpy(slur))


def half_integer_margin(xs, dur):
    """distance of exp(xs) - 1 to the nearest half-integer, and the margin 2 (dur + 1.5) (e^delta - 1) per unit delta"""
    y = xs.double().squeeze(-1).exp() - 1
    return (y - torch.floor(y) - 0.5).abs(), 2 * (dur.double() + 1.5)
