"""FastSpeech2 encoder, duration predictor and length regulator whose forward runs the sm_90a kernels of libdsx.so
(dsx_fs2enc_*, dsx_durpred_*, dsx_length_* in include/dsx.h).

* ``FastspeechEncoder(embed_tokens, hidden_size=None, num_layers=None, kernel_size=None, num_heads=2, *, hparams=None)``
  and ``FastspeechMIDIEncoder`` keep the reference's constructors, submodule names and state dicts
  (modules/fastspeech/tts_modules.py:310-347, modules/diffsinger_midi/fs2.py:11-36): ``layers.*``, ``layer_norm.*``, the
  shared ``embed_tokens`` and, for the sinusoidal positions, ``embed_positions._float_tensor``; RelPositionalEncoding
  (``rel_pos: true``) has no state, and there is no ``pos_embed_alpha``.
* ``DurationPredictor(idim, n_layers, n_chans, kernel_size, dropout_rate, offset, padding)`` (tts_modules.py:59-151,
  ``dur_loss: 'mse'``): ``conv.i.1.*``, ``conv.i.3.*``, ``linear.*``.
* ``LengthRegulator(pad_value=0.0)`` (tts_modules.py:154-189): no state.

So a FastSpeech2 checkpoint loads with ``strict=True``.  The modules only hold the parameters: ``forward`` packs them into
the library (once per storage and version, so again after ``load_state_dict`` or ``.to()``) and runs there.  There is no
eager or CPU path: a CPU tensor raises ``DsxError``, and so does a module in training mode, except the encoders under the
``dsx_train`` opt-in (hparams key or ``train=`` keyword): then a training-mode forward under autograd runs the sm_90a
training step of ``diffsinger_b200.fs2enctrain`` (dropout p = hparams['dropout'], gradients for every parameter,
``embed_tokens.weight`` included, and for the MIDI addends).  ``DurationPredictor`` under the same opt-in runs the
training step of ``diffsinger_b200.durtrain`` in ``forward`` (dropout p = its ``dropout_rate``, gradients for every
parameter and for its input); ``.inference()`` stays eval-only.  Construction does not touch the GPU
(FastSpeech2MIDI.__init__ builds and deletes a non-MIDI encoder).
"""
import ctypes
import math

import torch
import torch.nn as nn

from . import _capi
from ._capi import DsxError, check, lib
from .fs2dec import TransformerEncoderLayer, _fs2dec_config, fs2dec_params
from .modules import _get_hparams
from .pitch import LayerNorm, SinusoidalPositionalEmbedding
from .sampler import PackedModule, _need_cuda, _ptr, _stream, _strides_bct

_PADDING = {'SAME': 0, 'LEFT': 1}
REL_POS_MAX_LEN = 5000          # RelPositionalEncoding's max_len (espnet_positional_embedding.py:14)


def _eval_only(module, what):
    if module.training:
        raise DsxError(f"the dsx {what} runs in eval mode only (call .eval()); training stays with the reference's modules")


class RelPositionalEncoding(nn.Module):
    """espnet_positional_embedding.py:91-113 (reverse=True).  The table is not state: the kernel evaluates row t as
    position P - 1 - t, where P is the table length the reference would hold (max_len, or the longest input since)."""

    def __init__(self, d_model, dropout_rate=0.0, max_len=REL_POS_MAX_LEN):
        super().__init__()
        self.d_model, self.xscale, self.max_len = d_model, math.sqrt(d_model), max_len


class FastspeechEncoder(PackedModule):
    _what = "FastSpeech2 encoder"

    def __init__(self, embed_tokens, hidden_size=None, num_layers=None, kernel_size=None, num_heads=2, *, hparams=None,
                 train=None):
        super().__init__()
        hp = _get_hparams(hparams)
        hidden_size = hp['hidden_size'] if hidden_size is None else hidden_size          # tts_modules.py:311-314
        kernel_size = hp['enc_ffn_kernel_size'] if kernel_size is None else kernel_size
        num_layers = hp['dec_layers'] if num_layers is None else num_layers
        padding, act = hp['ffn_padding'], hp['ffn_act']
        if not hp.get('use_pos_embed', True):
            raise DsxError("unsupported FastSpeech2 encoder configuration: use_pos_embed = False (no shipped config "
                           "turns the encoder's position term off)")
        stack = _fs2dec_config(hidden_size, num_layers, kernel_size, num_heads, padding, act, "enc", "encoder")
        if not isinstance(embed_tokens, nn.Embedding) or embed_tokens.embedding_dim != stack.hidden:
            raise DsxError(f"embed_tokens must be an nn.Embedding of dim {stack.hidden}")
        self.hidden_size, self.num_layers, self.num_heads = stack.hidden, stack.layers, stack.heads
        self.kernel_size, self.padding, self.act = stack.kernel, padding, act
        self.dropout = hp.get('dropout', 0.0)      # identity in eval mode; the training step's p under dsx_train
        self.layers = nn.ModuleList([TransformerEncoderLayer(self.hidden_size, self.kernel_size, self.num_heads, padding, act)
                                     for _ in range(self.num_layers)])
        self.layer_norm = nn.LayerNorm(self.hidden_size)
        self.embed_tokens = embed_tokens
        self.embed_scale = math.sqrt(self.hidden_size)
        self.padding_idx = 0
        self.rel_pos = bool(hp.get('rel_pos'))
        if self.rel_pos:
            self.embed_positions = RelPositionalEncoding(self.hidden_size, dropout_rate=0.0)
        else:
            self.embed_positions = SinusoidalPositionalEmbedding(self.hidden_size, self.padding_idx)
        self._rel_len = REL_POS_MAX_LEN
        self._cfg = _capi.Fs2EncConfig(stack=stack, vocab=embed_tokens.num_embeddings, pos=int(self.rel_pos))
        self._dsx_train = bool(train if train is not None else hp.get("dsx_train", False))
        self._dsx_trainer = None

    def __getstate__(self):
        # the library handles are ctypes pointers: copies (EMA deepcopy, torch.save of the module) make their own
        state = self.__dict__.copy()
        state["_dsx"], state["_wkey"], state["_keep"] = None, None, None
        state["_dsx_trainer"] = None
        return state

    def _dsx_train_step(self):
        vocab = self.embed_tokens.num_embeddings
        if self._dsx_trainer is None or self._dsx_trainer.cfg.vocab != vocab:
            from .fs2enctrain import Fs2EncTrainStep
            cfg = _capi.Fs2EncConfig(stack=_fs2dec_config(self.hidden_size, self.num_layers, self.kernel_size,
                                                          self.num_heads, self.padding, self.act, "enc", "encoder"),
                                     vocab=vocab, pos=int(self.rel_pos))
            if self._dsx_trainer is not None:
                self._dsx_trainer.close()
            object.__setattr__(self, "_dsx_trainer", Fs2EncTrainStep(cfg))
        return self._dsx_trainer

    # -- library handle ---------------------------------------------------------------------------
    _lib_create, _lib_load, _lib_destroy = lib.dsx_fs2enc_create, lib.dsx_fs2enc_load, lib.dsx_fs2enc_destroy

    def _config(self):
        self._cfg.vocab = self.embed_tokens.num_embeddings
        return self._cfg

    def _params(self, sd, t, arr):
        return _capi.Fs2EncParams(stack=fs2dec_params(self.num_layers, self.padding, t, arr, alpha=False),
                                  embed_w=t("embed_tokens.weight"))

    def forward(self, txt_tokens):
        """txt_tokens [B, T] (0 = padding) -> encoder_out [B, T, hidden_size] fp32 (tts_modules.py:328-337)."""
        if self.rel_pos:
            raise DsxError("unsupported FastSpeech2 encoder configuration: FastspeechEncoder with rel_pos adds "
                           "RelPositionalEncoding(txt_tokens), which the reference itself cannot run; rel_pos is the "
                           "MIDI encoder's")
        return self._run(txt_tokens, ())

    def _run(self, txt_tokens, addends):
        train = self.training and self._dsx_train and torch.is_grad_enabled()
        if not train:
            _eval_only(self, self._what)
        if txt_tokens is None or txt_tokens.dim() != 2 or txt_tokens.dtype.is_floating_point:
            raise DsxError(f"txt_tokens must be integer [B, T] (got {None if txt_tokens is None else tuple(txt_tokens.shape)})")
        _need_cuda(txt_tokens)
        dev = txt_tokens.device
        B, T = txt_tokens.shape
        H = self.hidden_size
        adds = []
        for a in addends:
            if a is None or (not isinstance(a, torch.Tensor) and a == 0):   # FastSpeech2MIDI passes 0 for a missing one
                adds.append(None)
                continue
            _need_cuda(a)
            try:
                a.expand(B, T, H)
            except RuntimeError:
                raise DsxError(f"an embedding addend must broadcast to [B, T, {H}] = [{B}, {T}, {H}] "
                               f"(got {tuple(a.shape)})") from None
            adds.append(a)
        out = torch.empty((B, T, H), device=dev, dtype=torch.float32)
        if B == 0 or T == 0:
            return out
        tok = txt_tokens.long().contiguous()
        lo, hi = torch.stack(torch.aminmax(tok)).tolist()      # one copy to the host, as nn.Embedding's own check
        V = self.embed_tokens.num_embeddings
        if lo < 0 or hi >= V:
            raise DsxError(f"txt_tokens must be in [0, {V}) (got ids from {lo} to {hi})")
        if self.rel_pos:
            self._rel_len = max(self._rel_len, T)               # extend_pe keeps the longest table (:23-29)
        if train:
            from .fs2enctrain import fs2enc_train_forward
            return fs2enc_train_forward(self, tok, adds + [None] * (3 - len(adds)))
        adds = [None if a is None else a.float().expand(B, T, H) for a in adds]
        hnd = self._ensure(dev)
        ptrs = (ctypes.c_void_p * 3)(*[a.data_ptr() if a is not None else None for a in adds + [None] * (3 - len(adds))])
        strides = (_capi.Strides * 3)(*[_strides_bct(a, (0, 2, 1)) if a is not None else _capi.Strides()
                                        for a in adds + [None] * (3 - len(adds))])
        with torch.cuda.device(dev):
            check(lib.dsx_fs2enc_forward(hnd, _ptr(tok), B, T, ptrs, strides, self._rel_len, _ptr(out), _stream(dev)),
                  "dsx_fs2enc_forward")
        return out


class FastspeechMIDIEncoder(FastspeechEncoder):
    _what = "FastSpeech2 MIDI encoder"

    def forward(self, txt_tokens, midi_embedding, midi_dur_embedding, slur_embedding):
        """modules/diffsinger_midi/fs2.py:26-36: x = sqrt(H) E[txt_tokens] + midi_embedding + midi_dur_embedding +
        slur_embedding (each [B, T, H] or 0), then the position term and the FFTBlocks -> [B, T, hidden_size] fp32."""
        return self._run(txt_tokens, (midi_embedding, midi_dur_embedding, slur_embedding))


def _durpred_config(idim, n_layers, n_chans, kernel_size, offset, padding):
    idim, L, C, k = int(idim), int(n_layers), int(n_chans), int(kernel_size)
    problems = []
    for name, v in (("idim", idim), ("n_chans", C)):
        if not (16 <= v <= 256 and v % 16 == 0):
            problems.append(f"{name} = {v} (a multiple of 16 in [16, 256])")
    if not 1 <= L <= 16:
        problems.append(f"n_layers = {L} (1..16)")
    if padding not in _PADDING:
        problems.append(f"padding = {padding!r} ('SAME' or 'LEFT')")
    if not 1 <= k <= 31 or (padding == 'SAME' and k % 2 == 0):
        problems.append(f"kernel_size = {k} (odd for 'SAME', <= 31)")
    if not math.isfinite(float(offset)):
        problems.append(f"offset = {offset}")
    if problems:
        raise DsxError("unsupported DurationPredictor configuration: " + "; ".join(problems))
    return _capi.DurPredConfig(idim=idim, chans=C, layers=L, kernel=k, padding=_PADDING[padding], offset=float(offset))


class DurationPredictor(PackedModule):
    def __init__(self, idim, n_layers=2, n_chans=384, kernel_size=3, dropout_rate=0.1, offset=1.0, padding='SAME', *,
                 hparams=None, train=None):
        super().__init__()
        hp = _get_hparams(hparams)
        if hp['dur_loss'] != 'mse':
            raise DsxError(f"unsupported DurationPredictor configuration: dur_loss = {hp['dur_loss']!r} (only 'mse', "
                           "the one out2dur implements)")
        self._cfg = _durpred_config(idim, n_layers, n_chans, kernel_size, offset, padding)
        self.offset, self.kernel_size, self.padding = offset, kernel_size, padding
        self.dropout_rate = float(dropout_rate)      # identity in eval mode; the training step's p under dsx_train
        self._dsx_train = bool(train if train is not None else hp.get("dsx_train", False))
        self._dsx_trainer = None
        self.conv = nn.ModuleList()
        for idx in range(n_layers):                                          # tts_modules.py:82-93
            in_chans = idim if idx == 0 else n_chans
            self.conv += [nn.Sequential(
                nn.ConstantPad1d(((kernel_size - 1) // 2, (kernel_size - 1) // 2) if padding == 'SAME'
                                 else (kernel_size - 1, 0), 0),
                nn.Conv1d(in_chans, n_chans, kernel_size, stride=1, padding=0),
                nn.ReLU(),
                LayerNorm(n_chans, dim=1),
                nn.Dropout(dropout_rate))]
        self.linear = nn.Linear(n_chans, 1)

    _lib_create, _lib_load, _lib_destroy = lib.dsx_durpred_create, lib.dsx_durpred_load, lib.dsx_durpred_destroy

    def __getstate__(self):
        # the library handles are ctypes pointers: copies (EMA deepcopy, torch.save of the module) make their own
        state = self.__dict__.copy()
        state["_dsx"], state["_wkey"], state["_keep"] = None, None, None
        state["_dsx_trainer"] = None
        return state

    def _dsx_train_step(self):
        if self._dsx_trainer is None:
            from .durtrain import DurTrainStep
            object.__setattr__(self, "_dsx_trainer", DurTrainStep(self._cfg))
        return self._dsx_trainer

    def _config(self):
        return self._cfg

    def _params(self, sd, t, arr):
        n = self._cfg.layers
        return _capi.DurPredParams(conv_w=arr([f"conv.{i}.1.weight" for i in range(n)]),
                                   conv_b=arr([f"conv.{i}.1.bias" for i in range(n)]),
                                   ln_w=arr([f"conv.{i}.3.weight" for i in range(n)]),
                                   ln_b=arr([f"conv.{i}.3.bias" for i in range(n)]),
                                   linear_w=t("linear.weight"), linear_b=t("linear.bias"))

    def _run(self, xs, x_masks, with_dur):
        train = self.training and self._dsx_train and torch.is_grad_enabled() and not with_dur
        if not train:
            _eval_only(self, "DurationPredictor")
        if xs is None or xs.dim() != 3 or xs.shape[-1] != self._cfg.idim:
            raise DsxError(f"xs must be [B, T, {self._cfg.idim}] (got {None if xs is None else tuple(xs.shape)})")
        if x_masks is None or tuple(x_masks.shape) != tuple(xs.shape[:2]):
            raise DsxError("x_masks must be the [B, T] padding mask (the reference needs it too)")
        _need_cuda(xs, x_masks)
        if train:
            from .durtrain import durpred_train_forward
            return durpred_train_forward(self, xs, x_masks), None
        dev = xs.device
        B, T, _ = xs.shape
        out = torch.empty((B, T), device=dev, dtype=torch.float32)
        dur = torch.empty((B, T), device=dev, dtype=torch.int64) if with_dur else None
        if B > 0 and T > 0:
            hnd = self._ensure(dev)
            xf = xs.float()
            mask = x_masks.to(torch.uint8).contiguous()
            with torch.cuda.device(dev):
                check(lib.dsx_durpred_forward(hnd, _ptr(xf), _strides_bct(xf, (0, 2, 1)), _ptr(mask), B, T, _ptr(out),
                                              _ptr(dur), _stream(dev)), "dsx_durpred_forward")
        return out, dur

    def forward(self, xs, x_masks=None):
        """xs [B, T, idim], x_masks [B, T] (True = padding) -> the log-domain durations [B, T] (tts_modules.py:131-139)."""
        return self._run(xs, x_masks, False)[0]

    def inference(self, xs, x_masks=None):
        """-> (dur [B, T] int64, xs [B, T, 1]) (tts_modules.py:141-151, out2dur :119-129)."""
        out, dur = self._run(xs, x_masks, True)
        return dur, out[:, :, None]


class LengthRegulator(nn.Module):
    def __init__(self, pad_value=0.0):
        super().__init__()
        self.pad_value = pad_value

    def forward(self, dur, dur_padding=None, alpha=1.0):
        """dur [B, T_txt] integer durations, dur_padding [B, T_txt] (True = padding) or None, alpha > 0 ->
        mel2ph [B, T_mel] int64, T_mel = max over utterances of sum(round(dur * alpha) * !padding)
        (tts_modules.py:159-189).  Reads T_mel and the negative-duration check in one copy to the host."""
        if not alpha > 0:
            raise DsxError(f"alpha must be positive (got {alpha})")
        if dur is None or dur.dim() != 2 or dur.dtype.is_floating_point or dur.dtype.is_complex:
            raise DsxError("dur must be integer [B, T_txt] (DurationPredictor.inference's dur)")
        if dur_padding is not None and tuple(dur_padding.shape) != tuple(dur.shape):
            raise DsxError("dur_padding must have dur's shape [B, T_txt]")
        _need_cuda(dur, dur_padding)
        dev = dur.device
        B, T = dur.shape
        if B == 0 or T == 0:
            return torch.zeros((B, 0), device=dev, dtype=torch.int64)
        d = dur.long().contiguous()
        pad = dur_padding.to(torch.uint8).contiguous() if dur_padding is not None else None
        cum = torch.empty_like(d)
        totals = torch.empty(B + 1, device=dev, dtype=torch.int64)
        with torch.cuda.device(dev):
            check(lib.dsx_length_totals(_ptr(d), _ptr(pad), B, T, float(alpha), _ptr(cum), _ptr(totals), _stream(dev)),
                  "dsx_length_totals")
            tot = totals.tolist()
            if tot[B]:
                raise DsxError("LengthRegulator: negative durations")
            T_mel = max(tot[:B])
            mel2ph = torch.empty((B, T_mel), device=dev, dtype=torch.int64)
            check(lib.dsx_length_regulate(_ptr(cum), _ptr(totals), B, T, T_mel, _ptr(mel2ph), _stream(dev)),
                  "dsx_length_regulate")
        return mel2ph
