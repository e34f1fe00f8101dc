"""FastSpeech2 decoder whose forward runs the sm_90a kernels of libdsx.so (dsx_fs2dec_* in include/dsx.h).

``FastspeechDecoder(hidden_size=None, num_layers=None, kernel_size=None, num_heads=None, *, hparams=None)`` keeps the
reference's constructor, submodule names, parameter and buffer shapes (modules/fastspeech/tts_modules.py:251-357 with
modules/commons/common_layers.py:166-588), so the decoder of a FastSpeech2 checkpoint loads with ``strict=True``.  The
modules only hold the parameters: ``forward`` packs them into the library (once per storage and version, so again after
``load_state_dict`` or ``.to()``) and runs the whole decoder there.  There is no eager or CPU path: a CPU tensor raises
``DsxError``.  A module in training mode raises ``DsxError`` too, unless the ``dsx_train`` opt-in (hparams key or
``train=`` keyword) is set: then a training-mode forward under autograd runs the sm_90a training step of
``diffsinger_b200.fs2train`` (dropout p = hparams['dropout'], gradients for every parameter and for x).
"""
import torch
import torch.nn as nn

from . import _capi
from ._capi import DsxError, check, lib
from .modules import _get_hparams
from .pitch import SinusoidalPositionalEmbedding
from .sampler import PackedModule, _need_cuda, _ptr, _stream, _strides_bct

_PADDING = {'SAME': 0, 'LEFT': 1}
_ACT = {'gelu': 0, 'relu': 1}


class MultiheadAttention(nn.Module):
    """common_layers.py:166-234 with bias=False and self-attention: in_proj_weight [3H, H], out_proj without bias."""

    def __init__(self, embed_dim, num_heads):
        super().__init__()
        self.embed_dim, self.num_heads = embed_dim, num_heads
        self.in_proj_weight = nn.Parameter(torch.empty(3 * embed_dim, embed_dim))
        self.out_proj = nn.Linear(embed_dim, embed_dim, bias=False)
        nn.init.xavier_uniform_(self.in_proj_weight)
        nn.init.xavier_uniform_(self.out_proj.weight)


class TransformerFFNLayer(nn.Module):
    """common_layers.py:486-501: ffn_1 is a Conv1d ('SAME') or ConstantPad1d + Conv1d ('LEFT'), ffn_2 a Linear."""

    def __init__(self, hidden_size, filter_size, padding='SAME', kernel_size=1, act='gelu'):
        super().__init__()
        self.kernel_size, self.act = kernel_size, act
        if padding == 'SAME':
            self.ffn_1 = nn.Conv1d(hidden_size, filter_size, kernel_size, padding=kernel_size // 2)
        else:
            self.ffn_1 = nn.Sequential(nn.ConstantPad1d((kernel_size - 1, 0), 0.0),
                                       nn.Conv1d(hidden_size, filter_size, kernel_size))
        self.ffn_2 = nn.Linear(filter_size, hidden_size)
        nn.init.xavier_uniform_(self.ffn_2.weight)
        nn.init.constant_(self.ffn_2.bias, 0.)


class EncSALayer(nn.Module):
    """common_layers.py:542-562 with norm='ln' (LayerNorm eps 1e-5)."""

    def __init__(self, c, num_heads, kernel_size, padding, act='gelu'):
        super().__init__()
        self.layer_norm1 = nn.LayerNorm(c)
        self.self_attn = MultiheadAttention(c, num_heads)
        self.layer_norm2 = nn.LayerNorm(c)
        self.ffn = TransformerFFNLayer(c, 4 * c, kernel_size=kernel_size, padding=padding, act=act)


class TransformerEncoderLayer(nn.Module):
    """tts_modules.py:16-31 (the layer is held as ``op``)."""

    def __init__(self, hidden_size, kernel_size, num_heads, padding, act='gelu'):
        super().__init__()
        self.op = EncSALayer(hidden_size, num_heads, kernel_size, padding, act)


def _fs2dec_config(hidden_size, num_layers, kernel_size, num_heads, padding, act, prefix="dec", what="decoder"):
    """-> Fs2DecConfig, or DsxError for what the kernels do not run (prefix, what: the hparams' and the model's names)."""
    H, L, k, heads = int(hidden_size), int(num_layers), int(kernel_size), int(num_heads)
    problems = []
    if not (64 <= H <= 256 and H % 64 == 0):
        problems.append(f"hidden_size = {H} (a multiple of 64 in [64, 256])")
    if not 1 <= L <= 64:
        problems.append(f"{prefix}_layers = {L} (1..64)")
    if heads < 1 or H % heads or H // heads not in (64, 128):
        problems.append(f"num_heads = {heads} (hidden_size / num_heads must be 64 or 128)")
    if padding not in _PADDING:
        problems.append(f"ffn_padding = {padding!r} ('SAME' or 'LEFT')")
    if not 1 <= k <= 255 or (padding == 'SAME' and k % 2 == 0):
        problems.append(f"{prefix}_ffn_kernel_size = {k} (odd for 'SAME', <= 255)")
    if act not in _ACT:
        problems.append(f"ffn_act = {act!r} ('gelu' or 'relu')")
    if problems:
        raise DsxError(f"unsupported FastSpeech2 {what} configuration: " + "; ".join(problems))
    cfg = _capi.Fs2DecConfig()
    cfg.hidden, cfg.layers, cfg.kernel, cfg.heads = H, L, k, heads
    cfg.padding, cfg.act = _PADDING[padding], _ACT[act]
    return cfg


def fs2dec_params(num_layers, padding, t, arr, alpha=True):
    """Fs2DecParams of the FFTBlocks stack under the reference's state-dict names (t, arr: see PackedModule._ensure);
    alpha=False: a stack without pos_embed_alpha (the encoder's)."""
    ops = [f"layers.{i}.op" for i in range(num_layers)]
    ffn1 = ".ffn.ffn_1." if padding == 'SAME' else ".ffn.ffn_1.1."
    return _capi.Fs2DecParams(
        ln1_w=arr([o + ".layer_norm1.weight" for o in ops]), ln1_b=arr([o + ".layer_norm1.bias" for o in ops]),
        in_proj_w=arr([o + ".self_attn.in_proj_weight" for o in ops]),
        out_proj_w=arr([o + ".self_attn.out_proj.weight" for o in ops]),
        ln2_w=arr([o + ".layer_norm2.weight" for o in ops]), ln2_b=arr([o + ".layer_norm2.bias" for o in ops]),
        ffn1_w=arr([o + ffn1 + "weight" for o in ops]), ffn1_b=arr([o + ffn1 + "bias" for o in ops]),
        ffn2_w=arr([o + ".ffn.ffn_2.weight" for o in ops]), ffn2_b=arr([o + ".ffn.ffn_2.bias" for o in ops]),
        ln_w=t("layer_norm.weight"), ln_b=t("layer_norm.bias"), pos_embed_alpha=t("pos_embed_alpha") if alpha else None)


class FastspeechDecoder(PackedModule):
    def __init__(self, hidden_size=None, num_layers=None, kernel_size=None, num_heads=None, *, hparams=None, train=None):
        super().__init__()
        hp = _get_hparams(hparams)
        num_heads = hp['num_heads'] if num_heads is None else num_heads          # tts_modules.py:352-355
        hidden_size = hp['hidden_size'] if hidden_size is None else hidden_size
        kernel_size = hp['dec_ffn_kernel_size'] if kernel_size is None else kernel_size
        num_layers = hp['dec_layers'] if num_layers is None else num_layers
        padding, act = hp['ffn_padding'], hp['ffn_act']
        self._cfg = _fs2dec_config(hidden_size, num_layers, kernel_size, num_heads, padding, act)
        self.hidden_size, self.num_layers, self.num_heads = self._cfg.hidden, self._cfg.layers, self._cfg.heads
        self.kernel_size, self.padding, self.act = self._cfg.kernel, padding, act
        self.dropout = hp.get('dropout', 0.0)      # identity in eval mode; the training step's p under dsx_train
        self.padding_idx = 0
        self.pos_embed_alpha = nn.Parameter(torch.Tensor([1]))
        self.embed_positions = SinusoidalPositionalEmbedding(self.hidden_size, self.padding_idx)
        self.layers = nn.ModuleList([TransformerEncoderLayer(self.hidden_size, self.kernel_size, self.num_heads, padding, act)
                                     for _ in range(self.num_layers)])
        self.layer_norm = nn.LayerNorm(self.hidden_size)
        self._dsx_train = bool(train if train is not None else hp.get("dsx_train", False))
        self._dsx_trainer = None

    def __getstate__(self):
        # the library handles are ctypes pointers: copies (EMA deepcopy, torch.save of the module) make their own
        state = self.__dict__.copy()
        state["_dsx"], state["_wkey"], state["_keep"] = None, None, None
        state["_dsx_trainer"] = None
        return state

    def _dsx_train_step(self):
        if self._dsx_trainer is None:
            from .fs2train import Fs2DecTrainStep
            object.__setattr__(self, "_dsx_trainer", Fs2DecTrainStep(_fs2dec_config(
                self.hidden_size, self.num_layers, self.kernel_size, self.num_heads, self.padding, self.act)))
        return self._dsx_trainer

    # -- library handle ---------------------------------------------------------------------------
    _lib_create, _lib_load, _lib_destroy = lib.dsx_fs2dec_create, lib.dsx_fs2dec_load, lib.dsx_fs2dec_destroy

    def _config(self):
        return self._cfg

    def _params(self, sd, t, arr):
        return fs2dec_params(self.num_layers, self.padding, t, arr)

    def forward(self, x, padding_mask=None, attn_mask=None, return_hiddens=False):
        """x: decoder_inp [B, T, hidden_size] (any strides).  A frame whose channels are all 0 is padding.
        -> [B, T, hidden_size] fp32 (tts_modules.py:282-307)."""
        if padding_mask is not None or attn_mask is not None or return_hiddens:
            raise DsxError("the dsx FastSpeech2 decoder takes x only: padding_mask, attn_mask and return_hiddens are not "
                           "supported (the padding mask is derived from x, as at inference)")
        if x is None or x.dim() != 3 or x.shape[-1] != self.hidden_size:
            raise DsxError(f"x must be [B, T, {self.hidden_size}] (got {None if x is None else tuple(x.shape)})")
        if self.training and self._dsx_train and torch.is_grad_enabled():
            from .fs2train import fs2dec_train_forward
            return fs2dec_train_forward(self, x)
        if self.training:
            raise DsxError("the dsx FastSpeech2 decoder runs in eval mode only (call .eval()); training stays with the "
                           "reference's modules")
        _need_cuda(x)
        dev = x.device
        hnd = self._ensure(dev)
        B, T, H = x.shape
        xf = x.float()
        out = torch.empty((B, T, H), device=dev, dtype=torch.float32)
        if B > 0 and T > 0:
            with torch.cuda.device(dev):
                check(lib.dsx_fs2dec_forward(hnd, _ptr(xf), _strides_bct(xf, (0, 2, 1)), B, T, _ptr(out), _stream(dev)),
                      "dsx_fs2dec_forward")
        return out
