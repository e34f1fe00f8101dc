"""FastSpeech2's pitch and energy predictors whose forward runs the sm_90a kernels of libdsx.so (dsx_pitchpred_* and
dsx_pitchpred_train_* in include/dsx.h).

``PitchPredictor(idim, n_layers, n_chans, odim, kernel_size, dropout_rate, padding, *, hparams=None, train=None)`` and
``EnergyPredictor`` (the same class) keep the reference's constructor and state dict (modules/fastspeech/tts_modules.py:
192-240): ``conv.i.1.*``, ``conv.i.3.*``, ``linear.*``, ``pos_embed_alpha`` and ``embed_positions._float_tensor``, so a
FastSpeech2 checkpoint loads with ``strict=True``.  The module only holds the parameters: in eval mode ``forward`` packs
them into the library (once per storage and version) and runs there.  Under the ``dsx_train`` opt-in (hparams key or
``train=`` keyword), a training-mode forward under autograd runs the sm_90a training step instead (dropout p = its
``dropout_rate``), through a ``torch.autograd.Function`` that gives ordinary ``.grad`` tensors for every parameter,
``pos_embed_alpha`` included, and for its input.  There is no eager or CPU path: a CPU tensor raises ``DsxError``, and so
does training without the opt-in.  ``FastSpeech2.add_pitch``'s ``predictor_grad`` scaling of the input, ``cwt2f0``, the
CWT ``Linear`` in front of the predictor and the losses stay the caller's PyTorch code.
"""
import ctypes

import torch
import torch.nn as nn

from . import _capi
from ._capi import DsxError, check, lib
from .fs2train import draw_seed
from .modules import _get_hparams
from .pitch import LayerNorm, SinusoidalPositionalEmbedding
from .sampler import PackedModule, _need_cuda, _ptr, _stream

_PADDING = {'SAME': 0, 'LEFT': 1}


def param_names(L):
    """Every PitchPredictor parameter name, in the order the autograd function takes them."""
    out = []
    for fmt in ("conv.{}.1.weight", "conv.{}.1.bias", "conv.{}.3.weight", "conv.{}.3.bias"):
        out += [fmt.format(i) for i in range(L)]
    return out + ["linear.weight", "linear.bias", "pos_embed_alpha"]


def _pitchpred_config(idim, n_layers, n_chans, odim, kernel_size, padding):
    idim, L, C, od, k = int(idim), int(n_layers), int(n_chans), int(odim), int(kernel_size)
    problems = []
    for name, v in (("idim", idim), ("n_chans", C)):
        if not (16 <= v <= 256 and v % 16 == 0):
            problems.append(f"{name} = {v} (a multiple of 16 in [16, 256])")
    if not 1 <= L <= 16:
        problems.append(f"n_layers = {L} (1..16)")
    if not 1 <= od <= 16:
        problems.append(f"odim = {od} (1..16)")
    if padding not in _PADDING:
        problems.append(f"padding = {padding!r} ('SAME' or 'LEFT')")
    if not 1 <= k <= 31 or (padding == 'SAME' and k % 2 == 0):
        problems.append(f"kernel_size = {k} (odd for 'SAME', <= 31)")
    if problems:
        raise DsxError("unsupported PitchPredictor configuration: " + "; ".join(problems))
    return _capi.PitchPredConfig(idim=idim, chans=C, layers=L, kernel=k, padding=_PADDING[padding], odim=od)


class PitchPredictor(PackedModule):
    _what = "PitchPredictor"

    def __init__(self, idim, n_layers=5, n_chans=384, odim=2, kernel_size=5, dropout_rate=0.1, padding='SAME', *,
                 hparams=None, train=None):
        super().__init__()
        self._cfg = _pitchpred_config(idim, n_layers, n_chans, odim, kernel_size, padding)
        self.kernel_size, self.padding = kernel_size, padding
        self.dropout_rate = float(dropout_rate)      # identity in eval mode; the training step's p under dsx_train
        if train is None:
            train = _get_hparams(hparams).get("dsx_train", False)
        self._dsx_train = bool(train)
        self._dsx_trainer = None
        self.conv = nn.ModuleList()
        for idx in range(n_layers):                                          # tts_modules.py:205-216
            self.conv += [nn.Sequential(
                nn.ConstantPad1d(((kernel_size - 1) // 2, (kernel_size - 1) // 2) if padding == 'SAME'
                                 else (kernel_size - 1, 0), 0),
                nn.Conv1d(idim if idx == 0 else n_chans, n_chans, kernel_size, stride=1, padding=0),
                nn.ReLU(),
                LayerNorm(n_chans, dim=1),
                nn.Dropout(dropout_rate))]
        self.linear = nn.Linear(n_chans, odim)
        self.embed_positions = SinusoidalPositionalEmbedding(idim, 0)
        self.pos_embed_alpha = nn.Parameter(torch.Tensor([1]))

    _lib_create, _lib_load, _lib_destroy = lib.dsx_pitchpred_create, lib.dsx_pitchpred_load, lib.dsx_pitchpred_destroy

    def __getstate__(self):
        # the library handles are ctypes pointers: copies (EMA deepcopy, torch.save of the module) make their own
        state = self.__dict__.copy()
        state["_dsx"], state["_wkey"], state["_keep"] = None, None, None
        state["_dsx_trainer"] = None
        return state

    def _dsx_train_step(self):
        if self._dsx_trainer is None:
            object.__setattr__(self, "_dsx_trainer", PitchTrainStep(self._cfg))
        return self._dsx_trainer

    def _config(self):
        return self._cfg

    def _params(self, sd, t, arr):
        n = self._cfg.layers
        return _capi.PitchPredParams(conv_w=arr([f"conv.{i}.1.weight" for i in range(n)]),
                                     conv_b=arr([f"conv.{i}.1.bias" for i in range(n)]),
                                     ln_w=arr([f"conv.{i}.3.weight" for i in range(n)]),
                                     ln_b=arr([f"conv.{i}.3.bias" for i in range(n)]),
                                     linear_w=t("linear.weight"), linear_b=t("linear.bias"),
                                     pos_embed_alpha=t("pos_embed_alpha"))

    def forward(self, xs):
        """xs [B, T, idim] -> [B, T, odim] fp32 (tts_modules.py:222-235).  The positions count the frames whose channel 0
        is nonzero, as make_positions(xs[..., 0], 0) does."""
        train = self.training and self._dsx_train and torch.is_grad_enabled()
        if self.training and not train:
            raise DsxError(f"the dsx {self._what} runs in eval mode only (call .eval()), or in training under the "
                           "dsx_train opt-in (hparams key or train=True) with autograd enabled")
        if xs is None or xs.dim() != 3 or xs.shape[-1] != self._cfg.idim:
            raise DsxError(f"xs must be [B, T, {self._cfg.idim}] (got {None if xs is None else tuple(xs.shape)})")
        _need_cuda(xs)
        if train:
            return pitchpred_train_forward(self, xs)
        dev = xs.device
        B, T, _ = xs.shape
        out = torch.empty((B, T, self._cfg.odim), device=dev, dtype=torch.float32)
        if B > 0 and T > 0:
            hnd = self._ensure(dev)
            xf = xs.float().contiguous()
            with torch.cuda.device(dev):
                check(lib.dsx_pitchpred_forward(hnd, _ptr(xf), B, T, _ptr(out), _stream(dev)), "dsx_pitchpred_forward")
        return out


class EnergyPredictor(PitchPredictor):
    _what = "EnergyPredictor"


# ---- training step ---------------------------------------------------------------------------------------------------
def _struct(tensors, L, keep):
    """PitchPredParams of a list of fp32 contiguous CUDA tensors in param_names order; host arrays go to `keep`."""
    it = iter(tensors)
    kw = {}
    for f in ("conv_w", "conv_b", "ln_w", "ln_b"):
        a = (ctypes.c_void_p * L)(*[next(it).data_ptr() for _ in range(L)])
        keep.append(a)
        kw[f] = ctypes.cast(a, ctypes.POINTER(ctypes.c_void_p))
    kw["linear_w"], kw["linear_b"], kw["pos_embed_alpha"] = (next(it).data_ptr() for _ in range(3))
    return _capi.PitchPredParams(**kw)


class PitchTrainStep:
    """One dsx_pitchpred_train handle per (module, device)."""

    def __init__(self, cfg):
        self.cfg = cfg
        self._h = None
        self._device = None

    def close(self):
        if self._h is not None:
            lib.dsx_pitchpred_train_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def handle(self, device):
        if self._h is not None and self._device != device:
            self.close()
        if self._h is None:
            h = ctypes.c_void_p()
            check(lib.dsx_pitchpred_train_create(device.index if device.index is not None else torch.cuda.current_device(),
                                                 ctypes.byref(self.cfg), ctypes.byref(h)), "dsx_pitchpred_train_create")
            self._h, self._device = h, device
        return self._h

    def tape_bytes(self, device, B, T):
        n = ctypes.c_size_t()
        check(lib.dsx_pitchpred_train_tape_bytes(self.handle(device), B, T, ctypes.byref(n)),
              "dsx_pitchpred_train_tape_bytes")
        return n.value

    def workspace(self, device, B, T):
        """Scratch of one call, from PyTorch's allocator (released to its cache when the call's tensor dies)."""
        n = ctypes.c_size_t()
        check(lib.dsx_pitchpred_train_workspace_bytes(self.handle(device), B, T, ctypes.byref(n)),
              "dsx_pitchpred_train_workspace_bytes")
        return torch.empty(n.value, dtype=torch.uint8, device=device)

    def forward(self, params, x, p, seed):
        """out [B, T, odim] and the tape (uint8 CUDA tensor) of one forward.  params: fp32 CUDA tensors in param_names
        order; x: fp32 [B, T, idim] contiguous."""
        dev = x.device
        h = self.handle(dev)
        B, T, _ = x.shape
        keep = []
        w = _struct(params, self.cfg.layers, keep)
        tape = torch.empty(self.tape_bytes(dev, B, T), dtype=torch.uint8, device=dev)
        out = torch.empty((B, T, self.cfg.odim), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):     # the forward uses no workspace
            check(lib.dsx_pitchpred_train_forward(h, ctypes.byref(w), _ptr(x), B, T, float(p), int(seed), _ptr(tape),
                                                  tape.numel(), None, 0, _ptr(out), _stream(dev)),
                  "dsx_pitchpred_train_forward")
        return out, tape

    def backward(self, params, tape, d_out, B, T, want_x=True):
        """Gradients in param_names order, and d_x [B, T, idim] (or None)."""
        dev = d_out.device
        h = self.handle(dev)
        keep = []
        w = _struct(params, self.cfg.layers, keep)
        grads = [torch.empty_like(v) for v in params]
        g = _struct(grads, self.cfg.layers, keep)
        d_out = d_out.float().contiguous()
        d_x = torch.empty((B, T, self.cfg.idim), dtype=torch.float32, device=dev) if want_x else None
        ws = self.workspace(dev, B, T)
        with torch.cuda.device(dev):
            check(lib.dsx_pitchpred_train_backward(h, ctypes.byref(w), _ptr(tape), _ptr(d_out), ctypes.byref(g),
                                                   _ptr(d_x), B, T, _ptr(ws), ws.numel(), _stream(dev)),
                  "dsx_pitchpred_train_backward")
        return grads, d_x

    def masks(self, device, seed, p, B, T):
        """The n_layers keep masks (bool CUDA tensors [B, T, chans]) a forward with (seed, p) draws."""
        out = [torch.empty((B, T, self.cfg.chans), dtype=torch.uint8, device=device) for _ in range(self.cfg.layers)]
        arr = (ctypes.c_void_p * len(out))(*[m.data_ptr() for m in out])
        with torch.cuda.device(device):
            check(lib.dsx_pitchpred_train_masks(self.handle(device), int(seed), float(p), B, T, arr, _stream(device)),
                  "dsx_pitchpred_train_masks")
        return [m.bool() for m in out]


class PitchTrainFn(torch.autograd.Function):
    """PitchPredictor.forward in training with the parameters as explicit inputs: apply(step, p, seed, x, *params)."""

    @staticmethod
    def forward(ctx, step, p, seed, x, *params):
        out, tape = step.forward(params, x, p, seed)
        ctx.step, ctx.tape = step, tape
        ctx.BT = (x.shape[0], x.shape[1])
        ctx.save_for_backward(*params)     # the version check: an in-place update before backward raises
        return out

    @staticmethod
    def backward(ctx, g):
        if torch.is_grad_enabled():
            raise DsxError("dsx_train has no double backward (create_graph=True through the pitch predictor's training "
                           "step)")
        return _backward(ctx, g)


@torch.autograd.function.once_differentiable
def _backward(ctx, g):
    B, T = ctx.BT
    grads, d_x = ctx.step.backward(list(ctx.saved_tensors), ctx.tape, g, B, T, want_x=ctx.needs_input_grad[3])
    return (None, None, None, d_x) + tuple(grads)


def pitchpred_train_forward(pp, xs):
    """PitchPredictor.forward in training under the dsx_train opt-in: dropout p = the module's dropout_rate.
    xs: CUDA [B, T, idim]."""
    named = dict(pp.named_parameters())
    params = [named[n] for n in param_names(pp._cfg.layers)]
    _need_cuda(xs, *params)
    if any(p.dtype != torch.float32 for p in params):
        raise DsxError("dsx_train runs fp32 pitch predictor parameters")
    if any(not p.is_contiguous() for p in params):
        raise DsxError("dsx_train needs contiguous pitch predictor parameters")
    if xs.requires_grad and xs.dtype != torch.float32:
        raise DsxError("dsx_train needs an fp32 xs where it requires grad (its gradient is fp32)")
    B, T, _ = xs.shape
    if B == 0 or T == 0:      # nothing to run: an empty output, as in eval mode
        return xs.float()[..., :1].expand(B, T, pp._cfg.odim) * 0.0
    return PitchTrainFn.apply(pp._dsx_train_step(), float(pp.dropout_rate), draw_seed(), xs.float().contiguous(),
                              *params)
