"""FastSpeech2 encoder training step on libdsx: the forward with dropout and a saved tape, and the backward
(include/dsx.h, dsx_fs2enc_train_*), wrapped in a ``torch.autograd.Function`` so that ``FastspeechEncoder`` /
``FastspeechMIDIEncoder`` under ``dsx_train`` give ordinary ``.grad`` tensors to DDP and any optimizer: every stack
parameter, ``embed_tokens.weight``, and the MIDI addends, whose embeddings stay in the caller's PyTorch code."""
import ctypes

import torch

from . import _capi
from ._capi import DsxError, check, lib
from .fs2train import _LAYER, Fs2DecTrainStep, draw_seed
from .fs2train import param_names as _stack_names
from .sampler import _need_cuda, _ptr, _stream, _strides_bct


def param_names(L, padding):
    """Every encoder parameter name, in the order the autograd function takes them."""
    return _stack_names(L, padding)[:-1] + ["embed_tokens.weight"]    # the encoder's FFTBlocks have no pos_embed_alpha


def _struct(tensors, L, keep):
    """Fs2EncParams of a list of fp32 contiguous CUDA tensors in param_names order; host arrays go to `keep`."""
    it = iter(tensors)
    kw = {}
    for f, _ in _LAYER:
        a = (ctypes.c_void_p * L)(*[next(it).data_ptr() for _ in range(L)])
        keep.append(a)
        kw[f] = ctypes.cast(a, ctypes.POINTER(ctypes.c_void_p))
    kw["ln_w"], kw["ln_b"] = next(it).data_ptr(), next(it).data_ptr()
    return _capi.Fs2EncParams(stack=_capi.Fs2DecParams(**kw), embed_w=next(it).data_ptr())


class Fs2EncTrainStep:
    """One dsx_fs2enc_train handle per (module, device)."""

    def __init__(self, cfg):
        self.cfg = cfg
        self._h = None
        self._device = None
        self._masks = None

    def close(self):
        if self._h is not None:
            lib.dsx_fs2enc_train_destroy(self._h)
            self._h = None
        if self._masks is not None:
            self._masks.close()

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
            check(lib.dsx_fs2enc_train_create(device.index if device.index is not None else torch.cuda.current_device(),
                                              ctypes.byref(self.cfg), ctypes.byref(h)), "dsx_fs2enc_train_create")
            self._h, self._device = h, device
        return self._h

    def tape_bytes(self, device, B, T):
        n = ctypes.c_size_t()
        check(lib.dsx_fs2enc_train_tape_bytes(self.handle(device), B, T, ctypes.byref(n)), "dsx_fs2enc_train_tape_bytes")
        return n.value

    def workspace(self, device, B, T):
        """Scratch of one call, from PyTorch's allocator (released to its cache when the call's tensor dies)."""
        n = ctypes.c_size_t()
        check(lib.dsx_fs2enc_train_workspace_bytes(self.handle(device), B, T, ctypes.byref(n)),
              "dsx_fs2enc_train_workspace_bytes")
        return torch.empty(n.value, dtype=torch.uint8, device=device)

    def forward(self, params, tok, adds, rel_len, p, seed):
        """out [B, T, H] and the tape (uint8 CUDA tensor) of one forward.  params: fp32 CUDA tensors in param_names
        order; tok: int64 [B, T] contiguous; adds: three fp32 tensors broadcasting to [B, T, H], or None."""
        dev = tok.device
        h = self.handle(dev)
        B, T = tok.shape
        H = self.cfg.stack.hidden
        keep = []
        w = _struct(params, self.cfg.stack.layers, keep)
        ptrs = (ctypes.c_void_p * 3)(*[a.data_ptr() if a is not None else None for a in adds])
        strides = (_capi.Strides * 3)(*[_strides_bct(a.expand(B, T, H), (0, 2, 1)) if a is not None
                                        else _capi.Strides() for a in adds])
        tape = torch.empty(self.tape_bytes(dev, B, T), dtype=torch.uint8, device=dev)
        out = torch.empty((B, T, H), dtype=torch.float32, device=dev)
        ws = self.workspace(dev, B, T)
        with torch.cuda.device(dev):
            check(lib.dsx_fs2enc_train_forward(h, ctypes.byref(w), _ptr(tok), B, T, ptrs, strides, int(rel_len),
                                               float(p), int(seed), _ptr(tape), tape.numel(), _ptr(ws), ws.numel(),
                                               _ptr(out), _stream(dev)), "dsx_fs2enc_train_forward")
        return out, tape

    def backward(self, params, tape, d_out, B, T, want_add=True):
        """Gradients in param_names order, and d_add [B, T, H] (or None): the gradient of each addend."""
        dev = d_out.device
        h = self.handle(dev)
        keep = []
        w = _struct(params, self.cfg.stack.layers, keep)
        grads = [torch.empty_like(v) for v in params]
        g = _struct(grads, self.cfg.stack.layers, keep)
        d_out = d_out.float().contiguous()
        d_add = torch.empty((B, T, self.cfg.stack.hidden), dtype=torch.float32, device=dev) if want_add else None
        ws = self.workspace(dev, B, T)
        with torch.cuda.device(dev):
            check(lib.dsx_fs2enc_train_backward(h, ctypes.byref(w), _ptr(tape), _ptr(d_out), ctypes.byref(g),
                                                _ptr(d_add), B, T, _ptr(ws), ws.numel(), _stream(dev)),
                  "dsx_fs2enc_train_backward")
        return grads, d_add

    def masks(self, device, seed, p, B, T):
        """The 1 + 3 L keep masks a forward with (seed, p) draws: the decoder step's on a handle of cfg.stack."""
        if self._masks is None:
            self._masks = Fs2DecTrainStep(self.cfg.stack)
        return self._masks.masks(device, seed, p, B, T)


class Fs2EncTrainFn(torch.autograd.Function):
    """out = the encoder in training with the parameters as explicit inputs:
    apply(step, p, seed, rel_len, tok, add0, add1, add2, *params), an addend None when absent."""

    @staticmethod
    def forward(ctx, step, p, seed, rel_len, tok, a0, a1, a2, *params):
        adds = (a0, a1, a2)
        out, tape = step.forward(params, tok, adds, rel_len, p, seed)
        ctx.step, ctx.tape = step, tape
        ctx.BT = tuple(tok.shape)
        ctx.add_shapes = [None if a is None else a.shape for a in adds]
        ctx.save_for_backward(*params)     # the version check: an in-place update before backward raises
        return out

    @staticmethod
    def backward(ctx, g):
        if torch.is_grad_enabled():
            raise DsxError("dsx_train has no double backward (create_graph=True through the FastSpeech2 encoder's "
                           "training step)")
        return _backward(ctx, g)


@torch.autograd.function.once_differentiable
def _backward(ctx, g):
    B, T = ctx.BT
    need = ctx.needs_input_grad[5:8]
    grads, d_add = ctx.step.backward(list(ctx.saved_tensors), ctx.tape, g, B, T, want_add=any(need))
    d_adds, used = [], False
    for n, shape in zip(need, ctx.add_shapes):
        if not n or shape is None:
            d_adds.append(None)
            continue
        d = d_add.sum_to_size(shape)
        if d.data_ptr() == d_add.data_ptr():     # two addends never share one gradient tensor
            d = d.clone() if used else d
            used = True
        d_adds.append(d)
    return (None, None, None, None, None) + tuple(d_adds) + tuple(grads)


def fs2enc_train_forward(enc, tok, adds):
    """The encoder's forward in training under the dsx_train opt-in: dropout p = hparams['dropout'].  tok: int64 [B, T]
    contiguous CUDA ids in [0, vocab); adds: the three addends (CUDA tensors broadcasting to [B, T, H], or None)."""
    named = dict(enc.named_parameters())
    params = [named[n] for n in param_names(enc.num_layers, enc.padding)]
    _need_cuda(*params)
    if any(p.dtype != torch.float32 for p in params):
        raise DsxError("dsx_train runs fp32 encoder parameters")
    if any(not p.is_contiguous() for p in params):
        raise DsxError("dsx_train needs contiguous encoder parameters")
    if any(a is not None and a.requires_grad and a.dtype != torch.float32 for a in adds):
        raise DsxError("dsx_train needs fp32 embedding addends where they require grad (their gradient is fp32)")
    adds = [None if a is None else a.float() for a in adds]
    return Fs2EncTrainFn.apply(enc._dsx_train_step(), float(enc.dropout), draw_seed(), enc._rel_len, tok, *adds,
                               *params)
