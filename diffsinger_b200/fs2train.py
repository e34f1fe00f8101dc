"""FastSpeech2 decoder training step on libdsx: the forward with dropout and a saved tape, and the backward
(include/dsx.h, dsx_fs2dec_train_*), wrapped in a ``torch.autograd.Function`` so that ``FastspeechDecoder`` under
``dsx_train`` gives ordinary ``.grad`` tensors to DDP and any optimizer, and its gradient with respect to decoder_inp
flows back into the encoder.  ``mel_out`` and the loss stay in the caller's PyTorch code."""
import ctypes

import torch

from . import _capi
from ._capi import DsxError, check, lib
from .sampler import _need_cuda, _ptr, _stream, _strides_bct

# Fs2DecParams field -> name under layers.{i}.op. (per layer) or at the top of the decoder
_LAYER = (("ln1_w", "layer_norm1.weight"), ("ln1_b", "layer_norm1.bias"), ("in_proj_w", "self_attn.in_proj_weight"),
          ("out_proj_w", "self_attn.out_proj.weight"), ("ln2_w", "layer_norm2.weight"), ("ln2_b", "layer_norm2.bias"),
          ("ffn1_w", "{ffn1}weight"), ("ffn1_b", "{ffn1}bias"), ("ffn2_w", "ffn.ffn_2.weight"),
          ("ffn2_b", "ffn.ffn_2.bias"))
_TOP = (("ln_w", "layer_norm.weight"), ("ln_b", "layer_norm.bias"), ("pos_embed_alpha", "pos_embed_alpha"))


def param_names(L, padding):
    """Every decoder parameter name, in the order the autograd function takes them."""
    ffn1 = "ffn.ffn_1." if padding == 'SAME' else "ffn.ffn_1.1."
    out = []
    for _, n in _LAYER:
        out += [f"layers.{i}.op." + n.format(ffn1=ffn1) for i in range(L)]
    return out + [n for _, n in _TOP]


def _struct(tensors, L, keep):
    """Fs2DecParams of a list of fp32 contiguous CUDA tensors in param_names order; host arrays go to `keep`."""
    it = iter(tensors)
    kw = {}
    for f, _ in _LAYER:
        a = (ctypes.c_void_p * L)(*[next(it).data_ptr() for _ in range(L)])
        keep.append(a)
        kw[f] = ctypes.cast(a, ctypes.POINTER(ctypes.c_void_p))
    for f, _ in _TOP:
        kw[f] = next(it).data_ptr()
    return _capi.Fs2DecParams(**kw)


class Fs2DecTrainStep:
    """One dsx_fs2dec_train handle per (module, device)."""

    def __init__(self, cfg):
        self.cfg = cfg
        self._h = None
        self._device = None

    def close(self):
        if self._h is not None:
            lib.dsx_fs2dec_train_destroy(self._h)
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
            check(lib.dsx_fs2dec_train_create(device.index if device.index is not None else torch.cuda.current_device(),
                                              ctypes.byref(self.cfg), ctypes.byref(h)), "dsx_fs2dec_train_create")
            self._h, self._device = h, device
        return self._h

    def tape_bytes(self, device, B, T):
        n = ctypes.c_size_t()
        check(lib.dsx_fs2dec_train_tape_bytes(self.handle(device), B, T, ctypes.byref(n)), "dsx_fs2dec_train_tape_bytes")
        return n.value

    def workspace(self, device, B, T):
        """Scratch of one call, from PyTorch's allocator (released to its cache when the call's tensor dies)."""
        n = ctypes.c_size_t()
        check(lib.dsx_fs2dec_train_workspace_bytes(self.handle(device), B, T, ctypes.byref(n)),
              "dsx_fs2dec_train_workspace_bytes")
        return torch.empty(n.value, dtype=torch.uint8, device=device)

    def forward(self, params, x, p, seed):
        """out [B, T, H] and the tape (uint8 CUDA tensor) of one forward; params: fp32 CUDA tensors in param_names
        order."""
        dev = x.device
        h = self.handle(dev)
        B, T, H = x.shape
        keep = []
        w = _struct(params, self.cfg.layers, keep)
        tape = torch.empty(self.tape_bytes(dev, B, T), dtype=torch.uint8, device=dev)
        out = torch.empty((B, T, H), dtype=torch.float32, device=dev)
        ws = self.workspace(dev, B, T)
        with torch.cuda.device(dev):
            check(lib.dsx_fs2dec_train_forward(h, ctypes.byref(w), _ptr(x), _strides_bct(x, (0, 2, 1)), B, T, float(p),
                                               int(seed), _ptr(tape), tape.numel(), _ptr(ws), ws.numel(), _ptr(out),
                                               _stream(dev)), "dsx_fs2dec_train_forward")
        return out, tape

    def backward(self, params, tape, d_out, B, T, want_x=True):
        """Gradients in param_names order, and d_x [B, T, H] (or None)."""
        dev = d_out.device
        h = self.handle(dev)
        keep = []
        w = _struct(params, self.cfg.layers, keep)
        grads = [torch.empty_like(v) for v in params]
        g = _struct(grads, self.cfg.layers, keep)
        d_out = d_out.float().contiguous()
        d_x = torch.empty((B, T, self.cfg.hidden), dtype=torch.float32, device=dev) if want_x else None
        ws = self.workspace(dev, B, T)
        with torch.cuda.device(dev):
            check(lib.dsx_fs2dec_train_backward(h, ctypes.byref(w), _ptr(tape), _ptr(d_out), ctypes.byref(g), _ptr(d_x),
                                                B, T, _ptr(ws), ws.numel(), _stream(dev)), "dsx_fs2dec_train_backward")
        return grads, d_x

    def masks(self, device, seed, p, B, T):
        """The 1 + 3 L keep masks (bool CUDA tensors [B, T, H], sites 2 + 3 i [B, T, 4H]) a forward with (seed, p) draws."""
        H, L = self.cfg.hidden, self.cfg.layers
        out = [torch.empty((B, T, 4 * H if s > 0 and s % 3 == 2 else H), dtype=torch.uint8, device=device)
               for s in range(1 + 3 * L)]
        arr = (ctypes.c_void_p * len(out))(*[m.data_ptr() for m in out])
        with torch.cuda.device(device):
            check(lib.dsx_fs2dec_train_masks(self.handle(device), int(seed), float(p), B, T, arr, _stream(device)),
                  "dsx_fs2dec_train_masks")
        return [m.bool() for m in out]


class Fs2DecTrainFn(torch.autograd.Function):
    """out = FFTBlocks(x) in training with the parameters as explicit inputs: apply(step, p, seed, x, *params)."""

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
            raise DsxError("dsx_train has no double backward (create_graph=True through the FastSpeech2 decoder's "
                           "training step)")
        return _backward(ctx, g)


@torch.autograd.function.once_differentiable
def _backward(ctx, g):
    B, T = ctx.BT
    grads, d_x = ctx.step.backward(list(ctx.saved_tensors), ctx.tape, g, B, T, want_x=ctx.needs_input_grad[3])
    return (None, None, None, d_x) + tuple(grads)


def draw_seed():
    """A 64-bit seed from torch's default CPU generator, so torch.manual_seed reproduces a run."""
    return int(torch.empty((), dtype=torch.int64).random_().item())


def fs2dec_train_forward(dec, x):
    """FFTBlocks.forward of the decoder in training under the dsx_train opt-in: dropout p = hparams['dropout']."""
    named = dict(dec.named_parameters())
    params = [named[n] for n in param_names(dec.num_layers, dec.padding)]
    _need_cuda(x, *params)
    if any(p.dtype != torch.float32 for p in params):
        raise DsxError("dsx_train runs fp32 decoder parameters")
    if any(not p.is_contiguous() for p in params):
        raise DsxError("dsx_train needs contiguous decoder parameters")
    if x.shape[0] == 0 or x.shape[1] == 0:      # nothing to run: an empty output, as in eval mode
        return x.float() * 0.0
    return Fs2DecTrainFn.apply(dec._dsx_train_step(), float(dec.dropout), draw_seed(), x.float(), *params)
