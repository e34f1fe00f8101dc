"""Duration predictor training step on libdsx: the forward with dropout and a saved tape, and the backward
(include/dsx.h, dsx_durpred_train_*), wrapped in a ``torch.autograd.Function`` so that ``DurationPredictor`` under
``dsx_train`` gives ordinary ``.grad`` tensors to DDP and any optimizer, and its gradient with respect to its input flows
back into the encoder (scaled by ``predictor_grad`` in ``FastSpeech2.add_dur``, which stays the caller's).  The duration
losses stay in the caller's PyTorch code."""
import ctypes

import torch

from . import _capi
from ._capi import DsxError, check, lib
from .fs2train import draw_seed
from .sampler import _need_cuda, _ptr, _stream, _strides_bct


def param_names(L):
    """Every DurationPredictor parameter name, in the order the autograd function takes them."""
    out = []
    for fmt in ("conv.{}.1.weight", "conv.{}.1.bias", "conv.{}.3.weight", "conv.{}.3.bias"):
        out += [fmt.format(i) for i in range(L)]
    return out + ["linear.weight", "linear.bias"]


def _struct(tensors, L, keep):
    """DurPredParams of a list of fp32 contiguous CUDA tensors in param_names order; host arrays go to `keep`."""
    it = iter(tensors)
    kw = {}
    for f in ("conv_w", "conv_b", "ln_w", "ln_b"):
        a = (ctypes.c_void_p * L)(*[next(it).data_ptr() for _ in range(L)])
        keep.append(a)
        kw[f] = ctypes.cast(a, ctypes.POINTER(ctypes.c_void_p))
    kw["linear_w"], kw["linear_b"] = next(it).data_ptr(), next(it).data_ptr()
    return _capi.DurPredParams(**kw)


class DurTrainStep:
    """One dsx_durpred_train handle per (module, device)."""

    def __init__(self, cfg):
        self.cfg = cfg
        self._h = None
        self._device = None

    def close(self):
        if self._h is not None:
            lib.dsx_durpred_train_destroy(self._h)
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
            check(lib.dsx_durpred_train_create(device.index if device.index is not None else torch.cuda.current_device(),
                                               ctypes.byref(self.cfg), ctypes.byref(h)), "dsx_durpred_train_create")
            self._h, self._device = h, device
        return self._h

    def tape_bytes(self, device, B, T):
        n = ctypes.c_size_t()
        check(lib.dsx_durpred_train_tape_bytes(self.handle(device), B, T, ctypes.byref(n)),
              "dsx_durpred_train_tape_bytes")
        return n.value

    def workspace(self, device, B, T):
        """Scratch of one call, from PyTorch's allocator (released to its cache when the call's tensor dies)."""
        n = ctypes.c_size_t()
        check(lib.dsx_durpred_train_workspace_bytes(self.handle(device), B, T, ctypes.byref(n)),
              "dsx_durpred_train_workspace_bytes")
        return torch.empty(n.value, dtype=torch.uint8, device=device)

    def forward(self, params, x, mask, p, seed):
        """xs [B, T] and the tape (uint8 CUDA tensor) of one forward.  params: fp32 CUDA tensors in param_names order;
        x: fp32 [B, T, idim] (any strides); mask: uint8 [B, T] contiguous, 1 = padding."""
        dev = x.device
        h = self.handle(dev)
        B, T, _ = x.shape
        keep = []
        w = _struct(params, self.cfg.layers, keep)
        tape = torch.empty(self.tape_bytes(dev, B, T), dtype=torch.uint8, device=dev)
        xs = torch.empty((B, T), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):     # the forward uses no workspace
            check(lib.dsx_durpred_train_forward(h, ctypes.byref(w), _ptr(x), _strides_bct(x, (0, 2, 1)), _ptr(mask), B,
                                                T, float(p), int(seed), _ptr(tape), tape.numel(), None, 0, _ptr(xs),
                                                _stream(dev)), "dsx_durpred_train_forward")
        return xs, tape

    def backward(self, params, tape, d_xs, B, T, want_x=True):
        """Gradients in param_names order, and d_x [B, T, idim] (or None)."""
        dev = d_xs.device
        h = self.handle(dev)
        keep = []
        w = _struct(params, self.cfg.layers, keep)
        grads = [torch.empty_like(v) for v in params]
        g = _struct(grads, self.cfg.layers, keep)
        d_xs = d_xs.float().contiguous()
        d_x = torch.empty((B, T, self.cfg.idim), dtype=torch.float32, device=dev) if want_x else None
        ws = self.workspace(dev, B, T)
        with torch.cuda.device(dev):
            check(lib.dsx_durpred_train_backward(h, ctypes.byref(w), _ptr(tape), _ptr(d_xs), ctypes.byref(g), _ptr(d_x),
                                                 B, T, _ptr(ws), ws.numel(), _stream(dev)), "dsx_durpred_train_backward")
        return grads, d_x

    def masks(self, device, seed, p, B, T):
        """The n_layers keep masks (bool CUDA tensors [B, T, chans]) a forward with (seed, p) draws."""
        out = [torch.empty((B, T, self.cfg.chans), dtype=torch.uint8, device=device) for _ in range(self.cfg.layers)]
        arr = (ctypes.c_void_p * len(out))(*[m.data_ptr() for m in out])
        with torch.cuda.device(device):
            check(lib.dsx_durpred_train_masks(self.handle(device), int(seed), float(p), B, T, arr, _stream(device)),
                  "dsx_durpred_train_masks")
        return [m.bool() for m in out]


class DurTrainFn(torch.autograd.Function):
    """xs = DurationPredictor._forward in training with the parameters as explicit inputs:
    apply(step, p, seed, x, mask, *params)."""

    @staticmethod
    def forward(ctx, step, p, seed, x, mask, *params):
        xs, tape = step.forward(params, x, mask, p, seed)
        ctx.step, ctx.tape = step, tape
        ctx.BT = (x.shape[0], x.shape[1])
        ctx.save_for_backward(*params)     # the version check: an in-place update before backward raises
        return xs

    @staticmethod
    def backward(ctx, g):
        if torch.is_grad_enabled():
            raise DsxError("dsx_train has no double backward (create_graph=True through the duration predictor's "
                           "training step)")
        return _backward(ctx, g)


@torch.autograd.function.once_differentiable
def _backward(ctx, g):
    B, T = ctx.BT
    grads, d_x = ctx.step.backward(list(ctx.saved_tensors), ctx.tape, g, B, T, want_x=ctx.needs_input_grad[3])
    return (None, None, None, d_x, None) + tuple(grads)


def durpred_train_forward(dp, xs, x_masks):
    """DurationPredictor._forward in training under the dsx_train opt-in: dropout p = the module's dropout_rate.
    xs: CUDA [B, T, idim]; x_masks: [B, T] (True = padding)."""
    named = dict(dp.named_parameters())
    params = [named[n] for n in param_names(dp._cfg.layers)]
    _need_cuda(xs, x_masks, *params)
    if any(p.dtype != torch.float32 for p in params):
        raise DsxError("dsx_train runs fp32 duration predictor parameters")
    if any(not p.is_contiguous() for p in params):
        raise DsxError("dsx_train needs contiguous duration predictor parameters")
    if xs.requires_grad and xs.dtype != torch.float32:
        raise DsxError("dsx_train needs an fp32 xs where it requires grad (its gradient is fp32)")
    B, T, _ = xs.shape
    if B == 0 or T == 0:      # nothing to run: an empty output, as in eval mode
        return xs.float().sum(-1) * 0.0
    mask = x_masks.to(torch.uint8).contiguous()
    return DurTrainFn.apply(dp._dsx_train_step(), float(dp.dropout_rate), draw_seed(), xs.float(), mask, *params)
