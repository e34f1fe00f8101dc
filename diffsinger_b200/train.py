"""DiffNet training step on libdsx: the forward with a saved tape and the backward (include/dsx.h, dsx_train_*), wrapped
in a ``torch.autograd.Function`` so that ``DiffNet`` under ``dsx_train`` gives ordinary ``.grad`` tensors to DDP and any
optimizer.  The loss stays in the caller's PyTorch code."""
import ctypes

import torch

from . import _capi
from ._capi import DsxError, check, lib
from .sampler import _need_cuda, _ptr, _stream, _strides_bct

M, C, H = 80, 256, 256

# DiffNetParams field -> state-dict name (per-layer fields: a format string over the layer index)
_FIELDS = (
    ("in_w", "input_projection.weight"), ("in_b", "input_projection.bias"),
    ("mlp0_w", "mlp.0.weight"), ("mlp0_b", "mlp.0.bias"), ("mlp2_w", "mlp.2.weight"), ("mlp2_b", "mlp.2.bias"),
    ("dil_w", "residual_layers.{}.dilated_conv.weight"), ("dil_b", "residual_layers.{}.dilated_conv.bias"),
    ("dif_w", "residual_layers.{}.diffusion_projection.weight"),
    ("dif_b", "residual_layers.{}.diffusion_projection.bias"),
    ("cond_w", "residual_layers.{}.conditioner_projection.weight"),
    ("cond_b", "residual_layers.{}.conditioner_projection.bias"),
    ("out_w", "residual_layers.{}.output_projection.weight"),
    ("out_b", "residual_layers.{}.output_projection.bias"),
    ("skip_w", "skip_projection.weight"), ("skip_b", "skip_projection.bias"),
    ("fin_w", "output_projection.weight"), ("fin_b", "output_projection.bias"),
)


def param_names(L):
    """Every DiffNet parameter name, in the order the autograd function takes them."""
    out = []
    for _, n in _FIELDS:
        out += [n.format(l) for l in range(L)] if "{}" in n else [n]
    return out


def _struct(tensors, L, keep):
    """DiffNetParams of a mapping name -> fp32 contiguous CUDA tensor; host pointer arrays go to `keep`."""
    kw = {}
    for f, n in _FIELDS:
        if "{}" in n:
            a = (ctypes.c_void_p * L)(*[tensors[n.format(l)].data_ptr() for l in range(L)])
            keep.append(a)
            kw[f] = ctypes.cast(a, ctypes.POINTER(ctypes.c_void_p))
        else:
            kw[f] = tensors[n].data_ptr()
    return _capi.DiffNetParams(**kw)


def check_shapes(net, spec, cond):
    """DsxError unless the kernels run this module and these inputs: M = 80, C = H = 256, spec [B,1,80,T], cond
    [B,256,T]."""
    p = net.params
    if (p["residual_channels"], p["encoder_hidden"], net.input_projection.in_channels) != (C, H, M):
        raise DsxError(f"dsx_train runs residual_channels = hidden_size = {C} and in_dims = {M} only (got "
                       f"{p['residual_channels']}, {p['encoder_hidden']}, {net.input_projection.in_channels})")
    if spec.dim() != 4 or spec.shape[1] != 1 or spec.shape[2] != M:
        raise DsxError(f"dsx_train needs spec [B, 1, {M}, T] (got {tuple(spec.shape)})")
    B, T = spec.shape[0], spec.shape[3]
    if tuple(cond.shape) != (B, H, T):
        raise DsxError(f"dsx_train needs cond [B, {H}, T] = {(B, H, T)} (got {tuple(cond.shape)})")


class TrainStep:
    """One dsx_train handle per (module, device)."""

    def __init__(self, L, cycle):
        self.L, self.cycle = L, cycle
        self._h = None
        self._device = None

    def close(self):
        if self._h is not None:
            lib.dsx_train_destroy(self._h)
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
            cfg = _capi.TrainConfig(M, C, H, self.L, self.cycle)
            check(lib.dsx_train_create(device.index if device.index is not None else torch.cuda.current_device(),
                                       ctypes.byref(cfg), ctypes.byref(h)), "dsx_train_create")
            self._h, self._device = h, device
        return self._h

    def tape_bytes(self, device, B, T):
        n = ctypes.c_size_t()
        check(lib.dsx_train_tape_bytes(self.handle(device), B, T, ctypes.byref(n)), "dsx_train_tape_bytes")
        return n.value

    def workspace(self, device, B, T):
        """Scratch of one call, from PyTorch's allocator (released to its cache when the call's tensor dies)."""
        n = ctypes.c_size_t()
        check(lib.dsx_train_workspace_bytes(self.handle(device), B, T, ctypes.byref(n)), "dsx_train_workspace_bytes")
        return torch.empty(n.value, dtype=torch.uint8, device=device)

    def forward(self, params, spec, t, cond):
        """eps [B,1,80,T] and the tape (uint8 CUDA tensor) of one forward; params: name -> fp32 CUDA tensor."""
        dev = spec.device
        h = self.handle(dev)
        B, T = spec.shape[0], spec.shape[3]
        keep = []
        w = _struct(params, self.L, keep)
        t = t.to(torch.int64).contiguous()
        tape = torch.empty(self.tape_bytes(dev, B, T), dtype=torch.uint8, device=dev)
        eps = torch.empty((B, 1, M, T), dtype=torch.float32, device=dev)
        ws = self.workspace(dev, B, T)
        with torch.cuda.device(dev):
            check(lib.dsx_train_forward(h, ctypes.byref(w), _ptr(spec), _strides_bct(spec, (0, 2, 3)), _ptr(t),
                                        _ptr(cond), _strides_bct(cond, (0, 1, 2)), B, T, _ptr(tape), tape.numel(),
                                        _ptr(ws), ws.numel(), _ptr(eps), _stream(dev)), "dsx_train_forward")
        return eps, tape

    def backward(self, params, tape, d_eps, B, T, want_cond=True):
        """name -> gradient tensor, and d_cond [B,256,T] (or None)."""
        dev = d_eps.device
        h = self.handle(dev)
        keep = []
        w = _struct(params, self.L, keep)
        grads = {n: torch.empty_like(v) for n, v in params.items()}
        g = _struct(grads, self.L, keep)
        d_eps = d_eps.float().contiguous()
        d_cond = torch.empty((B, H, T), dtype=torch.float32, device=dev) if want_cond else None
        ws = self.workspace(dev, B, T)
        with torch.cuda.device(dev):
            check(lib.dsx_train_backward(h, ctypes.byref(w), _ptr(tape), _ptr(d_eps), ctypes.byref(g), _ptr(d_cond),
                                         B, T, _ptr(ws), ws.numel(), _stream(dev)), "dsx_train_backward")
        return grads, d_cond


class DiffNetTrainFn(torch.autograd.Function):
    """eps = DiffNet(spec, t, cond) with the parameters as explicit inputs: apply(step, names, spec, t, cond, *params)."""

    @staticmethod
    def forward(ctx, step, names, spec, t, cond, *params):
        tensors = dict(zip(names, params))
        eps, tape = step.forward(tensors, spec, t, cond)
        ctx.step, ctx.names, ctx.tape = step, names, tape
        ctx.BT = (spec.shape[0], spec.shape[3])
        ctx.save_for_backward(*params)     # the version check: an in-place update before backward raises
        return eps

    @staticmethod
    def backward(ctx, g):
        if torch.is_grad_enabled():
            raise DsxError("dsx_train has no double backward (create_graph=True through DiffNet's training step)")
        return _backward(ctx, g)


@torch.autograd.function.once_differentiable
def _backward(ctx, g):
    params = dict(zip(ctx.names, ctx.saved_tensors))
    B, T = ctx.BT
    grads, d_cond = ctx.step.backward(params, ctx.tape, g, B, T, want_cond=ctx.needs_input_grad[4])
    return (None, None, None, None, d_cond) + tuple(grads[n] for n in ctx.names)


def diffnet_train_forward(net, spec, diffusion_step, cond):
    """DiffNet.forward in training under the dsx_train opt-in: the libdsx forward, with the libdsx backward."""
    check_shapes(net, spec, cond)
    if spec.requires_grad:
        raise DsxError("dsx_train computes no gradient of spec (p_losses' x_noisy does not require grad); "
                       "spec.requires_grad is set")
    named = dict(net.named_parameters())
    names = param_names(len(net.residual_layers))
    params = [named[n] for n in names]
    _need_cuda(spec, diffusion_step, cond, *params)
    if any(p.dtype != torch.float32 for p in params) or spec.dtype != torch.float32 or cond.dtype != torch.float32:
        raise DsxError("dsx_train runs fp32 parameters and inputs")
    if any(not p.is_contiguous() for p in params):
        raise DsxError("dsx_train needs contiguous parameters")
    step = net._dsx_train_step()
    return DiffNetTrainFn.apply(step, names, spec, diffusion_step, cond, *params)
