"""FFT diffusion denoiser training step on libdsx: the forward with dropout and a saved tape, and the backward
(include/dsx.h, dsx_fft_train_*), wrapped in a ``torch.autograd.Function`` so that ``diffsinger_b200.FFT`` under
``dsx_train`` gives ordinary ``.grad`` tensors to DDP and any optimizer, and its gradient with respect to cond flows back
into FastSpeech2.  q_sample, the loss and the optimizer stay in the caller's PyTorch code (``p_losses``)."""
import ctypes

import torch

from . import _capi
from ._capi import DsxError, check, lib
from .fs2train import _struct as _dec_struct
from .fs2train import draw_seed, param_names as dec_param_names
from .sampler import _need_cuda, _ptr, _stream, _strides_bct

M = 80
# FftParams field -> state-dict name of the FFT's own parameters (those outside the FFTBlocks stack)
_OWN = (("in_w", "input_projection.weight"), ("in_b", "input_projection.bias"), ("mlp0_w", "mlp.0.weight"),
        ("mlp0_b", "mlp.0.bias"), ("mlp2_w", "mlp.2.weight"), ("mlp2_b", "mlp.2.bias"),
        ("decode_inp_w", "get_decode_inp.weight"), ("decode_inp_b", "get_decode_inp.bias"),
        ("mel_out_w", "get_mel_out.weight"), ("mel_out_b", "get_mel_out.bias"))


def param_names(L, padding):
    """Every FFT parameter name (the state dict less embed_positions._float_tensor), in the autograd function's order:
    the stack's (fs2train.param_names), then the entry and exit."""
    return dec_param_names(L, padding) + [n for _, n in _OWN]


def _struct(tensors, L, keep):
    """FftParams of fp32 contiguous CUDA tensors in param_names order; host arrays go to `keep`."""
    n_dec = len(tensors) - len(_OWN)
    dec = _dec_struct(tensors[:n_dec], L, keep)
    return _capi.FftParams(dec=dec, **{f: v.data_ptr() for (f, _), v in zip(_OWN, tensors[n_dec:])})


class FftTrainStep:
    """One dsx_fft_train handle per (module, device)."""

    def __init__(self, cfg):
        self.cfg = cfg
        self._h = None
        self._device = None

    def close(self):
        if self._h is not None:
            lib.dsx_fft_train_destroy(self._h)
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
            check(lib.dsx_fft_train_create(device.index if device.index is not None else torch.cuda.current_device(),
                                           ctypes.byref(self.cfg), ctypes.byref(h)), "dsx_fft_train_create")
            self._h, self._device = h, device
        return self._h

    def tape_bytes(self, device, B, T):
        n = ctypes.c_size_t()
        check(lib.dsx_fft_train_tape_bytes(self.handle(device), B, T, ctypes.byref(n)), "dsx_fft_train_tape_bytes")
        return n.value

    def workspace(self, device, B, T):
        """Scratch of one call, from PyTorch's allocator (released to its cache when the call's tensor dies)."""
        n = ctypes.c_size_t()
        check(lib.dsx_fft_train_workspace_bytes(self.handle(device), B, T, ctypes.byref(n)),
              "dsx_fft_train_workspace_bytes")
        return torch.empty(n.value, dtype=torch.uint8, device=device)

    def forward(self, params, spec, t, cond, p, seed):
        """eps [B, 1, 80, T] and the tape (uint8 CUDA tensor) of one forward; params: fp32 CUDA tensors in param_names
        order."""
        dev = spec.device
        h = self.handle(dev)
        B, T = spec.shape[0], spec.shape[3]
        keep = []
        w = _struct(params, self.cfg.dec.layers, keep)
        t = t.to(torch.int64).contiguous()
        tape = torch.empty(self.tape_bytes(dev, B, T), dtype=torch.uint8, device=dev)
        eps = torch.empty((B, 1, M, T), dtype=torch.float32, device=dev)
        ws = self.workspace(dev, B, T)
        with torch.cuda.device(dev):
            check(lib.dsx_fft_train_forward(h, ctypes.byref(w), _ptr(spec), _strides_bct(spec, (0, 2, 3)), _ptr(t),
                                            _ptr(cond), _strides_bct(cond, (0, 1, 2)), B, T, float(p), int(seed),
                                            _ptr(tape), tape.numel(), _ptr(ws), ws.numel(), _ptr(eps), _stream(dev)),
                  "dsx_fft_train_forward")
        return eps, tape

    def backward(self, params, tape, d_eps, B, T, want_cond=True):
        """Gradients in param_names order, and d_cond as a [B, H, T] view of a frames-major tensor (or None)."""
        dev = d_eps.device
        h = self.handle(dev)
        keep = []
        L = self.cfg.dec.layers
        w = _struct(params, L, keep)
        grads = [torch.empty_like(v) for v in params]
        g = _struct(grads, L, keep)
        d_eps = d_eps.float().contiguous()
        d_cond = torch.empty((B, T, self.cfg.dec.hidden), dtype=torch.float32, device=dev) if want_cond else None
        ws = self.workspace(dev, B, T)
        with torch.cuda.device(dev):
            check(lib.dsx_fft_train_backward(h, ctypes.byref(w), _ptr(tape), _ptr(d_eps), ctypes.byref(g),
                                             _ptr(d_cond), B, T, _ptr(ws), ws.numel(), _stream(dev)),
                  "dsx_fft_train_backward")
        return grads, (d_cond.transpose(1, 2) if want_cond else None)


class FftTrainFn(torch.autograd.Function):
    """eps = FFT(spec, t, cond) in training with the parameters as explicit inputs:
    apply(step, p, seed, spec, t, cond, *params)."""

    @staticmethod
    def forward(ctx, step, p, seed, spec, t, cond, *params):
        eps, tape = step.forward(params, spec, t, cond, p, seed)
        ctx.step, ctx.tape = step, tape
        ctx.BT = (spec.shape[0], spec.shape[3])
        ctx.save_for_backward(*params)     # the version check: an in-place update before backward raises
        return eps

    @staticmethod
    def backward(ctx, g):
        if torch.is_grad_enabled():
            raise DsxError("dsx_train has no double backward (create_graph=True through the FFT denoiser's training "
                           "step)")
        return _backward(ctx, g)


@torch.autograd.function.once_differentiable
def _backward(ctx, g):
    B, T = ctx.BT
    grads, d_cond = ctx.step.backward(list(ctx.saved_tensors), ctx.tape, g, B, T, want_cond=ctx.needs_input_grad[5])
    return (None, None, None, None, None, d_cond) + tuple(grads)


def fft_train_forward(net, spec, diffusion_step, cond):
    """FFT.forward in training under the dsx_train opt-in: dropout p = hparams['dropout'], the libdsx forward and
    backward."""
    H = net.hidden_size
    if spec.dim() != 4 or spec.shape[1] != 1 or spec.shape[2] != M:
        raise DsxError(f"spec must be [B, 1, {M}, T] (got {tuple(spec.shape)})")
    B, T = spec.shape[0], spec.shape[3]
    if tuple(cond.shape) != (B, H, T) or tuple(diffusion_step.shape) != (B,):
        raise DsxError(f"cond must be [B, {H}, T] and diffusion_step [B] for spec {tuple(spec.shape)} (got "
                       f"{tuple(cond.shape)}, {tuple(diffusion_step.shape)})")
    if spec.requires_grad:
        raise DsxError("dsx_train computes no gradient of spec (p_losses' x_noisy does not require grad); "
                       "spec.requires_grad is set")
    named = dict(net.named_parameters())
    params = [named[n] for n in param_names(net.num_layers, net.padding)]
    _need_cuda(spec, diffusion_step, cond, *params)
    if any(p.dtype != torch.float32 for p in params) or spec.dtype != torch.float32 or cond.dtype != torch.float32:
        raise DsxError("dsx_train runs fp32 parameters and inputs")
    if any(not p.is_contiguous() for p in params):
        raise DsxError("dsx_train needs contiguous parameters")
    return FftTrainFn.apply(net._dsx_train_step(), float(net.dropout), draw_seed(), spec, diffusion_step, cond,
                            *params)
