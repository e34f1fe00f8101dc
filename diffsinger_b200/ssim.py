"""The reference's ``ssim(img1, img2, window_size=11, size_average=True)`` (modules/commons/ssim.py:383-391) on the sm_90a
kernels of libdsx.so (``dsx_ssim_forward`` / ``dsx_ssim_backward`` in include/dsx.h), differentiable in both images.

Inputs are fp32 CUDA tensors [B, 1, H, W] of one shape (any strides), with W <= 256 (the mel bins or the CWT
scales).  The result is ``ssim_map.mean()`` when ``size_average`` is true, else ``ssim_map.mean(1)`` [B, H, W], as in
the reference.  The kernels work in fp32 on CUDA cores, never TF32, so the variance terms keep their precision after
``ssim_loss``'s bias of 6.  The backward saves the inputs, not the maps, and recomputes the moments.  There is no
eager or CPU path: a CPU tensor, another dtype or shape, a channel count other than 1, a window other than 11 and a
double backward raise ``DsxError``.
"""
import torch

from ._capi import DsxError, check, lib
from .sampler import _need_cuda, _ptr, _stream

WINDOW_SIZE = 11
MAX_WIDTH = 256


def _check(img1, img2, window_size):
    if window_size != WINDOW_SIZE:
        raise DsxError(f"ssim: window_size {window_size} is not supported (only {WINDOW_SIZE})")
    if not isinstance(img1, torch.Tensor) or not isinstance(img2, torch.Tensor):
        raise DsxError("ssim: img1 and img2 must be tensors")
    if img1.dim() != 4:
        raise DsxError(f"ssim: inputs must be [B, 1, H, W] (got dim {img1.dim()})")
    if img1.shape != img2.shape:
        raise DsxError(f"ssim: img1 {tuple(img1.shape)} and img2 {tuple(img2.shape)} differ in shape")
    if img1.device != img2.device:
        raise DsxError(f"ssim: img1 and img2 are on different devices ({img1.device}, {img2.device})")
    B, C, H, W = img1.shape
    if C != 1:
        raise DsxError(f"ssim: only one channel is supported (got {C})")
    if B < 1 or H < 1 or not 1 <= W <= MAX_WIDTH:
        raise DsxError(f"ssim: needs B >= 1, H >= 1 and 1 <= W <= {MAX_WIDTH} (got {B}, {H}, {W})")
    if img1.dtype != torch.float32 or img2.dtype != torch.float32:
        raise DsxError(f"ssim: inputs must be float32 (got {img1.dtype}, {img2.dtype})")
    _need_cuda(img1, img2)


class _SsimMap(torch.autograd.Function):
    """[B, 1, H, W] x 2 -> the SSIM map [B, H, W]."""

    @staticmethod
    def forward(ctx, img1, img2):
        B, _, H, W = img1.shape
        x, y = img1.detach().contiguous(), img2.detach().contiguous()
        dev = x.device
        out = torch.empty((B, H, W), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            check(lib.dsx_ssim_forward(_ptr(x), _ptr(y), B, H, W, _ptr(out), _stream(dev)), "dsx_ssim_forward")
        ctx.save_for_backward(x, y)
        return out

    @staticmethod
    def backward(ctx, d_map):
        if torch.is_grad_enabled():
            raise DsxError("ssim: double backward is not supported")
        x, y = ctx.saved_tensors
        B, _, H, W = x.shape
        need_x, need_y = ctx.needs_input_grad
        d_x = torch.empty_like(x) if need_x else None
        d_y = torch.empty_like(y) if need_y else None
        if d_x is None and d_y is None:
            return None, None
        g = d_map.to(torch.float32).expand(B, H, W).contiguous()
        dev = x.device
        with torch.cuda.device(dev):
            check(lib.dsx_ssim_backward(_ptr(x), _ptr(y), _ptr(g), B, H, W, _ptr(d_x), _ptr(d_y), _stream(dev)),
                  "dsx_ssim_backward")
        return d_x, d_y


def ssim(img1, img2, window_size=11, size_average=True):
    """modules/commons/ssim.py:383-391 on dsx: img1, img2 fp32 CUDA [B, 1, H, W] -> a scalar (size_average) or
    [B, H, W]."""
    _check(img1, img2, window_size)
    ssim_map = _SsimMap.apply(img1, img2)
    return ssim_map.mean() if size_average else ssim_map
