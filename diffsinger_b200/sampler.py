"""Host-side owner of one dsx handle: packs a DiffNet module's weights, mirrors the registered schedule
buffers, and exposes the C-ABI entry points on torch CUDA tensors.

PyTorch is plumbing here (device memory, the current stream); all arithmetic runs in libdsx.so.
"""
import ctypes
import os

import torch

from . import _capi
from ._capi import DsxError, Strides, check, lib


def _strides_bct(t, perm):
    """Element strides (b, c, t) of a tensor whose dims `perm` = (b_dim, c_dim, t_dim)."""
    s = t.stride()
    return Strides(s[perm[0]], s[perm[1]], s[perm[2]])


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _stream(dev):
    return ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _need_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise DsxError("dsx runs on CUDA tensors only -- there is no CPU fallback (got a CPU tensor)")


def default_precision():
    return os.environ.get("DSX_PRECISION", "fp16s")


class DsxSampler:
    """One per (denoise_fn module, device).  `net` is any module with the reference DiffNet's parameter
    names (usr/diff/net.py:91-104): the reference class itself or diffsinger_b200.DiffNet."""

    def __init__(self, net, precision=None, dilation_cycle_length=None):
        self.net = net
        self.precision = _capi.PRECISIONS[precision or default_precision()]
        self._cycle = dilation_cycle_length
        self._h = None
        self._device = None
        self._wkey = None
        self._skey = None
        self._keep = None
        self._cond_key = None          # conditioner currently packed in the handle (see _cond_arg)
        self._cond_hold = None

    # -- lifecycle ------------------------------------------------------------------------------
    def close(self):
        if self._h is not None:
            lib.dsx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _handle(self, device):
        if self._h is not None and self._device != device:
            self.close()
        if self._h is None:
            h = ctypes.c_void_p()
            check(lib.dsx_create(device.index if device.index is not None else torch.cuda.current_device(),
                                 ctypes.byref(h)), "dsx_create")
            self._h, self._device, self._wkey, self._skey = h, device, None, None
            self._cond_key = self._cond_hold = None
        return self._h

    def set_precision(self, precision):
        p = _capi.PRECISIONS[precision] if isinstance(precision, str) else precision
        if p != self.precision:
            self.precision, self._wkey = p, None

    def set_option(self, what, value):
        check(lib.dsx_set_option(self._handle(self._device or torch.device("cuda", torch.cuda.current_device())),
                                 what, value), "dsx_set_option")
        if what == _capi.OPT_TC_CTA_GROUP:
            pass

    def info(self, what):
        out = ctypes.c_int64()
        check(lib.dsx_get_info(self._h, what, ctypes.byref(out)), "dsx_get_info")
        return out.value

    # -- weights --------------------------------------------------------------------------------
    def _cycle_len(self):
        if self._cycle is not None:
            return int(self._cycle)
        params = getattr(self.net, "params", None)
        if params is not None and "dilation_cycle_length" in params:
            return int(params["dilation_cycle_length"])
        # recover it from the modules: dilation of layer i is 2**(i % cycle)
        dil = [int(l.dilated_conv.dilation[0]) for l in self.net.residual_layers]
        for i, d in enumerate(dil):
            if i > 0 and d == 1:
                return i
        return len(dil)

    def ensure_weights(self, device):
        h = self._handle(device)
        sd = {k: v for k, v in self.net.state_dict().items()}
        key = (self.precision,) + tuple((k, v.data_ptr(), v._version, tuple(v.shape)) for k, v in sd.items())
        if key == self._wkey:
            return h
        L = len(self.net.residual_layers)
        f = lambda name: sd[name].detach().to(device=device, dtype=torch.float32).contiguous()
        keep = {}

        def g(name):
            keep[name] = f(name)
            return keep[name]

        def arr(fmt):
            a = (ctypes.c_void_p * L)(*[g(fmt.format(l)).data_ptr() for l in range(L)])
            keep["arr_" + fmt] = a
            return ctypes.cast(a, ctypes.POINTER(ctypes.c_void_p))

        p = _capi.DiffNetParams(
            in_w=g("input_projection.weight").data_ptr(), in_b=g("input_projection.bias").data_ptr(),
            mlp0_w=g("mlp.0.weight").data_ptr(), mlp0_b=g("mlp.0.bias").data_ptr(),
            mlp2_w=g("mlp.2.weight").data_ptr(), mlp2_b=g("mlp.2.bias").data_ptr(),
            dil_w=arr("residual_layers.{}.dilated_conv.weight"), dil_b=arr("residual_layers.{}.dilated_conv.bias"),
            dif_w=arr("residual_layers.{}.diffusion_projection.weight"),
            dif_b=arr("residual_layers.{}.diffusion_projection.bias"),
            cond_w=arr("residual_layers.{}.conditioner_projection.weight"),
            cond_b=arr("residual_layers.{}.conditioner_projection.bias"),
            out_w=arr("residual_layers.{}.output_projection.weight"),
            out_b=arr("residual_layers.{}.output_projection.bias"),
            skip_w=g("skip_projection.weight").data_ptr(), skip_b=g("skip_projection.bias").data_ptr(),
            fin_w=g("output_projection.weight").data_ptr(), fin_b=g("output_projection.bias").data_ptr())
        C, M = sd["input_projection.weight"].shape[0], sd["input_projection.weight"].shape[1]
        H = sd["residual_layers.0.conditioner_projection.weight"].shape[1]
        self.M, self.C, self.H, self.L = M, C, H, L
        with torch.cuda.device(device):
            check(lib.dsx_load_diffnet(h, ctypes.byref(p), M, C, H, L, self._cycle_len(), self.precision,
                                       _stream(device)), "dsx_load_diffnet")
        self._wkey = key
        self._cond_key = self._cond_hold = None      # (re)loading frees the workspace
        return h

    # -- schedule -------------------------------------------------------------------------------
    def set_schedule(self, buffers):
        """buffers: mapping name -> fp32 tensor [T], the module's registered buffers verbatim
        (usr/diff/shallow_diffusion_tts.py:101-123)."""
        host = [buffers[n].detach().to("cpu", torch.float32).contiguous() for n in _capi.SCHEDULE_BUFFERS]
        key = tuple(t.numpy().tobytes() for t in host)
        if key == self._skey:
            return
        T = host[0].numel()
        arr = (ctypes.c_void_p * len(host))(*[t.data_ptr() for t in host])
        check(lib.dsx_set_schedule(self._h, ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p)), T), "dsx_set_schedule")
        self._skey = key

    # -- conditioner cache ---------------------------------------------------------------------
    def _cond_arg(self, cond, B, T):
        """Pointer to hand to the C ABI: NULL when the handle already holds the pack + projection of this very
        conditioner for (B, T) (same storage -- kept alive here so its address cannot be recycled -- same view, same
        version counter), so per-step callers do not re-run them (reference loop usr/diff/shallow_diffusion_tts.py:261-270)."""
        st = cond.untyped_storage()
        key = (st.data_ptr(), cond.storage_offset(), tuple(cond.shape), tuple(cond.stride()), cond._version, B, T,
               self._wkey is not None)
        if key == self._cond_key:
            return ctypes.c_void_p(0), key, st
        return _ptr(cond), key, st

    def _cond_done(self, key, st):
        self._cond_key, self._cond_hold = key, st

    # -- entry points ---------------------------------------------------------------------------
    def diffnet_forward(self, spec, diffusion_step, cond):
        """DiffNet.forward (usr/diff/net.py:107-130): spec [B,1,M,T], step [B] int64, cond [B,H,T]."""
        _need_cuda(spec, diffusion_step, cond)
        dev = spec.device
        h = self.ensure_weights(dev)
        B, _, M, T = spec.shape
        spec = spec.float()
        cond = cond.float()
        t = diffusion_step.to(torch.int64).contiguous()
        eps = torch.empty((B, 1, M, T), device=dev, dtype=torch.float32)
        cptr, ckey, chold = self._cond_arg(cond, B, T)
        self._cond_key = None
        with torch.cuda.device(dev):
            check(lib.dsx_diffnet_forward(h, _ptr(spec), _strides_bct(spec, (0, 2, 3)), _ptr(t), cptr,
                                          _strides_bct(cond, (0, 1, 2)), _ptr(eps), B, T, _stream(dev)),
                  "dsx_diffnet_forward")
        self._cond_done(ckey, chold)
        return eps

    def sample_ddpm(self, x, cond, t_start, n_steps=None, noise=None, seed=0):
        """x [B,1,M,T] (returned as a new contiguous tensor), cond [B,H,T] any strides."""
        _need_cuda(x, cond, noise)
        dev = x.device
        h = self.ensure_weights(dev)
        B, _, M, T = x.shape
        n_steps = t_start if n_steps is None else n_steps
        xs = x.float().contiguous().clone()
        cond = cond.float()
        if noise is not None:
            noise = noise.float().contiguous()
            assert noise.shape == (n_steps, B, 1, M, T), noise.shape
        cptr, ckey, chold = self._cond_arg(cond, B, T)
        self._cond_key = None
        with torch.cuda.device(dev):
            check(lib.dsx_sample_ddpm(h, _ptr(xs), cptr, _strides_bct(cond, (0, 1, 2)), B, T, t_start, n_steps,
                                      _ptr(noise), seed, _stream(dev)), "dsx_sample_ddpm")
        self._cond_done(ckey, chold)
        return xs

    def sample_plms(self, x, cond, t_start, interval):
        _need_cuda(x, cond)
        dev = x.device
        h = self.ensure_weights(dev)
        B, _, M, T = x.shape
        xs = x.float().contiguous().clone()
        cond = cond.float()
        cptr, ckey, chold = self._cond_arg(cond, B, T)
        self._cond_key = None
        with torch.cuda.device(dev):
            check(lib.dsx_sample_plms(h, _ptr(xs), cptr, _strides_bct(cond, (0, 1, 2)), B, T, t_start, interval,
                                      _stream(dev)), "dsx_sample_plms")
        self._cond_done(ckey, chold)
        return xs

    def plms_update(self, x, eps_list, mode, t, interval):
        """One linear-multistep combination + get_x_pred (shallow_diffusion_tts.py:174-199) -> new x [B,1,M,T]."""
        _need_cuda(x, *eps_list)
        dev = x.device
        B, _, M, T = x.shape
        xi = x.float().contiguous()
        es = [e.float().contiguous() for e in eps_list]
        out = torch.empty_like(xi)
        arr = (ctypes.c_void_p * 4)(*([e.data_ptr() for e in es] + [None] * (4 - len(es))))
        with torch.cuda.device(dev):
            check(lib.dsx_plms_update(self._h, _ptr(out), _ptr(xi), ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p)), mode,
                                      int(t), int(interval), B, T, _stream(dev)), "dsx_plms_update")
        return out

    def infer(self, cond, K_step, spec_min, spec_max, fs2_mel=None, start_noise=None, x_start=None,
              step_noise=None, seed=0, mel2ph=None, pndm_interval=0):
        """The infer branch after self.fs2 (usr/diff/shallow_diffusion_tts.py:248-275) -> mel_out [B,T,M]."""
        _need_cuda(cond, fs2_mel, start_noise, x_start, step_noise, mel2ph, spec_min, spec_max)
        dev = cond.device
        h = self.ensure_weights(dev)
        B, _, T = cond.shape
        M = self.M
        cond = cond.float()
        c = lambda t: None if t is None else t.float().contiguous()
        fs2_mel, start_noise, x_start, step_noise = c(fs2_mel), c(start_noise), c(x_start), c(step_noise)
        smin = spec_min.float().reshape(-1).contiguous()
        smax = spec_max.float().reshape(-1).contiguous()
        m2p = None if mel2ph is None else mel2ph.to(torch.int64).contiguous()
        out = torch.empty((B, T, M), device=dev, dtype=torch.float32)
        self._cond_key = None
        with torch.cuda.device(dev):
            check(lib.dsx_infer(h, _ptr(cond), _strides_bct(cond, (0, 1, 2)), _ptr(fs2_mel), _ptr(start_noise),
                                _ptr(x_start), _ptr(step_noise), seed, _ptr(m2p), _ptr(smin), _ptr(smax), B, T, K_step,
                                pndm_interval, _ptr(out), _stream(dev)), "dsx_infer")
        return out

    def infer_host(self, cond, K_step, spec_min, spec_max, fs2_mel=None, x_start=None, seed=0, mel2ph=None,
                   pndm_interval=0, out=None, device=None):
        """Same, on HOST tensors (pinned for full copy speed): H2D/D2H copies happen inside the C call."""
        dev = device or self._device or torch.device("cuda", torch.cuda.current_device())
        h = self.ensure_weights(dev)
        B, _, T = cond.shape
        M = self.M
        for name, t in (("cond", cond), ("fs2_mel", fs2_mel), ("x_start", x_start), ("mel2ph", mel2ph), ("out", out)):
            if t is not None and t.is_cuda:
                raise DsxError(f"infer_host takes HOST tensors ({name} is a CUDA tensor); use infer() for device tensors")
        cond = cond.float()
        # the C side copies B*H*T contiguous floats and then addresses them through the strides: the view must be dense
        # (a permutation of a contiguous [B,H,T] block, e.g. the reference's transposed [B,T,H]); anything else is compacted
        span = sum((n - 1) * st for n, st in zip(cond.shape, cond.stride())) + 1
        if span != cond.numel() or min(cond.stride()) < 1:
            cond = cond.contiguous()
        c = lambda t: None if t is None else t.float().contiguous()
        fs2_mel, x_start = c(fs2_mel), c(x_start)
        smin, smax = spec_min.float().reshape(-1).contiguous().cpu(), spec_max.float().reshape(-1).contiguous().cpu()
        m2p = None if mel2ph is None else mel2ph.to(torch.int64).contiguous()
        if out is None:
            out = torch.empty((B, T, M), dtype=torch.float32).pin_memory()
        self._cond_key = None
        with torch.cuda.device(dev):
            check(lib.dsx_infer_host(h, _ptr(cond), _strides_bct(cond, (0, 1, 2)), _ptr(fs2_mel), _ptr(x_start), seed,
                                     _ptr(m2p), _ptr(smin), _ptr(smax), B, T, K_step, pndm_interval, _ptr(out),
                                     _stream(dev)), "dsx_infer_host")
        return out

    def debug_read(self, which, B, T):
        out = torch.empty((B, T, self.C), device=self._device, dtype=torch.float32)
        with torch.cuda.device(self._device):
            check(lib.dsx_debug_read(self._h, which, _ptr(out), B, T, _stream(self._device)), "dsx_debug_read")
        return out

    def set_layer_limit(self, n):
        check(lib.dsx_debug_set_layer_limit(self._h, n), "dsx_debug_set_layer_limit")


def selftest(device=0, which=-1):
    buf = ctypes.create_string_buffer(16384)
    rc = lib.dsx_selftest(device, which, buf, 16384)
    return rc, buf.value.decode(errors="replace")
