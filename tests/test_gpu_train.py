"""GPU: the DiffNet training step (dsx_train_*) against fp32 autograd of the same module with TF32 off, its dynamic
gradient scale, determinism, the reference's zero-initialised output projection, several forwards before one backward,
and the p_losses training branch with Adam."""

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0) if torch.cuda.is_available() else None
BOUND_TENSOR, BOUND_MEDIAN, BOUND_COND, BOUND_EPS = 5e-2, 3e-2, 5e-2, 1e-2
# the golden fixture has 2 x 24 frames, so a bias gradient sums few terms: TF32 autograd (cuDNN's defaults, the
# reference's own training numerics on an H100) is off by up to 7.7e-2 per tensor there, dsx by up to 5.1e-2
BOUND_GOLDEN_TENSOR = 6e-2


def _net(L, cycle, seed=0, zero_final=False):
    import diffsinger_b200 as dsx
    hp = dict(hidden_size=256, residual_layers=L, residual_channels=256, dilation_cycle_length=cycle)
    torch.manual_seed(seed)
    net = dsx.DiffNet(80, hparams=hp, train=True)
    if not zero_final:
        torch.nn.init.normal_(net.output_projection.weight, std=0.02)
    return net.to(DEV).train()


def _inputs(B, T, seed=1):
    g = torch.Generator().manual_seed(seed)
    spec = torch.randn(B, 1, 80, T, generator=g)
    cond = torch.randn(B, T, 256, generator=g).transpose(1, 2)      # the reference's strided view
    t = torch.randint(0, 100, (B,), generator=g)
    noise = torch.randn(B, 1, 80, T, generator=g)
    return spec.to(DEV), t.to(DEV), cond.to(DEV), noise.to(DEV)


def _loss(kind, noise, eps):
    return (noise - eps).abs().mean() if kind == "l1" else F.mse_loss(noise, eps)


def _grads(net, spec, t, cond, noise, kind, path):
    """(loss, eps, {name: grad}, d_cond) through dsx ('dsx') or autograd ('fp32': TF32 off, 'cudnn': defaults)."""
    net.zero_grad(set_to_none=True)
    c = cond.detach().clone().requires_grad_(True)
    if path == "dsx":
        eps = net(spec, t, c)
    else:
        old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = path == "cudnn"
        try:
            eps = net._forward_autograd(spec, t, c)
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    loss = _loss(kind, noise, eps)
    loss.backward()
    return loss.item(), eps.detach(), {n: p.grad.detach().clone() for n, p in net.named_parameters()}, c.grad.detach()


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _errors(test, ref):
    _, eps1, g1, c1 = test
    _, eps0, g0, c0 = ref
    per = {n: _rel(g1[n], g0[n]) for n in g0}
    return per, _rel(c1, c0), _rel(eps1, eps0)


def _check_bound1(per, dcond, deps=None):
    worst = max(per, key=per.get)
    med = sorted(per.values())[len(per) // 2]
    assert per[worst] <= BOUND_TENSOR, (worst, per[worst])
    assert med <= BOUND_MEDIAN, med
    assert dcond <= BOUND_COND, dcond
    if deps is not None:
        assert deps <= BOUND_EPS, deps


@pytest.mark.parametrize("B,T,cycle,L", [(2, 1000, 4, 20), (3, 37, 1, 20), (1, 2048, 4, 20), (2, 200, 4, 2)])
@pytest.mark.parametrize("kind", ["l1", "l2"])
def test_parity_with_fp32_autograd(lib_built, B, T, cycle, L, kind):
    net = _net(L, cycle)
    spec, t, cond, noise = _inputs(B, T)
    ref = _grads(net, spec, t, cond, noise, kind, "fp32")
    mine = _grads(net, spec, t, cond, noise, kind, "dsx")
    cud = _grads(net, spec, t, cond, noise, kind, "cudnn")
    per, dc, de = _errors(mine, ref)
    per_c, dc_c, de_c = _errors(cud, ref)
    med = lambda p: sorted(p.values())[len(p) // 2]
    print(f"\n[{kind} B={B} T={T} cycle={cycle} L={L}] dsx: worst {max(per.values()):.2e} ({max(per, key=per.get)}), "
          f"median {med(per):.2e}, d_cond {dc:.2e}, eps {de:.2e}; autograd with cuDNN defaults: worst "
          f"{max(per_c.values()):.2e}, median {med(per_c):.2e}, d_cond {dc_c:.2e}, eps {de_c:.2e}; "
          f"loss {mine[0]:.6f} vs {ref[0]:.6f}")
    _check_bound1(per, dc, de)


def _direct(net, B, T, seed=1):
    from diffsinger_b200 import train
    spec, t, cond, _ = _inputs(B, T, seed)
    step = net._dsx_train_step()
    params = {n: p.detach() for n, p in net.named_parameters()}
    eps, tape = step.forward(params, spec, t, cond)
    return step, params, eps, tape, train


def test_scale_invariance_and_zero_gradient(lib_built):
    net = _net(20, 4)
    B, T = 2, 300
    step, params, eps, tape, _ = _direct(net, B, T)
    d = torch.randn(B, 1, 80, T, device=DEV) / (B * 80 * T)
    g0, c0 = step.backward(params, tape, d, B, T)
    for k in (-20, 0, 12):
        gk, ck = step.backward(params, tape, d * 2.0 ** k, B, T)
        for n in g0:
            assert torch.equal(gk[n], g0[n] * 2.0 ** k), (k, n)
        assert torch.equal(ck, c0 * 2.0 ** k), k
    gz, cz = step.backward(params, tape, torch.zeros_like(d), B, T)
    for n, v in gz.items():
        assert torch.isfinite(v).all() and (v == 0).all(), n
    assert (cz == 0).all()


def test_two_backwards_from_one_tape_are_bitwise_equal(lib_built):
    net = _net(20, 4)
    B, T = 2, 500
    step, params, eps, tape, _ = _direct(net, B, T)
    d = torch.sign(torch.randn(B, 1, 80, T, device=DEV)) / (B * 80 * T)
    g1, c1 = step.backward(params, tape, d, B, T)
    g2, c2 = step.backward(params, tape, d, B, T)
    assert all(torch.equal(g1[n], g2[n]) for n in g1) and torch.equal(c1, c2)


def test_reference_initialisation(lib_built):
    """The reference zero-initialises output_projection: every other gradient is exactly 0."""
    net = _net(20, 4, zero_final=True)
    spec, t, cond, noise = _inputs(2, 200)
    _, _, g, c = _grads(net, spec, t, cond, noise, "l1", "dsx")
    _, _, g0, _ = _grads(net, spec, t, cond, noise, "l1", "fp32")
    for n, v in g.items():
        if not n.startswith("output_projection."):
            assert (v == 0).all(), n
    assert (c == 0).all()
    for n in ("output_projection.weight", "output_projection.bias"):
        assert _rel(g[n], g0[n]) <= BOUND_TENSOR, n


def test_two_forwards_one_backward(lib_built):
    net = _net(20, 4)
    a, b = _inputs(2, 300, seed=3), _inputs(1, 700, seed=4)
    sep = []
    for spec, t, cond, noise in (a, b):
        net.zero_grad(set_to_none=True)
        _loss("l1", noise, net(spec, t, cond)).backward()
        sep.append({n: p.grad.clone() for n, p in net.named_parameters()})
    net.zero_grad(set_to_none=True)
    (_loss("l1", a[3], net(*a[:3])) + _loss("l1", b[3], net(*b[:3]))).backward()
    for n, p in net.named_parameters():
        want = sep[0][n] + sep[1][n]
        tol = 1e-6 * want.abs().max().item() + 1e-30
        assert (p.grad - want).abs().max().item() <= tol, n


def test_refusals_on_the_gpu(lib_built):
    from diffsinger_b200 import DsxError
    net = _net(2, 1)
    spec, t, cond, noise = _inputs(1, 64)
    with pytest.raises(DsxError):
        net(spec.clone().requires_grad_(True), t, cond)
    c = cond.clone().requires_grad_(True)
    eps = net(spec, t, c)
    with pytest.raises(DsxError):
        torch.autograd.grad(_loss("l1", noise, eps), c, create_graph=True)


class _Stub(torch.nn.Module):
    def __init__(self, dec):
        super().__init__()
        self.dec = dec

    def forward(self, *a, **k):
        return {"decoder_inp": self.dec}


def _diffusion(train, seed=0):
    import diffsinger_b200 as dsx
    from oracle import diffnet_oracle as O
    hp = dict(hidden_size=256, residual_layers=20, residual_channels=256, dilation_cycle_length=4, keep_bins=80,
              dsx_train=train)
    torch.manual_seed(seed)
    net = dsx.DiffNet(80, hparams=hp)
    torch.nn.init.normal_(net.output_projection.weight, std=0.02)
    m = dsx.GaussianDiffusion(None, 80, net, timesteps=100, K_step=100, loss_type="l1",
                              betas=O.linear_beta_schedule(100, 0.06), spec_min=[-6.0] * 80, spec_max=[0.5] * 80,
                              fs2=_Stub(None), hparams=hp)
    return m.to(DEV).train()


def test_p_losses_and_adam(lib_built):
    """GaussianDiffusion.forward(infer=False) -> ret['diff_loss'].backward() with the opt-in, then 20 Adam steps on one
    batch against the same run in fp32 autograd (TF32 off).  This drives the package's own GaussianDiffusion mirror,
    whose forward(infer=False) and p_losses restate the reference's (shallow_diffusion_tts.py:213-231, 233-247): the
    stand-in tree of tests/standin_ref.py has no training branch (its forward raises)."""
    B, T = 2, 256
    g = torch.Generator().manual_seed(7)
    mel = (torch.rand(B, T, 80, generator=g) * 6.5 - 6.0).to(DEV)
    dec = torch.randn(B, T, 256, generator=g).to(DEV)
    tok = torch.zeros(B, 5, dtype=torch.long, device=DEV)
    runs = {}
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        for train in (True, False):
            m = _diffusion(train)
            m.fs2 = _Stub(dec)
            torch.manual_seed(11)
            ret = m(tok, ref_mels=mel, infer=False)
            ret["diff_loss"].backward()
            grads = {n: p.grad.clone() for n, p in m.denoise_fn.named_parameters()}
            opt = torch.optim.Adam(m.denoise_fn.parameters(), lr=2e-4)
            losses = []
            for i in range(20):
                opt.zero_grad(set_to_none=True)
                torch.manual_seed(100)            # the same t and noise every step: one fixed batch
                loss = m(tok, ref_mels=mel, infer=False)["diff_loss"]
                loss.backward()
                opt.step()
                losses.append(loss.item())
            runs[train] = grads, losses
    finally:
        torch.backends.cudnn.allow_tf32 = old
    per = {n: _rel(runs[True][0][n], runs[False][0][n]) for n in runs[False][0]}
    print(f"\np_losses grads: worst {max(per.values()):.2e}, losses dsx {runs[True][1][0]:.4f} -> "
          f"{runs[True][1][-1]:.4f}, fp32 {runs[False][1][0]:.4f} -> {runs[False][1][-1]:.4f}")
    _check_bound1(per, 0.0)
    ld, lf = runs[True][1], runs[False][1]
    assert ld[-1] < ld[0]
    assert abs(ld[-1] - lf[-1]) <= 0.05 * lf[-1]


def test_golden_gradients(lib_built):
    """The reference's own p_losses gradients (tests/golden/diffnet_train_grad.npz, L = 20, cycle 4, B = 2, T = 24)."""
    import numpy as np
    import diffsinger_b200 as dsx
    from conftest import golden
    from oracle import diffnet_oracle as O
    from oracle import gen_golden_train as G
    g = golden("diffnet_train_grad.npz")
    L, cycle = int(g["L"]), int(g["cycle"])
    net = dsx.DiffNet(80, hparams=dict(hidden_size=256, residual_layers=L, residual_channels=256,
                                       dilation_cycle_length=cycle), train=True)
    net.load_state_dict(O.build_state_dict(int(g["seed"]), residual_layers=L, dilation_cycle_length=cycle), strict=True)
    net = net.to(DEV).train()
    x_start, t, noise, cond = (v.to(DEV) for v in G.inputs())
    S = O.make_schedule(O.linear_beta_schedule(int(g["steps"]), 0.06))
    e = lambda a: a.to(DEV).gather(-1, t).reshape(t.shape[0], 1, 1, 1)
    x_noisy = e(S["sqrt_alphas_cumprod"]) * x_start + e(S["sqrt_one_minus_alphas_cumprod"]) * noise
    rel = lambda a, b: float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))

    def errors(forward):
        """Per-tensor relative Frobenius error against the golden, estimated from the stored entries (their squared
        error scaled to the whole tensor, over the reference's norm) and from the norm itself; and d_cond's."""
        net.zero_grad(set_to_none=True)
        c = cond.clone().requires_grad_(True)
        loss = (noise - forward(x_noisy, t, c)).abs().mean()
        loss.backward()
        per = {}
        for n, p in net.named_parameters():
            flat = p.grad.reshape(-1).cpu()
            d = flat[torch.from_numpy(G.sample_index(n, flat.numel())).long()].numpy() - g["val." + n]
            est = float(np.sqrt((d.astype(np.float64) ** 2).mean() * flat.numel()) / float(g["norm." + n]))
            per[n] = max(rel(flat.norm().numpy(), g["norm." + n]), est)
        return loss.item(), per, rel(c.grad.cpu().numpy(), g["d_cond"])

    loss, per, dc = errors(net)
    old = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = True
    try:
        _, per_c, dc_c = errors(net._forward_autograd)
    finally:
        torch.backends.cudnn.allow_tf32 = old
    print(f"\ngolden: loss {loss:.6f} vs {float(g['loss']):.6f}, worst {max(per.values()):.2e} "
          f"({max(per, key=per.get)}), d_cond {dc:.2e}; autograd with cuDNN defaults: worst {max(per_c.values()):.2e} "
          f"({max(per_c, key=per_c.get)}), d_cond {dc_c:.2e}")
    assert max(per.values()) <= BOUND_GOLDEN_TENSOR, (max(per, key=per.get), max(per.values()))
    assert sorted(per.values())[len(per) // 2] <= BOUND_MEDIAN
    assert dc <= BOUND_COND


def _guarded(n, dtype, like=None):
    """A view of n elements in the middle of a buffer whose 64 KiB on each side are 0xFF bytes (NaN as fp16 and fp32),
    and the buffer: a read past the view would bring NaN into the results, a write past it would change the guards."""
    es = torch.empty((), dtype=dtype).element_size()
    gn = 65536 // es
    big = torch.empty((n + 2 * gn) * es, dtype=torch.uint8, device=DEV).fill_(255).view(dtype)
    v = big[gn:gn + n]
    if like is not None:
        v.copy_(like.reshape(-1))
    return big, v, gn


@pytest.mark.parametrize("B,T,cycle,L", [(2, 200, 4, 3), (3, 37, 1, 2), (1, 65, 2, 3)])
def test_no_access_outside_the_buffers(lib_built, B, T, cycle, L):
    """Every input, output, weight, gradient, the tape and the workspace in NaN-guarded buffers: the results equal an
    unguarded run bitwise and the guards are untouched."""
    import ctypes
    from diffsinger_b200 import _capi, train
    from diffsinger_b200.sampler import _stream, _strides_bct
    net = _net(L, cycle)
    step = net._dsx_train_step()
    spec, t, cond, _ = _inputs(B, T)
    cond = cond.contiguous()
    params = {n: p.detach() for n, p in net.named_parameters()}
    d_eps = torch.randn(B, 1, 80, T, device=DEV) / (B * 80 * T)
    eps_ref, tape_ref = step.forward(params, spec, t, cond)
    g_ref, c_ref = step.backward(params, tape_ref, d_eps, B, T)

    bufs = []

    def guard(n, dtype, like=None):
        big, v, gn = _guarded(n, dtype, like)
        bufs.append((big, gn, n))
        return v

    gp = {k: guard(v.numel(), torch.float32, v).view(v.shape) for k, v in params.items()}
    gg = {k: guard(v.numel(), torch.float32).view(v.shape) for k, v in params.items()}
    gspec = guard(spec.numel(), torch.float32, spec).view(spec.shape)
    gcond = guard(cond.numel(), torch.float32, cond).view(cond.shape)
    gd = guard(d_eps.numel(), torch.float32, d_eps).view(d_eps.shape)
    geps = guard(eps_ref.numel(), torch.float32).view(eps_ref.shape)
    gdc = guard(c_ref.numel(), torch.float32).view(c_ref.shape)
    tape = guard(step.tape_bytes(DEV, B, T), torch.uint8)
    ws = guard(step.workspace(DEV, B, T).numel(), torch.uint8)
    keep = []
    w, gs = train._struct(gp, L, keep), train._struct(gg, L, keep)
    h, s = step.handle(DEV), _stream(DEV)
    tt = t.to(torch.int64).contiguous()
    _capi.check(_capi.lib.dsx_train_forward(
        h, ctypes.byref(w), gspec.data_ptr(), _strides_bct(gspec, (0, 2, 3)), tt.data_ptr(), gcond.data_ptr(),
        _strides_bct(gcond, (0, 1, 2)), B, T, tape.data_ptr(), tape.numel(), ws.data_ptr(), ws.numel(),
        geps.data_ptr(), s), "dsx_train_forward")
    ws.fill_(255)                                   # nothing of the forward's scratch may reach the backward
    _capi.check(_capi.lib.dsx_train_backward(
        h, ctypes.byref(w), tape.data_ptr(), gd.data_ptr(), ctypes.byref(gs), gdc.data_ptr(), B, T, ws.data_ptr(),
        ws.numel(), s), "dsx_train_backward")
    torch.cuda.synchronize()
    assert torch.equal(geps, eps_ref)
    assert torch.equal(gdc, c_ref)
    for k in g_ref:
        assert torch.equal(gg[k], g_ref[k]), k
    for big, gn, n in bufs:
        raw = big.view(torch.uint8)
        es = big.element_size()
        assert bool((raw[:gn * es] == 255).all()) and bool((raw[(gn + n) * es:] == 255).all())
