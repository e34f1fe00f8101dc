"""GPU: the FastSpeech2 decoder's training step (dsx_fs2dec_train_*, diffsinger_b200.fs2train) against fp32 autograd of
oracle/fs2dec_train_oracle.py with the masks dsx_fs2dec_train_masks reports, and its exactness properties: scale
invariance, determinism, the keep fraction, zero gradient on padding frames, several forwards before their backwards,
no access outside the buffers, and a short Adam run.

Errors are per-tensor relative Frobenius norms ||dsx - ref|| / ||ref|| over out, d_x and every parameter gradient.  The
same error of TF32 autograd (TF32 matmuls and convolutions) on the same case is printed beside it; dsx rounds GEMM operands to
fp16 (10 mantissa bits, as TF32) and the worst tensor must be within 5e-2 and within 1.5 x TF32's worst.  TF32's worst
is taken as at least FP16_FLOOR = 2^-10, the error of one fp16 rounding of each GEMM operand: at the smallest cases
(1 x 1, 3 x 37) cuBLAS runs autograd's matmuls without tensor cores, so "TF32" autograd is plain fp32 there (median
error 2e-5 at 1 x 1) and its error says nothing about TF32 rounding.

The golden test pins the step to the reference's own gradients (tests/golden/fs2dec_train_grad.npz, written by
oracle/gen_golden_fs2dec_train.py, which also pins the oracle's dropout sites to the reference bit for bit)."""
import numpy as np
import pytest
import torch

from oracle import fs2dec_oracle as O
from oracle.fs2dec_train_oracle import decoder_train

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
FP16_FLOOR = 2.0 ** -10
HP = dict(hidden_size=256, dec_layers=4, dec_ffn_kernel_size=9, num_heads=2, ffn_padding='SAME', ffn_act='gelu',
          dropout=0.1)


def hp_of(H, heads, k, padding, act, L, p=0.1):
    return dict(hidden_size=H, dec_layers=L, dec_ffn_kernel_size=k, num_heads=heads, ffn_padding=padding, ffn_act=act,
                dropout=p)


def model(hp, seed=3):
    from diffsinger_b200 import FastspeechDecoder
    m = FastspeechDecoder(hparams=dict(hp, dsx_train=True))
    sd = O.random_state_dict(seed, hp)
    m.load_state_dict(sd, strict=True)
    return m.train().to(DEV)


def inputs(B, T, H, tail=None, seed=5):
    x = O.fixture_input(seed, B, T, H, tail).to(DEV)
    tgt = torch.from_numpy(np.random.RandomState(seed + 1).standard_normal((B, T, H)).astype(np.float32)).to(DEV)
    return x, tgt


def dsx_step(m, x, tgt, seed):
    """loss = MSE(out, tgt) through the module; -> out, d_x, {name: grad}, the masks of the step"""
    from diffsinger_b200 import fs2train
    orig = fs2train.draw_seed
    fs2train.draw_seed = lambda: seed
    try:
        m.zero_grad(set_to_none=True)
        xr = x.clone().requires_grad_(True)
        out = m(xr)
        ((out - tgt) ** 2).mean().backward()
    finally:
        fs2train.draw_seed = orig
    masks = m._dsx_train_step().masks(DEV, seed, m.dropout, x.shape[0], x.shape[1])
    return out.detach(), xr.grad, {n: p.grad.clone() for n, p in m.named_parameters()}, masks


def ref_step(m, hp, x, tgt, masks, tf32):
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    try:
        sd = {n: p.detach().clone().requires_grad_(True) for n, p in m.named_parameters()}
        xr = x.clone().requires_grad_(True)
        out = decoder_train(sd, xr, hp, masks, hp['dropout'])
        ((out - tgt) ** 2).mean().backward()
        return out.detach(), xr.grad, {n: v.grad for n, v in sd.items()}
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def errors(res, ref):
    out, dx, g = res
    e = {"out": rel(out, ref[0]), "d_x": rel(dx, ref[1])}
    e.update({n: rel(g[n], ref[2][n]) for n in ref[2]})
    return e


def parity(hp, B, T, tail=None, seed=11):
    m = model(hp)
    x, tgt = inputs(B, T, hp['hidden_size'], tail)
    out, dx, g, masks = dsx_step(m, x, tgt, seed)
    ref = ref_step(m, hp, x, tgt, masks, tf32=False)
    tf = ref_step(m, hp, x, tgt, masks, tf32=True)
    e, et = errors((out, dx, g), ref), errors(tf, ref)
    worst, med = max(e.values()), float(np.median(list(e.values())))
    tworst, tmed = max(et.values()), float(np.median(list(et.values())))
    print(f"\nB x T = {B} x {T} p = {hp['dropout']}: dsx worst {worst:.2e} ({max(e, key=e.get)}) median {med:.2e}; "
          f"TF32 autograd worst {tworst:.2e} median {tmed:.2e}")
    assert all(np.isfinite(v) for v in e.values()), e
    assert worst <= 5e-2 and worst <= 1.5 * max(tworst, FP16_FLOOR), (worst, tworst, e)
    pad = x.abs().sum(-1) == 0
    assert (dx[pad] == 0).all()
    return m, x, tgt


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("B,T,tail", [(2, 1000, 700), (3, 37, None), (1, 4000, None), (1, 1, None)])
def test_parity_shipped(p, B, T, tail):
    parity(dict(HP, dropout=p), B, T, tail)


@pytest.mark.parametrize("cfg", [(192, 3, 5, 'SAME', 'relu', 2), (128, 1, 3, 'LEFT', 'gelu', 1),
                                 (64, 1, 1, 'SAME', 'gelu', 3)])
def test_parity_edges(cfg):
    parity(hp_of(*cfg), 2, 150, tail=90)


def raw_step(m, x, seed, d_out):
    """forward and backward through the step without autograd: out, grads, d_x"""
    from diffsinger_b200 import fs2train
    step = m._dsx_train_step()
    params = [p.detach() for p in (dict(m.named_parameters())[n] for n in fs2train.param_names(m.num_layers, m.padding))]
    out, tape = step.forward(params, x, m.dropout, seed)
    grads, dx = step.backward(params, tape, d_out, x.shape[0], x.shape[1])
    return out, grads, dx


def test_scale_invariance_and_zero():
    m = model(HP)
    x, tgt = inputs(2, 300, 256, tail=200)
    g = torch.randn(2, 300, 256, device=DEV) * 1e-4
    _, g1, d1 = raw_step(m, x, 7, g)
    for k in (-20, 13):
        _, g2, d2 = raw_step(m, x, 7, g * 2.0 ** k)
        for a, b in zip(g1 + [d1], g2 + [d2]):
            assert torch.equal(a * 2.0 ** k, b)
    _, g0, d0 = raw_step(m, x, 7, torch.zeros_like(g))
    assert all((t == 0).all() for t in g0 + [d0])


def test_determinism_and_seeds():
    m = model(HP)
    x, _ = inputs(2, 500, 256, tail=321)
    g = torch.randn(2, 500, 256, device=DEV)
    o1, g1, d1 = raw_step(m, x, 99, g)
    o2, g2, d2 = raw_step(m, x, 99, g)
    assert torch.equal(o1, o2) and torch.equal(d1, d2) and all(torch.equal(a, b) for a, b in zip(g1, g2))
    o3, _, _ = raw_step(m, x, 100, g)
    assert not torch.equal(o1, o3)
    step = m._dsx_train_step()
    ma, mb = step.masks(DEV, 99, 0.1, 2, 500), step.masks(DEV, 100, 0.1, 2, 500)
    assert all(not torch.equal(a, b) for a, b in zip(ma, mb))


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_keep_fraction(p):
    m = model(HP)
    masks = m._dsx_train_step().masks(DEV, 1234, p, 4, 1000)
    for mk in masks:
        n = mk.numel()
        frac = mk.float().mean().item()
        assert abs(frac - (1 - p)) <= 6 * (p * (1 - p) / n) ** 0.5, (frac, p, n)


def test_two_forwards_before_backward():
    m = model(HP)
    from diffsinger_b200 import fs2train
    step = m._dsx_train_step()
    params = [p.detach() for p in (dict(m.named_parameters())[n] for n in fs2train.param_names(m.num_layers, m.padding))]
    xa, _ = inputs(2, 200, 256, tail=150, seed=1)
    xb, _ = inputs(3, 90, 256, seed=2)
    ga, gb = torch.randn(2, 200, 256, device=DEV), torch.randn(3, 90, 256, device=DEV)
    _, ta = step.forward(params, xa, 0.1, 5)
    _, tb = step.forward(params, xb, 0.1, 6)
    rb = step.backward(params, tb, gb, 3, 90)
    ra = step.backward(params, ta, ga, 2, 200)
    _, ea, dxa = raw_step(m, xa, 5, ga)
    _, eb, dxb = raw_step(m, xb, 6, gb)
    assert torch.equal(ra[1], dxa) and all(torch.equal(a, b) for a, b in zip(ra[0], ea))
    assert torch.equal(rb[1], dxb) and all(torch.equal(a, b) for a, b in zip(rb[0], eb))


def test_no_access_outside_the_buffers():
    """Every buffer of a step sits between NaN-filled guard regions; the results must equal an unguarded run's bit for
    bit and the guards must stay NaN."""
    from diffsinger_b200 import fs2train
    m = model(HP)
    step = m._dsx_train_step()
    names = fs2train.param_names(m.num_layers, m.padding)
    B, T, H = 2, 130, 256
    x, _ = inputs(B, T, H, tail=77)
    g = torch.randn(B, T, H, device=DEV)
    o_ref, g_ref, d_ref = raw_step(m, x, 8, g)
    GUARD = 4096
    held = []

    def guarded(shape, dtype, src=None):
        n = int(np.prod(shape))
        if dtype == torch.uint8:   # 0xFF bytes: NaN as fp16 and fp32
            base = torch.full((n + 2 * GUARD,), 0xFF, dtype=torch.uint8, device=DEV)
        else:
            base = torch.full((n + 2 * GUARD,), float("nan"), dtype=torch.float32, device=DEV)
        held.append((base, GUARD, n))
        v = base[GUARD:GUARD + n]
        v = v.view(shape)
        if src is not None:
            v.copy_(src)
        return v

    params = [guarded(tuple(p.shape), torch.float32, p.detach()) for p in
              (dict(m.named_parameters())[n] for n in names)]
    xg = guarded((B, T, H), torch.float32, x)
    tape = guarded((step.tape_bytes(DEV, B, T),), torch.uint8)
    n_ws = step.workspace(DEV, B, T).numel()
    ws = guarded((n_ws,), torch.uint8)
    out = guarded((B, T, H), torch.float32)
    import ctypes
    from diffsinger_b200._capi import check, lib
    from diffsinger_b200.sampler import _ptr, _stream, _strides_bct
    keep = []
    w = fs2train._struct(params, m.num_layers, keep)
    h = step.handle(DEV)
    check(lib.dsx_fs2dec_train_forward(h, ctypes.byref(w), _ptr(xg), _strides_bct(xg, (0, 2, 1)), B, T, 0.1, 8,
                                       _ptr(tape), tape.numel(), _ptr(ws), ws.numel(), _ptr(out), _stream(DEV)))
    grads = [guarded(tuple(p.shape), torch.float32) for p in params]
    gw = fs2train._struct(grads, m.num_layers, keep)
    dg = guarded((B, T, H), torch.float32, g)
    dx = guarded((B, T, H), torch.float32)
    check(lib.dsx_fs2dec_train_backward(h, ctypes.byref(w), _ptr(tape), _ptr(dg), ctypes.byref(gw), _ptr(dx), B, T,
                                        _ptr(ws), ws.numel(), _stream(DEV)))
    torch.cuda.synchronize()
    assert torch.equal(out, o_ref) and torch.equal(dx, d_ref)
    assert all(torch.equal(a, b) for a, b in zip(grads, g_ref))
    for base, gsz, n in held:
        if base.dtype == torch.uint8:
            assert (base[:gsz] == 0xFF).all() and (base[gsz + n:] == 0xFF).all()
        else:
            assert torch.isnan(base[:gsz]).all() and torch.isnan(base[gsz + n:]).all()


def test_adam_tracks_fp32_autograd():
    """20 Adam steps of decoder + Linear(256, 80) + L1 on a fixed batch, p = 0.1 with the step's masks in the fp32 run"""
    torch.manual_seed(0)
    m = model(HP)
    head = torch.nn.Linear(256, 80).to(DEV)
    ref_sd = {n: p.detach().clone().requires_grad_(True) for n, p in m.named_parameters()}
    ref_head = torch.nn.Linear(256, 80).to(DEV)
    ref_head.load_state_dict(head.state_dict())
    x, _ = inputs(4, 300, 256, tail=250)
    y = torch.from_numpy(np.random.RandomState(9).standard_normal((4, 300, 80)).astype(np.float32)).to(DEV)
    opt = torch.optim.Adam(list(m.parameters()) + list(head.parameters()), lr=3e-4)
    ropt = torch.optim.Adam(list(ref_sd.values()) + list(ref_head.parameters()), lr=3e-4)
    from diffsinger_b200 import fs2train
    orig = fs2train.draw_seed
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    la, lb = [], []
    try:
        for it in range(20):
            seed = 1000 + it
            fs2train.draw_seed = (lambda s: (lambda: s))(seed)
            opt.zero_grad()
            loss = (head(m(x)) - y).abs().mean()
            loss.backward()
            opt.step()
            la.append(loss.item())
            masks = m._dsx_train_step().masks(DEV, seed, 0.1, 4, 300)
            ropt.zero_grad()
            rl = (ref_head(decoder_train(ref_sd, x, HP, masks, 0.1)) - y).abs().mean()
            rl.backward()
            ropt.step()
            lb.append(rl.item())
    finally:
        fs2train.draw_seed = orig
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu
    print("\ndsx  ", " ".join(f"{v:.4f}" for v in la), "\nfp32 ", " ".join(f"{v:.4f}" for v in lb))
    assert la[-1] < la[0] - 0.02
    assert max(abs(a - b) / b for a, b in zip(la, lb)) < 5e-3


def test_golden_reference_gradients():
    """p = 0 at 2 x 40 (utterance 1 padded from frame 29): the loss, d_x and per parameter the norm and 64 sampled
    entries of the reference's own fp32 gradients"""
    from conftest import golden
    from oracle.gen_golden_train import sample_index
    g = golden("fs2dec_train_grad.npz")
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    hp["dropout"] = 0.0
    B, T = int(g["B"]), int(g["T"])
    m = model(hp, seed=int(g["seed"]))
    x = O.fixture_input(int(g["input_seed"]), B, T, 256, tail=int(g["tail"])).to(DEV)
    tgt = torch.from_numpy(np.random.RandomState(int(g["input_seed"]) + 1).standard_normal((B, T, 256))
                           .astype(np.float32)).to(DEV)
    out, dx, grads, _ = dsx_step(m, x, tgt, 1)
    loss = ((out - tgt) ** 2).mean().item()
    assert abs(loss - float(g["loss"])) <= 1e-3 * abs(float(g["loss"]))
    errs = {"d_x": rel(dx.cpu(), torch.from_numpy(g["d_x"]))}
    for n, v in grads.items():
        flat = v.reshape(-1).cpu()
        errs["norm." + n] = abs(flat.norm().item() - float(g["norm." + n])) / float(g["norm." + n])
        errs["val." + n] = rel(flat[torch.from_numpy(sample_index(n, flat.numel())).long()], torch.from_numpy(g["val." + n]))
    worst = max(errs, key=errs.get)
    print(f"\ngolden: worst {errs[worst]:.2e} ({worst}), median {float(np.median(list(errs.values()))):.2e}")
    assert errs[worst] <= 5e-2, errs


def test_refusals_on_the_gpu():
    import copy
    from diffsinger_b200 import DsxError
    m = model(HP)
    x, tgt = inputs(1, 50, 256)
    xr = x.clone().requires_grad_(True)
    out = m(xr)
    with pytest.raises(DsxError, match="double backward"):
        torch.autograd.grad((out ** 2).mean(), xr, create_graph=True)
    copy.deepcopy(m)                                                        # handles are not copied
    empty = m(torch.zeros(0, 7, 256, device=DEV))
    assert empty.shape == (0, 7, 256)
    w = m.layers[0].op.self_attn.in_proj_weight
    w.data = w.data.t().contiguous().t()
    with pytest.raises(DsxError, match="contiguous"):
        m(x)


def test_backward_with_another_shape_gives_nan():
    m = model(HP)
    from diffsinger_b200 import fs2train
    step = m._dsx_train_step()
    params = [p.detach() for p in (dict(m.named_parameters())[n] for n in fs2train.param_names(m.num_layers, m.padding))]
    x, _ = inputs(2, 100, 256)
    _, tape = step.forward(params, x, 0.1, 3)
    grads, dx = step.backward(params, tape, torch.randn(2, 99, 256, device=DEV), 2, 99)
    assert torch.isnan(dx).all() and all(torch.isnan(v).all() for v in grads)


def test_dropin_trains_through_fastspeech2(lib_built, tmp_path, monkeypatch):
    """install_fs2_decoder() on the stand-in tree, a strict load, then training steps under dsx_train: the decoder's
    gradient reaches the module that produced decoder_inp, and matches fp32 autograd with the step's masks"""
    import sys
    import textwrap
    from test_gpu_fs2dec import STANDIN
    for rel_, body in STANDIN.items():
        f = tmp_path / rel_
        f.parent.mkdir(parents=True, exist_ok=True)
        f.write_text(textwrap.dedent(body).lstrip("\n"))
    monkeypatch.syspath_prepend(str(tmp_path))
    roots = ("modules", "utils")
    drop = lambda: [n for n in sys.modules if n in roots or n.startswith(tuple(r + "." for r in roots))]
    for n in drop():
        monkeypatch.delitem(sys.modules, n)
    import utils.hparams
    utils.hparams.hparams.update(dict(HP, dsx_train=True))
    import modules.fastspeech.fs2 as fs2
    import diffsinger_b200.dropin as dropin
    from diffsinger_b200 import fs2train
    new_cls = dropin.install_fs2_decoder()
    try:
        net = fs2.FastSpeech2()
        assert type(net.decoder) is new_cls and net.decoder._dsx_train
        sd = O.random_state_dict(3, HP)
        net.decoder.load_state_dict(sd, strict=True)
        net = net.to(DEV).train()
        enc = torch.nn.Linear(32, 256).to(DEV)                 # stands in for the encoder + embeddings
        src = torch.randn(2, 120, 32, device=DEV)
        nonpad = torch.ones(2, 120, 1, device=DEV)
        nonpad[1, 90:] = 0
        y = torch.randn(2, 120, 80, device=DEV)
        orig = fs2train.draw_seed
        fs2train.draw_seed = lambda: 77
        try:
            loss = (net.mel_out(net.decoder(enc(src) * nonpad)) - y).abs().mean()
            loss.backward()
        finally:
            fs2train.draw_seed = orig
        assert enc.weight.grad is not None and enc.weight.grad.abs().sum() > 0
        masks = net.decoder._dsx_train_step().masks(DEV, 77, HP['dropout'], 2, 120)
        ref_enc = torch.nn.Linear(32, 256).to(DEV)
        ref_enc.load_state_dict(enc.state_dict())
        ref_sd = {n: p.detach().clone().requires_grad_(True) for n, p in net.decoder.named_parameters()}
        mm = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            rl = (net.mel_out(decoder_train(ref_sd, ref_enc(src) * nonpad, HP, masks, HP['dropout'])) - y).abs().mean()
            rl.backward()
        finally:
            torch.backends.cuda.matmul.allow_tf32 = mm
        assert abs(loss.item() - rl.item()) <= 1e-3 * rl.item()
        assert rel(enc.weight.grad, ref_enc.weight.grad) <= 5e-2
        for n, p in net.decoder.named_parameters():
            assert rel(p.grad, ref_sd[n].grad) <= 5e-2, n
        opt = torch.optim.Adam(list(net.parameters()) + list(enc.parameters()), lr=1e-3)
        losses = []
        for _ in range(10):
            opt.zero_grad()
            lo = (net.mel_out(net.decoder(enc(src) * nonpad)) - y).abs().mean()
            lo.backward()
            opt.step()
            losses.append(lo.item())
        assert losses[-1] < losses[0]
    finally:
        dropin.uninstall_fs2_decoder()
    for n in drop():
        del sys.modules[n]
