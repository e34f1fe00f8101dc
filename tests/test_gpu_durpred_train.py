"""GPU: the duration predictor training step (dsx_durpred_train_*, diffsinger_b200.durtrain) against autograd of
oracle/durpred_train_oracle.py with the masks the step reports.

Parity: per tensor (xs, d_x and every gradient) the relative Frobenius error; the worst tensor must be within 5e-2 and
within 1.5x the worst of TF32 autograd on the same case (taken as at least 2^-10).  The reference is autograd of the
oracle whose convolutions take fp16-rounded operands, as dsx_durpred_forward rounds them and as the training forward
must (its xs equals the eval forward's bit for bit at p = 0), in fp32; tests/test_gpu_train_edges.py holds the edges of
the accepted configurations to float64.  oracle/precision_study_durtrain.py shows why the rounding belongs in the
reference: it flips the sign of 1e-4 to 3e-4 of the ReLU inputs against an unrounded forward, which moves the
gradients of five layers by about 4.5e-2 whatever the backward's format (TF32 autograd, whose forward rounds the same
mantissa, moves them as much), while the backward's scaled fp16 operands alone cost 6.7e-4.  The shipped predictors
(ds100_adj_rel at 16 x 250, the 2-layer one) are also held to the same bound against the unrounded fp32 oracle.  Then
the exact properties (2^k scale invariance, zero in zero out, bitwise reproducibility, several forwards before their
backwards, guard regions, the (B, T) check, p = 0 against the eval forward, the keep fraction), the reference's
fixture, a short Adam run, and the drop-in chain encoder -> predictor with predictor_grad 0.1."""
import ctypes

import numpy as np
import pytest
import torch

from oracle.durpred_train_oracle import durpred_train

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
HP = dict(dur_loss='mse')


def model(idim=256, L=5, P=256, k=3, padding='SAME', p=0.5, seed=3):
    from diffsinger_b200 import DurationPredictor
    from oracle.gen_golden_durpred_train import random_state_dict
    m = DurationPredictor(idim, L, P, k, p, padding=padding, hparams=HP, train=True)
    sd = random_state_dict(seed, idim, L, P, k)
    m.load_state_dict(sd, strict=True)
    return m.to(DEV).train()


def inputs(B, T, idim, tails=(), seed=5):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, idim, generator=g)
    mask = torch.zeros(B, T, dtype=torch.bool)
    for b, t in tails:
        mask[b, t:] = True
    d = torch.randn(B, T, generator=g)
    return x.to(DEV), mask.to(DEV), d.to(DEV)


def raw_step(m, x, mask, d_xs, seed, p=None):
    """xs, grads (param_names order), d_x and the masks of one dsx step"""
    from diffsinger_b200 import durtrain
    step = m._dsx_train_step()
    names = durtrain.param_names(m._cfg.layers)
    params = [dict(m.named_parameters())[n].detach() for n in names]
    p = m.dropout_rate if p is None else p
    xs, tape = step.forward(params, x, mask.to(torch.uint8).contiguous(), p, seed)
    B, T, _ = x.shape
    grads, d_x = step.backward(params, tape, d_xs, B, T)
    return xs, grads, d_x, step.masks(DEV, seed, p, B, T)


def ref_step(m, x, mask, d_xs, masks, p, dtype=torch.float32, tf32=False, fp16=True):
    from diffsinger_b200 import durtrain
    names = durtrain.param_names(m._cfg.layers)
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    try:
        sd = {n: v.detach().to(dtype).clone().requires_grad_(True) for n, v in m.named_parameters()}
        xr = x.detach().to(dtype).clone().requires_grad_(True)
        xs = durpred_train(sd, xr, mask, masks, p, m._cfg.kernel, m.padding, fp16=fp16)
        xs.backward(d_xs.to(dtype))
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu
    return xs.detach(), [sd[n].grad for n in names], xr.grad


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def worst(res, ref):
    xs, grads, d_x = res[:3]
    rx, rg, rd = ref[:3]
    errs = [rel(xs, rx), rel(d_x, rd)] + [rel(a, b) for a, b in zip(grads, rg) if b.norm() > 0]
    return max(errs)


def check_parity(m, B, T, tails, seed=11, dtype=torch.float32, unrounded=False):
    x, mask, d = inputs(B, T, m._cfg.idim, tails)
    res = raw_step(m, x, mask, d, seed)
    masks = res[3]
    for fp16 in (True, False) if unrounded else (True,):
        ref = ref_step(m, x, mask, d, masks, m.dropout_rate, dtype, fp16=fp16)
        tf = ref_step(m, x, mask, d, masks, m.dropout_rate, torch.float32, tf32=True, fp16=fp16)
        e_dsx, e_tf = worst(res, ref), worst(tf, ref)
        bound = min(5e-2, 1.5 * max(e_tf, 2 ** -10))
        print(f"parity B {B} T {T} {m._cfg.idim}->{m._cfg.chans} L {m._cfg.layers} k {m._cfg.kernel} {dtype} "
              f"{'fp16 operands' if fp16 else 'unrounded'}: dsx {e_dsx:.2e} TF32 {e_tf:.2e} bound {bound:.2e}")
        assert e_dsx <= bound, (fp16, e_dsx, e_tf)
    return res, ref


@pytest.mark.parametrize("case", ["ds100_16x250", "tts_2layer", "all_padding", "T1", "T_below_k"])
def test_parity(case):
    if case == "ds100_16x250":
        m, B, T, tails = model(), 16, 250, [(b, 250 - 13 * b) for b in range(1, 16)]
    elif case == "tts_2layer":
        m, B, T, tails = model(L=2), 8, 120, [(1, 70), (5, 3)]
    elif case == "all_padding":
        m, B, T, tails = model(), 3, 50, [(1, 0), (2, 30)]
    elif case == "T1":
        m, B, T, tails = model(), 4, 1, [(2, 0)]
    else:
        m, B, T, tails = model(k=5), 3, 3, [(1, 2)]
    res, ref = check_parity(m, B, T, tails, unrounded=case in ("ds100_16x250", "tts_2layer"))
    if case == "all_padding":
        assert torch.equal(res[0][1], torch.zeros_like(res[0][1]))
        # nothing of utterance 1 reaches a gradient, and no gradient reaches its input
        assert torch.equal(res[2][1], torch.zeros_like(res[2][1]))


def test_scale_invariance_and_zero():
    m = model()
    x, mask, d = inputs(4, 100, 256, [(1, 60)])
    base = raw_step(m, x, mask, d, 7)
    for k in (-9, 13):
        r = raw_step(m, x, mask, d * 2.0 ** k, 7)
        assert all(torch.equal(a * 2.0 ** k, b) for a, b in zip(base[1], r[1]))
        assert torch.equal(base[2] * 2.0 ** k, r[2])
    z = raw_step(m, x, mask, torch.zeros_like(d), 7)
    assert all(torch.count_nonzero(g) == 0 for g in z[1]) and torch.count_nonzero(z[2]) == 0


def test_two_backwards_of_one_tape_and_several_forwards():
    from diffsinger_b200 import durtrain
    m = model()
    step = m._dsx_train_step()
    params = [dict(m.named_parameters())[n].detach() for n in durtrain.param_names(5)]
    x1, mask1, d1 = inputs(4, 90, 256, [(2, 40)], seed=1)
    x2, mask2, d2 = inputs(4, 90, 256, [(0, 10)], seed=2)
    u8 = lambda mk: mk.to(torch.uint8).contiguous()
    a1, t1 = step.forward(params, x1, u8(mask1), 0.5, 21)
    g1, dx1 = step.backward(params, t1, d1, 4, 90)
    g1b, dx1b = step.backward(params, t1, d1, 4, 90)
    assert torch.equal(dx1, dx1b) and all(torch.equal(a, b) for a, b in zip(g1, g1b))
    b1, s1 = step.forward(params, x1, u8(mask1), 0.5, 21)
    b2, s2 = step.forward(params, x2, u8(mask2), 0.5, 22)
    mask1.fill_(True)                     # the tape holds its own copy of the mask
    h2, hx2 = step.backward(params, s2, d2, 4, 90)
    h1, hx1 = step.backward(params, s1, d1, 4, 90)
    assert torch.equal(a1, b1) and torch.equal(hx1, dx1) and all(torch.equal(a, b) for a, b in zip(h1, g1))
    a2, t2 = step.forward(params, x2, u8(mask2), 0.5, 22)
    g2, dx2 = step.backward(params, t2, d2, 4, 90)
    assert torch.equal(a2, b2) and torch.equal(hx2, dx2) and all(torch.equal(a, b) for a, b in zip(h2, g2))


def test_no_access_outside_the_buffers():
    """Every buffer of a step sits between guard regions; the results must equal an unguarded run's bit for bit and the
    guards must stay untouched."""
    guarded_step(128, 192, 3, 5, 'SAME', 130, 77)


@pytest.mark.parametrize("idim,P,L,k,padding,T,tail", [(80, 144, 3, 31, 'LEFT', 3, 1),
                                                       (240, 240, 3, 9, 'SAME', 129, 97)])
def test_no_access_outside_the_buffers_at_edges(idim, P, L, k, padding, T, tail):
    """test_no_access_outside_the_buffers at ragged column tiles with 31 LEFT taps over T = 3, and at 240 channels"""
    guarded_step(idim, P, L, k, padding, T, tail)


def guarded_step(idim, P, L, k, padding, T, tail):
    """one step of B = 3 (utterance 1 padding from `tail` on) with every buffer between guard regions"""
    from diffsinger_b200 import durtrain
    from diffsinger_b200._capi import check, lib
    from diffsinger_b200.sampler import _ptr, _stream, _strides_bct
    m = model(idim=idim, P=P, L=L, k=k, padding=padding)
    step = m._dsx_train_step()
    names = durtrain.param_names(L)
    B = 3
    x, mask, d = inputs(B, T, idim, [(1, tail)])
    xs_ref, g_ref, d_ref, _ = raw_step(m, x, mask, d, 8)
    GUARD = 4096
    held = []

    def guarded(shape, dtype, src=None):
        n = int(np.prod(shape))
        fill = 0xFF if dtype == torch.uint8 else float("nan")
        base = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device=DEV)
        held.append((base, n))
        v = base[GUARD:GUARD + n].view(shape)
        if src is not None:
            v.copy_(src)
        return v

    named = dict(m.named_parameters())
    params = [guarded(tuple(named[n].shape), torch.float32, named[n].detach()) for n in names]
    xg = guarded((B, T, idim), torch.float32, x)
    mg = guarded((B, T), torch.uint8, mask.to(torch.uint8))
    tape = guarded((step.tape_bytes(DEV, B, T),), torch.uint8)
    ws = guarded((step.workspace(DEV, B, T).numel(),), torch.uint8)
    xs = guarded((B, T), torch.float32)
    keep = []
    w = durtrain._struct(params, L, keep)
    h = step.handle(DEV)
    check(lib.dsx_durpred_train_forward(h, ctypes.byref(w), _ptr(xg), _strides_bct(xg, (0, 2, 1)), _ptr(mg), B, T, 0.5,
                                        8, _ptr(tape), tape.numel(), _ptr(ws), ws.numel(), _ptr(xs), _stream(DEV)))
    grads = [guarded(tuple(p.shape), torch.float32) for p in params]
    gw = durtrain._struct(grads, L, keep)
    dg = guarded((B, T), torch.float32, d)
    dx = guarded((B, T, idim), torch.float32)
    check(lib.dsx_durpred_train_backward(h, ctypes.byref(w), _ptr(tape), _ptr(dg), ctypes.byref(gw), _ptr(dx), B, T,
                                         _ptr(ws), ws.numel(), _stream(DEV)))
    torch.cuda.synchronize()
    assert torch.equal(xs, xs_ref) and torch.equal(dx, d_ref)
    assert all(torch.equal(a, b) for a, b in zip(grads, g_ref))
    for base, n in held:
        for part in (base[:GUARD], base[GUARD + n:]):
            assert torch.isnan(part).all() if base.dtype == torch.float32 else (part == 0xFF).all()


def test_backward_with_another_shape_gives_nan():
    from diffsinger_b200 import durtrain
    m = model()
    step = m._dsx_train_step()
    params = [dict(m.named_parameters())[n].detach() for n in durtrain.param_names(5)]
    x, mask, d = inputs(4, 100, 256, [(1, 60)])
    _, tape = step.forward(params, x, mask.to(torch.uint8).contiguous(), 0.5, 3)
    grads, d_x = step.backward(params, tape, d[:, :90].contiguous(), 4, 90)
    assert all(torch.isnan(g).all() for g in grads) and torch.isnan(d_x).all()


def test_p0_forward_matches_the_eval_forward():
    from diffsinger_b200 import DurationPredictor
    m = model(p=0.0)
    x, mask, d = inputs(16, 250, 256, [(b, 250 - 13 * b) for b in range(16)])
    xs = raw_step(m, x, mask, d, 5)[0]
    ev = DurationPredictor(256, 5, 256, 3, 0.0, hparams=HP).to(DEV)
    ev.load_state_dict(m.state_dict())
    with torch.no_grad():
        assert torch.equal(xs, ev.eval()(x, mask))


def test_keep_fraction():
    m = model(P=256)
    masks = m._dsx_train_step().masks(DEV, 99, 0.5, 16, 250)
    assert len(masks) == 5
    for mk in masks:
        assert abs(mk.float().mean().item() - 0.5) < 0.01
    assert not torch.equal(masks[0], masks[1])
    m3 = m._dsx_train_step().masks(DEV, 99, 0.1, 16, 250)
    assert abs(m3[0].float().mean().item() - 0.9) < 0.01


@pytest.mark.parametrize("case", ["midi", "tts"])
def test_golden_reference_gradients(case):
    """The module at p = 0 on the fixture's inputs against the reference's own gradients (float32 on the CPU)"""
    from conftest import golden
    from diffsinger_b200 import durtrain
    from oracle import gen_golden_durpred_train as G
    from oracle.gen_golden_train import sample_index
    g = golden("durpred_train_grad.npz")
    cfg = dict((c, f) for c, _, f in G.CASES)[case]
    m = model(*[cfg[i] for i in (0, 1, 2, 3)], padding=cfg[4], p=0.0)
    m.load_state_dict(G.random_state_dict(G.SEED, *cfg[:4]))
    x, mask, tgt = (t.to(DEV) for t in G.case_inputs(cfg))
    xr = x.clone().requires_grad_(True)
    xs = m(xr, mask)
    loss = ((xs - tgt) ** 2).mean()
    loss.backward()
    pre = f"{case}.p0."
    assert rel(xs.detach().cpu(), torch.from_numpy(g[pre + "xs"])) < 2e-2
    assert rel(xr.grad.cpu(), torch.from_numpy(g[pre + "d_x"])) < 5e-2
    assert xr.grad[1, G.TAIL].abs().sum() > 0
    for n in durtrain.param_names(cfg[1]):
        v = dict(m.named_parameters())[n].grad.reshape(-1).cpu()
        ref = float(g[pre + "norm." + n])
        assert abs(v.norm().item() - ref) <= 5e-2 * ref, n
        idx = torch.from_numpy(sample_index(n, v.numel())).long()
        assert rel(v[idx], torch.from_numpy(g[pre + "val." + n])) < 1e-1, n


def test_adam_lowers_the_duration_loss():
    m = model(L=2)
    x, mask, _ = inputs(16, 60, 256, [(b, 60 - 3 * b) for b in range(16)])
    tgt = torch.log(torch.randint(1, 20, (16, 60), device=DEV).float() + 1)
    nonpad = (~mask).float()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        xs = m(x, mask)
        loss = (((xs - tgt) ** 2) * nonpad).sum() / nonpad.sum()      # the pdur loss (dur_loss 'mse')
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.5 * losses[0], losses


def test_dropin_chain_encoder_to_predictor(monkeypatch):
    """FastSpeech2.add_dur under dsx_train on a stand-in tree: dsx MIDI encoder (p = 0) -> (enc * nonpad) with
    predictor_grad 0.1 -> dsx DurationPredictor (p = 0.5).  The encoder's gradients carry 0.1 d_x of the predictor and
    match the same chain with the oracle predictor (fp32 autograd, the step's masks) within the parity bound."""
    from diffsinger_b200 import FastspeechMIDIEncoder, durtrain
    from oracle import fs2enc_oracle as O
    from test_gpu_fs2enc_train import HP as ENC_HP, model as enc_model
    seed = 1234
    monkeypatch.setattr(durtrain, "draw_seed", lambda: seed)
    enc, sd_enc = enc_model(dict(ENC_HP, dropout=0.0))
    assert isinstance(enc, FastspeechMIDIEncoder)
    dp = model()
    B, T = 4, 40
    g = torch.Generator().manual_seed(3)
    tok = torch.randint(1, 50, (B, T), generator=g)
    tok[1, 25:] = 0
    tok, tgt = tok.to(DEV), torch.randn(B, T, generator=g).to(DEV)
    pad = tok.eq(0)

    def run(pred):
        enc.zero_grad()
        out = enc(tok, 0, 0, 0)
        dur_input = out * (~pad).float()[:, :, None]
        dur_input = dur_input.detach() + 0.1 * (dur_input - dur_input.detach())      # fs2.py:161
        xs = pred(dur_input)
        loss = (((xs - tgt) ** 2) * (~pad).float()).sum() / (~pad).float().sum()
        loss.backward()
        return [p.grad.clone() for p in enc.parameters() if p.grad is not None]

    dsx = run(lambda d: dp(d, pad))
    masks = dp._dsx_train_step().masks(DEV, seed, 0.5, B, T)
    sd = {n: v.detach() for n, v in dp.named_parameters()}
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        eager = run(lambda d: durpred_train(sd, d, pad, masks, 0.5, 3))
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu
    assert len(dsx) == len(eager) > 0 and all(e.norm() > 0 for e in eager)
    assert max(rel(a, b) for a, b in zip(dsx, eager)) < 5e-2


def test_refusals_on_the_device():
    from diffsinger_b200 import DsxError
    x, mask, _ = inputs(2, 10, 256)
    m = model().double()
    with pytest.raises(DsxError, match="fp32"):
        m(x.double(), mask)
    m = model()
    w = m.conv[0][1].weight
    w.data = w.data.transpose(0, 1).contiguous().transpose(0, 1)
    with pytest.raises(DsxError, match="contiguous"):
        m(x, mask)
    with pytest.raises(DsxError, match="fp32 xs"):
        model()(x.half().requires_grad_(True), mask)
    xs = model()(x.requires_grad_(True), mask)
    with pytest.raises(DsxError, match="double backward"):
        g, = torch.autograd.grad(xs.sum(), x, create_graph=True)
