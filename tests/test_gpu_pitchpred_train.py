"""GPU: the pitch and energy predictors (dsx_pitchpred_*, dsx_pitchpred_train_*, diffsinger_b200.pitchpred) against
autograd of oracle/pitchpred_train_oracle.py with the masks the step reports.

Parity: per tensor (the output, d_x and every gradient, d pos_embed_alpha's included) the relative Frobenius error
against float64 autograd of the oracle whose convolutions take fp16-rounded operands, as the eval forward rounds them and
the training forward must (at p = 0 it equals the eval forward bit for bit).  The bound is the rule of
oracle/precision_study_pitchtrain.py: the step's error is the fp32 forward's sensitivity to how it is evaluated (ReLU and
LayerNorm flips, which depend on the instance) plus the fp16 backward's own cost (at most 4.9e-4 in the study).  The
first is measured on each case as the worst of TF32 autograd and fp32 autograd under ORDERS relabelings of the hidden
channels, each with the reference's sinusoidal table and with the table as the kernel evaluates it (its last bits move
the fp16 rounding of some layer-0 operands); the bound is twice the sum, at most 5e-2.  d pos_embed_alpha is also checked against a float64 sum of the
step's own d_x . table[pos], to fp32 summation.  Cases: 16 x 1000 frames of the aux_rel frame predictor with ragged utterances, T = 1, T < k, an utterance of zero frames, a real frame whose channel 0 is exactly 0,
T > 4096 (past the reference table's init_size), the 'ph', CWT and LEFT predictors.  Then the eval forward against the
reference's, the exact properties (p = 0 against the eval forward, 2^k scale invariance, zero in zero out, bitwise
reproducibility, several forwards before their backwards, the (B, T) check, the keep fraction, guard regions), the
reference's fixture, a short Adam run on the f0 + uv loss, the hand-built chain encoder -> predictor with predictor_grad 0.1,
and the refusals."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle.pe_oracle import make_positions, sinusoidal_table
from oracle.pitchpred_train_oracle import INIT_SIZE, pitchpred_train

pytestmark = pytest.mark.gpu
ORDERS = 4                     # fp32 summation orders (hidden-channel relabelings) per parity case
DEV = torch.device("cuda", 0)
HP = dict(dsx_train=False)


def model(idim=256, L=5, P=256, odim=2, k=5, padding='SAME', p=0.5, seed=3, cls=None):
    from diffsinger_b200 import PitchPredictor
    from oracle.gen_golden_pitchpred_train import random_state_dict
    m = (cls or PitchPredictor)(idim, L, P, odim, k, p, padding, hparams=HP, train=True)
    m.load_state_dict(random_state_dict(seed, idim, L, P, odim, k), strict=True)
    return m.to(DEV).train()


def inputs(B, T, idim, odim, tails=(), seed=5):
    """x [B, T, idim] zero from each (b, t) tail on (padding frames, as FastSpeech2 feeds them), d_out [B, T, odim]"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, idim, generator=g)
    for b, t in tails:
        x[b, t:] = 0
    d = torch.randn(B, T, odim, generator=g)
    return x.to(DEV), d.to(DEV)


def raw_step(m, x, d_out, seed, p=None):
    """out, grads (param_names order), d_x and the masks of one dsx step"""
    from diffsinger_b200 import pitchpred
    step = m._dsx_train_step()
    params = [dict(m.named_parameters())[n].detach() for n in pitchpred.param_names(m._cfg.layers)]
    p = m.dropout_rate if p is None else p
    out, tape = step.forward(params, x.contiguous(), p, seed)
    B, T, _ = x.shape
    grads, d_x = step.backward(params, tape, d_out, B, T)
    return out, grads, d_x, step.masks(DEV, seed, p, B, T)


def kernel_table(T, H):
    """the sinusoidal table as k_pos_add evaluates it: sinf / cosf of float(ps) * expf(i * neg_emb) in fp32, on the device"""
    neg = torch.tensor(-math.log(10000.0) / (H // 2 - 1), dtype=torch.float32).to(DEV)
    freq = torch.exp(torch.arange(H // 2, device=DEV, dtype=torch.float32) * neg)
    arg = torch.arange(1 + T, device=DEV, dtype=torch.float32)[:, None] * freq[None, :]
    t = torch.cat([torch.sin(arg), torch.cos(arg)], 1)
    t[0] = 0
    return t


def ref_step(m, x, d_out, masks, p, dtype=torch.float64, tf32=False, fp16=True, perm=None, table=None):
    """out, grads (param_names order) and d_x of autograd of the oracle; perm relabels the hidden channels (the same
    function, another fp32 summation order in every conv and LayerNorm), and the gradients are mapped back"""
    from diffsinger_b200 import pitchpred
    names = pitchpred.param_names(m._cfg.layers)
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    try:
        sd = {n: v.detach().to(dtype).clone() for n, v in m.named_parameters()}
        if perm is not None:
            for n in sd:
                if n.startswith("conv."):
                    sd[n] = sd[n][perm]
                    if n.endswith(".1.weight") and not n.startswith("conv.0."):
                        sd[n] = sd[n][:, perm]
            sd["linear.weight"] = sd["linear.weight"][:, perm]
            masks = [mk[..., perm] for mk in masks]
        sd = {n: v.contiguous().requires_grad_(True) for n, v in sd.items()}
        xr = x.detach().to(dtype).clone().requires_grad_(True)
        out = pitchpred_train(sd, xr, masks, p, m._cfg.kernel, m.padding, fp16=fp16, table=table)
        out.backward(d_out.to(dtype))
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu
    grads = {n: v.grad for n, v in sd.items()}
    if perm is not None:
        inv = torch.argsort(perm)
        for n in grads:
            if n.startswith("conv."):
                grads[n] = grads[n][inv]
                if n.endswith(".1.weight") and not n.startswith("conv.0."):
                    grads[n] = grads[n][:, inv]
        grads["linear.weight"] = grads["linear.weight"][:, inv]
    return out.detach(), [grads[n] for n in names], xr.grad


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def alpha_terms(x, d_x):
    """d_x . table[pos] per element, in float64: d pos_embed_alpha is their sum"""
    B, T, H = x.shape
    table = sinusoidal_table(max(INIT_SIZE, 1 + T), H, dtype=torch.float64).to(DEV)
    pos = make_positions(x[..., 0])
    return d_x.double() * table.index_select(0, pos.view(-1)).view(B, T, H)


def check_alpha_is_its_own_sum(x, res):
    """dsx's d pos_embed_alpha against a float64 sum of dsx's own d_x . table[pos]: they differ by fp32 summation only"""
    own = alpha_terms(x, res[2]).sum().item()
    a = res[1][-1].double().item()
    assert abs(a - own) <= 1e-3 * abs(own) + 1e-30, (a, own)


def errors(res, ref):
    """per-tensor relative errors: out, d_x, every gradient, d pos_embed_alpha against |d pos_embed_alpha|"""
    out, grads, d_x = res[:3]
    ro, rg, rd = ref[:3]
    errs = [rel(out, ro), rel(d_x, rd) if rd.norm() > 0 else d_x.abs().max().item()]
    errs += [rel(a, b) for a, b in zip(grads, rg) if b.norm() > 0]
    return errs


def check_parity(m, B, T, tails, case, seed=11, x=None):
    """the rule of oracle/precision_study_pitchtrain.py: the step's error is the fp32 forward's sensitivity to its
    summation order plus the fp16 backward's own cost.  The first is measured here, as the worst of fp32 autograd under
    ORDERS relabelings of the hidden channels and of TF32 autograd; the second is the study's, per configuration."""
    from oracle.precision_study_pitchtrain import STUDY
    xd, d = inputs(B, T, m._cfg.idim, m._cfg.odim, tails)
    x = xd if x is None else x
    res = raw_step(m, x, d, seed)
    check_alpha_is_its_own_sum(x, res)
    masks = res[3]
    ref = ref_step(m, x, d, masks, m.dropout_rate)
    spread = max(errors(ref_step(m, x, d, masks, m.dropout_rate, torch.float32, tf32=True), ref))
    g = torch.Generator().manual_seed(0)
    ktab = kernel_table(T, m._cfg.idim)
    for i in range(ORDERS):
        perm = torch.randperm(m._cfg.chans, generator=g).to(DEV)
        for tab in (None, ktab):
            e = errors(ref_step(m, x, d, masks, m.dropout_rate, torch.float32, perm=perm if i else None, table=tab), ref)
            spread = max(spread, max(e))
    e_dsx = max(errors(res, ref))
    bound = min(5e-2, 2 * (spread + STUDY[case][0]))
    c = m._cfg
    print(f"parity B {B} T {T} {c.idim}->{c.chans} L {c.layers} k {c.kernel} odim {c.odim}: dsx {e_dsx:.2e} "
          f"fp32 order spread {spread:.2e} bound {bound:.2e}")
    assert e_dsx <= bound, (e_dsx, spread, errors(res, ref))
    return res, ref


@pytest.mark.parametrize("case", ["aux_rel_16x1000", "T1", "T_below_k", "all_padding", "zero_channel0", "T_above_4096",
                                  "ph", "cwt", "left"])
def test_parity(case):
    x = None
    if case == "aux_rel_16x1000":
        m, B, T, tails = model(), 16, 1000, [(b, 1000 - 37 * b) for b in range(1, 16)]
    elif case == "T1":
        m, B, T, tails = model(), 4, 1, [(2, 0)]
    elif case == "T_below_k":
        m, B, T, tails = model(k=9), 3, 3, [(1, 2)]
    elif case == "all_padding":
        m, B, T, tails = model(), 3, 50, [(1, 0), (2, 30)]
    elif case == "zero_channel0":
        m, B, T, tails = model(), 2, 60, [(1, 40)]
        x, _ = inputs(B, T, 256, 2, tails)
        x[0, 7, 0] = 0
        x[1, 0, 0] = 0
    elif case == "T_above_4096":
        m, B, T, tails = model(L=2), 2, 4200, [(1, 4150)]
    elif case == "ph":
        m, B, T, tails = model(L=2, odim=1), 8, 120, [(1, 70), (5, 3)]
    elif case == "cwt":
        m, B, T, tails = model(idim=128, L=2, odim=11), 8, 300, [(3, 200)]
    else:
        m, B, T, tails = model(L=3, padding='LEFT'), 4, 200, [(2, 150)]
    check_parity(m, B, T, tails, {"ph": "ph", "cwt": "cwt", "left": "left"}.get(case, "frame"), x=x)
    if case == "all_padding":     # zero frames: the bias path only, the same at every frame beyond the convolutions'
        x, _ = inputs(B, T, 256, 2, tails)     # reach of the ends (2 frames per layer), without dropout
        with torch.no_grad():
            out = m.eval()(x)[1, 10:T - 10]
        assert torch.allclose(out, out[:1].expand_as(out), rtol=0, atol=1e-6)


def test_eval_forward_matches_the_reference_eval():
    for kw in (dict(), dict(idim=128, L=2, odim=11), dict(L=3, padding='LEFT')):
        m = model(**kw).eval()
        x, _ = inputs(4, 300, m._cfg.idim, m._cfg.odim, [(1, 200)])
        x[0, 3, 0] = 0
        with torch.no_grad():
            out = m(x)
            sd = {n: v.double() for n, v in m.named_parameters()}
            ones = [None] * m._cfg.layers
            ref16 = pitchpred_train(sd, x.double(), ones, 0.0, m._cfg.kernel, m.padding, fp16=True)
            ref = pitchpred_train(sd, x.double(), ones, 0.0, m._cfg.kernel, m.padding)
        print(f"eval {kw}: vs fp16-operand reference {rel(out, ref16):.2e}, vs reference {rel(out, ref):.2e}")
        assert rel(out, ref16) < 2e-3 and rel(out, ref) < 5e-2


def test_p0_forward_matches_the_eval_forward():
    from diffsinger_b200 import EnergyPredictor
    for kw in (dict(p=0.0), dict(p=0.0, idim=128, L=2, odim=11), dict(p=0.0, L=2, odim=1, cls=EnergyPredictor)):
        m = model(**kw)
        x, d = inputs(16, 250, m._cfg.idim, m._cfg.odim, [(b, 250 - 13 * b) for b in range(16)])
        out = raw_step(m, x, d, 5)[0]
        with torch.no_grad():
            assert torch.equal(out, m.eval()(x))


def test_scale_invariance_and_zero():
    m = model()
    x, d = inputs(4, 300, 256, 2, [(1, 160)])
    base = raw_step(m, x, d, 7)
    for k in (-9, 13):
        r = raw_step(m, x, d * 2.0 ** k, 7)
        assert all(torch.equal(a * 2.0 ** k, b) for a, b in zip(base[1], r[1]))
        assert torch.equal(base[2] * 2.0 ** k, r[2])
    z = raw_step(m, x, torch.zeros_like(d), 7)
    assert all(torch.count_nonzero(g) == 0 for g in z[1]) and torch.count_nonzero(z[2]) == 0


def test_two_backwards_of_one_tape_and_several_forwards():
    from diffsinger_b200 import pitchpred
    m = model()
    step = m._dsx_train_step()
    params = [dict(m.named_parameters())[n].detach() for n in pitchpred.param_names(5)]
    x1, d1 = inputs(4, 90, 256, 2, [(2, 40)], seed=1)
    x2, d2 = inputs(4, 90, 256, 2, [(0, 10)], seed=2)
    a1, t1 = step.forward(params, x1, 0.5, 21)
    g1, dx1 = step.backward(params, t1, d1, 4, 90)
    g1b, dx1b = step.backward(params, t1, d1, 4, 90)
    assert torch.equal(dx1, dx1b) and all(torch.equal(a, b) for a, b in zip(g1, g1b))
    g1c, none = step.backward(params, t1, d1, 4, 90, want_x=False)
    assert none is None and all(torch.equal(a, b) for a, b in zip(g1, g1c))
    b1, s1 = step.forward(params, x1, 0.5, 21)
    b2, s2 = step.forward(params, x2, 0.5, 22)
    x1.fill_(0)                           # the tape holds what the backward needs of x
    h2, hx2 = step.backward(params, s2, d2, 4, 90)
    h1, hx1 = step.backward(params, s1, d1, 4, 90)
    assert torch.equal(a1, b1) and torch.equal(hx1, dx1) and all(torch.equal(a, b) for a, b in zip(h1, g1))
    a2, t2 = step.forward(params, x2, 0.5, 22)
    g2, dx2 = step.backward(params, t2, d2, 4, 90)
    assert torch.equal(a2, b2) and torch.equal(hx2, dx2) and all(torch.equal(a, b) for a, b in zip(h2, g2))


@pytest.mark.parametrize("idim,P,L,odim,k,padding,T", [(256, 256, 5, 2, 5, 'SAME', 130), (128, 144, 3, 11, 31, 'LEFT', 3),
                                                       (80, 240, 2, 16, 9, 'SAME', 129)])
def test_no_access_outside_the_buffers(idim, P, L, odim, k, padding, T):
    """Every buffer of a step sits between guard regions; the results must equal an unguarded run's bit for bit and the
    guards must stay untouched"""
    from diffsinger_b200 import pitchpred
    from diffsinger_b200._capi import check, lib
    from diffsinger_b200.sampler import _ptr, _stream
    m = model(idim=idim, P=P, L=L, odim=odim, k=k, padding=padding)
    step = m._dsx_train_step()
    names = pitchpred.param_names(L)
    B = 3
    x, d = inputs(B, T, idim, odim, [(1, T // 2)])
    out_ref, g_ref, d_ref, _ = raw_step(m, x, d, 8)
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
    tape = guarded((step.tape_bytes(DEV, B, T),), torch.uint8)
    ws = guarded((step.workspace(DEV, B, T).numel(),), torch.uint8)
    out = guarded((B, T, odim), torch.float32)
    keep = []
    w = pitchpred._struct(params, L, keep)
    h = step.handle(DEV)
    check(lib.dsx_pitchpred_train_forward(h, ctypes.byref(w), _ptr(xg), B, T, 0.5, 8, _ptr(tape), tape.numel(), _ptr(ws),
                                          ws.numel(), _ptr(out), _stream(DEV)))
    grads = [guarded(tuple(p.shape), torch.float32) for p in params]
    gw = pitchpred._struct(grads, L, keep)
    dg = guarded((B, T, odim), torch.float32, d)
    dx = guarded((B, T, idim), torch.float32)
    check(lib.dsx_pitchpred_train_backward(h, ctypes.byref(w), _ptr(tape), _ptr(dg), ctypes.byref(gw), _ptr(dx), B, T,
                                           _ptr(ws), ws.numel(), _stream(DEV)))
    torch.cuda.synchronize()
    assert torch.equal(out, out_ref) and torch.equal(dx, d_ref)
    assert all(torch.equal(a, b) for a, b in zip(grads, g_ref))
    for base, n in held:
        for part in (base[:GUARD], base[GUARD + n:]):
            assert torch.isnan(part).all() if base.dtype == torch.float32 else (part == 0xFF).all()


def test_backward_with_another_shape_gives_nan():
    from diffsinger_b200 import pitchpred
    m = model()
    step = m._dsx_train_step()
    params = [dict(m.named_parameters())[n].detach() for n in pitchpred.param_names(5)]
    x, d = inputs(4, 100, 256, 2, [(1, 60)])
    _, tape = step.forward(params, x, 0.5, 3)
    grads, d_x = step.backward(params, tape, d[:, :90].contiguous(), 4, 90)
    assert all(torch.isnan(g).all() for g in grads) and torch.isnan(d_x).all()


def test_keep_fraction():
    m = model()
    masks = m._dsx_train_step().masks(DEV, 99, 0.5, 16, 250)
    assert len(masks) == 5
    for mk in masks:
        assert abs(mk.float().mean().item() - 0.5) < 0.01
    assert not torch.equal(masks[0], masks[1])
    m3 = m._dsx_train_step().masks(DEV, 99, 0.1, 16, 250)
    assert abs(m3[0].float().mean().item() - 0.9) < 0.01


@pytest.mark.parametrize("case", ["frame", "ph", "cwt", "left"])
def test_golden_reference_gradients(case):
    """The module at p = 0 on the fixture's inputs against the reference's own gradients (float32 on the CPU)"""
    from conftest import golden
    from diffsinger_b200 import pitchpred
    from oracle import gen_golden_pitchpred_train as G
    from oracle.gen_golden_train import sample_index
    g = golden("pitchpred_train_grad.npz")
    cfg = dict((c, f) for c, _, _, f in G.CASES)[case]
    idim, L, C, odim, k, padding = cfg
    m = model(idim, L, C, odim, k, padding, p=0.0)
    m.load_state_dict(G.random_state_dict(G.SEED, *cfg[:5]))
    x, tgt = (t.to(DEV) for t in G.case_inputs(cfg))
    xr = x.clone().requires_grad_(True)
    out = m(xr)
    loss = ((out - tgt) ** 2).mean()
    loss.backward()
    pre = f"{case}.p0."
    assert rel(out.detach().cpu(), torch.from_numpy(g[pre + "out"])) < 2e-2
    assert rel(xr.grad.cpu(), torch.from_numpy(g[pre + "d_x"])) < 5e-2
    # d pos_embed_alpha: dsx's is the float64 sum of its own d_x . table[pos] to fp32 summation, and it differs from the
    # reference's by no more than its d_x does (Cauchy-Schwarz: |sum (d_x - d_x_ref) . t| <= |d_x - d_x_ref| |t|)
    a, a_ref = m.pos_embed_alpha.grad.item(), float(g[pre + "val.pos_embed_alpha"][0])
    d_x_ref = torch.from_numpy(g[pre + "d_x"]).to(DEV)
    own = alpha_terms(x, xr.grad).sum().item()
    assert abs(a - own) <= 1e-3 * abs(own), (a, own)
    t = alpha_terms(x, torch.ones_like(xr.grad))
    assert abs(a - a_ref) <= (xr.grad - d_x_ref).double().norm().item() * t.norm().item() + 1e-3 * abs(a_ref), (a, a_ref)
    for n in pitchpred.param_names(L)[:-1]:                   # all but pos_embed_alpha
        v = dict(m.named_parameters())[n].grad.reshape(-1).cpu()
        ref = float(g[pre + "norm." + n])
        assert abs(v.norm().item() - ref) <= 5e-2 * ref, n
        idx = torch.from_numpy(sample_index(n, v.numel())).long()
        assert rel(v[idx], torch.from_numpy(g[pre + "val." + n])) < 1e-1, n


def test_adam_lowers_the_f0_and_uv_loss():
    m = model(L=2)
    x, _ = inputs(16, 200, 256, 2, [(b, 200 - 9 * b) for b in range(16)])
    g = torch.Generator().manual_seed(9)
    f0 = torch.randn(16, 200, generator=g).to(DEV)
    uv = (torch.rand(16, 200, generator=g) > 0.7).float().to(DEV)
    nonpad = (x.abs().sum(-1) > 0).float()
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    losses = []
    for _ in range(30):
        opt.zero_grad()
        out = m(x)
        l_f0 = (((out[..., 0] - f0) ** 2) * nonpad).sum() / nonpad.sum()
        l_uv = (torch.nn.functional.binary_cross_entropy_with_logits(out[..., 1], uv, reduction='none') * nonpad).sum() \
            / nonpad.sum()
        loss = l_f0 + l_uv                 # add_pitch_loss with pitch_loss 'l2' and use_uv (fs2.py)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert losses[-1] < 0.6 * losses[0], losses


def test_chain_encoder_to_predictor(monkeypatch):
    """The graph of FastSpeech2.add_pitch under dsx_train, built by hand (not a FastSpeech2MIDI forward, and without the
    drop-in): dsx MIDI encoder (p = 0) -> with predictor_grad 0.1 -> dsx PitchPredictor (p = 0.5).  The encoder's gradients carry 0.1 d_x of the predictor and match the same chain with the oracle predictor
    (fp32 autograd, the step's masks) within the parity bound."""
    from diffsinger_b200 import FastspeechMIDIEncoder, pitchpred
    from test_gpu_fs2enc_train import HP as ENC_HP, model as enc_model
    seed = 4321
    monkeypatch.setattr(pitchpred, "draw_seed", lambda: seed)
    enc, _ = enc_model(dict(ENC_HP, dropout=0.0))
    assert isinstance(enc, FastspeechMIDIEncoder)
    pp = model()
    B, T = 4, 40
    g = torch.Generator().manual_seed(3)
    tok = torch.randint(1, 50, (B, T), generator=g)
    tok[1, 25:] = 0
    tok, tgt = tok.to(DEV), torch.randn(B, T, 2, generator=g).to(DEV)

    def run(pred):
        enc.zero_grad()
        out = enc(tok, 0, 0, 0)
        inp = out.detach() + 0.1 * (out - out.detach())      # fs2.py:199
        loss = ((pred(inp) - tgt) ** 2).mean()
        loss.backward()
        return [p.grad.clone() for p in enc.parameters() if p.grad is not None]

    dsx = run(pp)
    masks = pp._dsx_train_step().masks(DEV, seed, 0.5, B, T)
    sd = {n: v.detach() for n, v in pp.named_parameters()}
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        eager = run(lambda d: pitchpred_train(sd, d, masks, 0.5, 5, fp16=True))
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu
    assert len(dsx) == len(eager) > 0 and all(e.norm() > 0 for e in eager)
    assert max(rel(a, b) for a, b in zip(dsx, eager)) < 5e-2


def test_refusals_on_the_device():
    from diffsinger_b200 import DsxError
    x, _ = inputs(2, 10, 256, 2)
    m = model().double()
    with pytest.raises(DsxError, match="fp32"):
        m(x.double())
    m = model()
    w = m.conv[0][1].weight
    w.data = w.data.transpose(0, 1).contiguous().transpose(0, 1)
    with pytest.raises(DsxError, match="contiguous"):
        m(x)
    with pytest.raises(DsxError, match="fp32 xs"):
        model()(x.half().requires_grad_(True))
    out = model()(x.requires_grad_(True))
    with pytest.raises(DsxError, match="double backward"):
        torch.autograd.grad(out.sum(), x, create_graph=True)
