"""GPU: the FastSpeech2 encoder's training step (dsx_fs2enc_train_*, diffsinger_b200.fs2enctrain) against fp32 autograd
of oracle/fs2enc_train_oracle.py with the masks the step reports, and its exactness properties: scale invariance,
determinism, zero gradients on padding tokens and unused embedding rows, several forwards before their backwards, no
access outside the buffers, the shape check, utterance independence, the p = 0 forward against the eval encoder, the
reference's gradients, a short Adam run, the chain into the DiffNet training step and the drop-in.

Errors are per-tensor relative Frobenius norms ||dsx - ref|| / ||ref|| over out, d_add, the embed_tokens gradient and
every stack gradient, bounded as in test_gpu_fs2dec_train.py: the worst within 5e-2 and within 1.5 x the worst of TF32
autograd on the same case, that taken as at least 2^-10 (one fp16 rounding of each GEMM operand)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import fs2enc_oracle as O
from oracle.fs2enc_train_oracle import encoder_train

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
FP16_FLOOR = 2.0 ** -10
VOCAB = 61
HP = dict(O.HPARAMS_MIDI)                 # ds100_adj_rel: H 256, 4 layers, 2 heads, k 9, rel_pos, dropout 0.1
HP_SIN = dict(O.HPARAMS_POPCS)


def hp_of(H, heads, k, padding, act, L, rel=True, p=0.1):
    return dict(HP, hidden_size=H, enc_layers=L, enc_ffn_kernel_size=k, num_heads=heads, ffn_padding=padding,
                ffn_act=act, rel_pos=rel, dropout=p)


def model(hp, midi=True, vocab=VOCAB, seed=3):
    """(dsx encoder in training mode under dsx_train, the full seeded state dict on the GPU)"""
    from diffsinger_b200 import FastspeechEncoder, FastspeechMIDIEncoder
    H = hp['hidden_size']
    sd = {k: v.to(DEV) for k, v in O.random_state_dict(seed, hp, vocab, midi=midi).items()}
    cls = FastspeechMIDIEncoder if midi else FastspeechEncoder
    m = cls(torch.nn.Embedding(vocab, H, 0), H, hp['enc_layers'], hp['enc_ffn_kernel_size'], num_heads=hp['num_heads'],
            hparams=dict(hp, dsx_train=True))
    m.load_state_dict({k: v for k, v in O.sub(sd, "encoder.").items()}, strict=True)
    return m.to(DEV).train(), sd


def inputs(B, T, tails, sd, midi=True, vocab=VOCAB, seed=5):
    """tokens and the three addends ([B, T, H] fp32 leaves, or ()) and an MSE target"""
    tok, pm, md, sl = O.fixture_inputs(seed, B, T, tails, vocab) if vocab > 1 else (
        torch.zeros(B, T, dtype=torch.long),) * 2 + (torch.zeros(B, T),) + (torch.zeros(B, T, dtype=torch.long),)
    tok = tok.to(DEV)
    H = sd["encoder.embed_tokens.weight"].shape[1]
    adds = ()
    if midi:
        with torch.no_grad():
            adds = tuple(a.contiguous() for a in O.midi_addends(sd, pm.to(DEV), md.to(DEV), sl.to(DEV)))
    tgt = torch.from_numpy(np.random.RandomState(seed + 1).standard_normal((B, T, H)).astype(np.float32)).to(DEV)
    return tok, adds, tgt


def _run(m, tok, adds):
    return m(tok, *adds) if adds else m(tok)


def dsx_step(m, tok, adds, tgt, seed):
    """loss = MSE(out, tgt) through the module; -> out, d_add (or None), {name: grad}, the masks of the step"""
    from diffsinger_b200 import fs2enctrain
    orig = fs2enctrain.draw_seed
    fs2enctrain.draw_seed = lambda: seed
    try:
        m.zero_grad(set_to_none=True)
        ar = [a.clone().requires_grad_(True) for a in adds]
        out = _run(m, tok, ar)
        ((out - tgt) ** 2).mean().backward()
    finally:
        fs2enctrain.draw_seed = orig
    masks = m._dsx_train_step().masks(DEV, seed, m.dropout, tok.shape[0], tok.shape[1])
    if ar:
        assert all(torch.equal(a.grad, ar[0].grad) for a in ar)
    return out.detach(), ar[0].grad if ar else None, {n: p.grad.clone() for n, p in m.named_parameters()}, masks


def ref_step(m, hp, tok, adds, tgt, masks, tf32):
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    try:
        sd = {n: p.detach().clone().requires_grad_(True) for n, p in m.named_parameters()}
        ar = [a.clone().requires_grad_(True) for a in adds]
        out = encoder_train(sd, tok, hp, masks, hp['dropout'], tuple(ar), m._rel_len)
        ((out - tgt) ** 2).mean().backward()
        return out.detach(), ar[0].grad if ar else None, {n: v.grad for n, v in sd.items()}
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def errors(res, ref):
    e = {"out": rel(res[0], ref[0])}
    if ref[1] is not None:
        e["d_add"] = rel(res[1], ref[1])
    e.update({n: rel(res[2][n], ref[2][n]) for n in ref[2]})
    return e


def parity(hp, B, T, tails, midi=True, vocab=VOCAB, tok=None, seed=11):
    m, sd = model(hp, midi, vocab)
    t0, adds, tgt = inputs(B, T, tails, sd, midi, vocab)
    tok = t0 if tok is None else tok.to(DEV)
    out, d_add, g, masks = dsx_step(m, tok, adds, tgt, seed)
    ref = ref_step(m, hp, tok, adds, tgt, masks, tf32=False)
    tf = ref_step(m, hp, tok, adds, tgt, masks, tf32=True)
    e, et = errors((out, d_add, g), ref), errors(tf, ref)
    worst, tworst = max(e.values()), max(et.values())
    print(f"\n{'MIDI' if midi else 'sin'} B x T = {B} x {T} p = {hp['dropout']}: dsx worst {worst:.2e} "
          f"({max(e, key=e.get)}) median {float(np.median(list(e.values()))):.2e}; TF32 autograd worst {tworst:.2e}")
    assert all(np.isfinite(v) for v in e.values()), e
    assert worst <= 5e-2 and worst <= 1.5 * max(tworst, FP16_FLOOR), (worst, tworst, e)
    pad = tok == 0
    if d_add is not None:
        assert (d_add[pad] == 0).all()
    dE = g["embed_tokens.weight"]
    used = torch.zeros(vocab, dtype=torch.bool, device=DEV)
    used[tok[~pad]] = True
    assert (dE[0] == 0).all() and (dE[~used] == 0).all()
    return m


def _one_token_batch():
    tok = torch.randint(1, VOCAB, (3, 20), generator=torch.Generator().manual_seed(4))
    tok[1, 1:] = 0
    tok[2, 13:] = 0
    return tok


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("midi", [True, False])
@pytest.mark.parametrize("B,T,tails", [(16, 250, tuple(250 - 9 * b if b % 2 else None for b in range(16))),
                                       (3, 37, (None, 20, 5)), (1, 1, (None,)), (3, 20, None)])
def test_parity(p, midi, B, T, tails):
    hp = dict(HP if midi else HP_SIN, dropout=p)
    if tails is None:                                     # a batch holding a one-token utterance
        parity(hp, B, T, (None,) * B, midi, tok=_one_token_batch())
    else:
        parity(hp, B, T, tails, midi)


@pytest.mark.parametrize("cfg", [(64, 1, 1, 'SAME', 'gelu', 2), (128, 1, 3, 'LEFT', 'relu', 1),
                                 (192, 3, 5, 'SAME', 'relu', 2), (256, 2, 9, 'LEFT', 'gelu', 1)])
def test_parity_edges(cfg):
    parity(hp_of(*cfg), 2, 150, (None, 90))


def test_parity_large_vocabulary_and_one_dominant_id():
    parity(HP, 4, 300, (None, 200, None, 17), vocab=4096)
    tok = torch.randint(1, VOCAB, (8, 512), generator=torch.Generator().manual_seed(9))
    tok[torch.rand(8, 512, generator=torch.Generator().manual_seed(10)) < 0.97] = 7
    tok[3, 400:] = 0
    parity(HP, 8, 512, (None,) * 8, tok=tok)


def raw_step(m, tok, adds, seed, d_out, p=None):
    """forward and backward through the step without autograd: out, grads, d_add"""
    from diffsinger_b200 import fs2enctrain
    step = m._dsx_train_step()
    params = [dict(m.named_parameters())[n].detach() for n in fs2enctrain.param_names(m.num_layers, m.padding)]
    adds3 = list(adds) + [None] * (3 - len(adds))
    out, tape = step.forward(params, tok, adds3, m._rel_len, m.dropout if p is None else p, seed)
    grads, d_add = step.backward(params, tape, d_out, tok.shape[0], tok.shape[1])
    return out, grads, d_add


def test_scale_invariance_and_zero():
    m, sd = model(HP)
    tok, adds, _ = inputs(2, 300, (None, 200), sd)
    g = torch.randn(2, 300, 256, device=DEV) * 1e-4
    _, g1, d1 = raw_step(m, tok, adds, 7, g)
    for k in (-20, 13):
        _, g2, d2 = raw_step(m, tok, adds, 7, g * 2.0 ** k)
        for a, b in zip(g1 + [d1], g2 + [d2]):
            assert torch.equal(a * 2.0 ** k, b)
    _, g0, d0 = raw_step(m, tok, adds, 7, torch.zeros_like(g))
    assert all((t == 0).all() for t in g0 + [d0])


def test_determinism_and_seeds():
    m, sd = model(HP)
    tok, adds, _ = inputs(3, 200, (None, 150, 1), sd)
    g = torch.randn(3, 200, 256, device=DEV)
    from diffsinger_b200 import fs2enctrain
    step = m._dsx_train_step()
    params = [dict(m.named_parameters())[n].detach() for n in fs2enctrain.param_names(m.num_layers, m.padding)]
    out, tape = step.forward(params, tok, list(adds), m._rel_len, 0.1, 99)
    ga, da = step.backward(params, tape, g, 3, 200)
    gb, db = step.backward(params, tape, g, 3, 200)                       # two backwards of one tape
    assert torch.equal(da, db) and all(torch.equal(a, b) for a, b in zip(ga, gb))
    o2, g2, d2 = raw_step(m, tok, adds, 99, g)                            # a repeated step with the same seed
    assert torch.equal(out, o2) and torch.equal(da, d2) and all(torch.equal(a, b) for a, b in zip(ga, g2))
    o3, _, _ = raw_step(m, tok, adds, 100, g)
    assert not torch.equal(out, o3)
    ma, mb = step.masks(DEV, 99, 0.1, 3, 200), step.masks(DEV, 100, 0.1, 3, 200)
    assert all(not torch.equal(a, b) for a, b in zip(ma, mb))


def test_several_forwards_before_their_backwards():
    m, sd = model(HP)
    from diffsinger_b200 import fs2enctrain
    step = m._dsx_train_step()
    params = [dict(m.named_parameters())[n].detach() for n in fs2enctrain.param_names(m.num_layers, m.padding)]
    ta_, aa, _ = inputs(2, 200, (None, 150), sd, seed=1)
    tb_, ab, _ = inputs(3, 90, (None, None, 40), sd, seed=2)
    ga, gb = torch.randn(2, 200, 256, device=DEV), torch.randn(3, 90, 256, device=DEV)
    _, tpa = step.forward(params, ta_, list(aa), m._rel_len, 0.1, 5)
    _, tpb = step.forward(params, tb_, list(ab), m._rel_len, 0.1, 6)
    ta_.fill_(3)                                            # the tape holds its own copy of the tokens
    rb = step.backward(params, tpb, gb, 3, 90)
    ra = step.backward(params, tpa, ga, 2, 200)
    ta_, aa, _ = inputs(2, 200, (None, 150), sd, seed=1)
    _, ea, da = raw_step(m, ta_, aa, 5, ga)
    _, eb, db = raw_step(m, tb_, ab, 6, gb)
    assert torch.equal(ra[1], da) and all(torch.equal(a, b) for a, b in zip(ra[0], ea))
    assert torch.equal(rb[1], db) and all(torch.equal(a, b) for a, b in zip(rb[0], eb))


def test_no_access_outside_the_buffers():
    """Every buffer of a step sits between NaN-filled guard regions; the results must equal an unguarded run's bit for
    bit and the guards must stay NaN."""
    guarded_step(256, 2, 130, VOCAB, 77)


@pytest.mark.parametrize("H,heads,T,vocab", [(64, 1, 65, 1), (64, 1, 65, 70000)])
def test_no_access_outside_the_buffers_at_edges(H, heads, T, vocab):
    """test_no_access_outside_the_buffers at H 64 with one head, over a one-row (all padding) and a 70000-row
    vocabulary"""
    guarded_step(H, heads, T, vocab, T - T // 4)


def guarded_step(H, heads, T, vocab, tail):
    """one step of B = 2 (utterance 1 padding from `tail` on) with every buffer between guard regions"""
    import ctypes
    from diffsinger_b200 import _capi, fs2enctrain
    from diffsinger_b200._capi import check, lib
    from diffsinger_b200.sampler import _ptr, _stream, _strides_bct
    m, sd = model(dict(HP, hidden_size=H, num_heads=heads), vocab=vocab)
    step = m._dsx_train_step()
    names = fs2enctrain.param_names(m.num_layers, m.padding)
    B = 2
    tok, adds, _ = inputs(B, T, (None, tail), sd, vocab=vocab)
    g = torch.randn(B, T, H, device=DEV)
    o_ref, g_ref, d_ref = raw_step(m, tok, adds, 8, g)
    GUARD = 4096
    held = []

    def guarded(shape, dtype, src=None):
        n = int(np.prod(shape))
        fill = 0xFF if dtype == torch.uint8 else (-1 if dtype == torch.int64 else float("nan"))
        base = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device=DEV)
        held.append((base, n))
        v = base[GUARD:GUARD + n].view(shape)
        if src is not None:
            v.copy_(src)
        return v

    params = [guarded(tuple(dict(m.named_parameters())[n].shape), torch.float32, dict(m.named_parameters())[n].detach())
              for n in names]
    tg = guarded((B, T), torch.int64, tok)
    ag = [guarded((B, T, H), torch.float32, a) for a in adds]
    tape = guarded((step.tape_bytes(DEV, B, T),), torch.uint8)
    ws = guarded((step.workspace(DEV, B, T).numel(),), torch.uint8)
    out = guarded((B, T, H), torch.float32)
    keep = []
    w = fs2enctrain._struct(params, m.num_layers, keep)
    ptrs = (ctypes.c_void_p * 3)(*[a.data_ptr() for a in ag])
    strides = (_capi.Strides * 3)(*[_strides_bct(a, (0, 2, 1)) for a in ag])
    h = step.handle(DEV)
    check(lib.dsx_fs2enc_train_forward(h, ctypes.byref(w), _ptr(tg), B, T, ptrs, strides, m._rel_len, 0.1, 8, _ptr(tape),
                                       tape.numel(), _ptr(ws), ws.numel(), _ptr(out), _stream(DEV)))
    grads = [guarded(tuple(p.shape), torch.float32) for p in params]
    gw = fs2enctrain._struct(grads, m.num_layers, keep)
    dg = guarded((B, T, H), torch.float32, g)
    da = guarded((B, T, H), torch.float32)
    check(lib.dsx_fs2enc_train_backward(h, ctypes.byref(w), _ptr(tape), _ptr(dg), ctypes.byref(gw), _ptr(da), B, T,
                                        _ptr(ws), ws.numel(), _stream(DEV)))
    torch.cuda.synchronize()
    assert torch.equal(out, o_ref) and torch.equal(da, d_ref)
    assert all(torch.equal(a, b) for a, b in zip(grads, g_ref))
    for base, n in held:
        for part in (base[:GUARD], base[GUARD + n:]):
            if base.dtype == torch.float32:
                assert torch.isnan(part).all()
            else:
                assert (part == (0xFF if base.dtype == torch.uint8 else -1)).all()


def test_backward_with_another_shape_gives_nan():
    m, sd = model(HP)
    tok, adds, _ = inputs(2, 100, (None, 60), sd)
    from diffsinger_b200 import fs2enctrain
    step = m._dsx_train_step()
    params = [dict(m.named_parameters())[n].detach() for n in fs2enctrain.param_names(m.num_layers, m.padding)]
    _, tape = step.forward(params, tok, list(adds), m._rel_len, 0.1, 3)
    grads, d_add = step.backward(params, tape, torch.randn(2, 99, 256, device=DEV), 2, 99)
    assert torch.isnan(d_add).all() and all(torch.isnan(v).all() for v in grads)


def test_all_padding_gives_zeros():
    """a vocabulary of 1 (every token padding), and one all-padding utterance in a batch"""
    m, sd = model(HP, vocab=1)
    tok, adds, _ = inputs(2, 40, None, sd, vocab=1)
    out, grads, d_add = raw_step(m, tok, adds, 4, torch.randn(2, 40, 256, device=DEV))
    assert (out == 0).all() and (d_add == 0).all() and all((v == 0).all() for v in grads)
    m, sd = model(HP)
    tok, adds, _ = inputs(3, 50, (None, 0, 30), sd)
    out, grads, d_add = raw_step(m, tok, adds, 4, torch.randn(3, 50, 256, device=DEV))
    assert (out[1] == 0).all() and (d_add[1] == 0).all()
    assert all(torch.isfinite(v).all() for v in grads)


def test_utterances_are_independent():
    """each utterance's out and d_add equal those of the utterance alone at the same T, bit for bit.  The backward's
    gradient scale is a power of two from amax |d_out| over the whole call, so every utterance's d_out carries the same
    largest element: alone, each gets the batch's scale."""
    m, sd = model(HP)
    B, T = 3, 90
    tok, adds, _ = inputs(B, T, (None, 50, 1), sd)
    g = torch.randn(B, T, 256, device=DEV)
    g[:, 0, 0] = 8.0
    out, _, d_add = raw_step(m, tok, adds, 0, g, p=0.0)
    for b in range(B):
        ob, _, db = raw_step(m, tok[b:b + 1].contiguous(), tuple(a[b:b + 1].contiguous() for a in adds), 0, g[b:b + 1],
                             p=0.0)
        assert torch.equal(ob[0], out[b]) and torch.equal(db[0], d_add[b]), b


@pytest.mark.parametrize("midi", [True, False])
def test_p0_forward_matches_the_eval_encoder(midi):
    m, sd = model(dict(HP if midi else HP_SIN, dropout=0.0), midi)
    tok, adds, _ = inputs(3, 120, (None, 70, 9), sd, midi)
    out, _, _ = raw_step(m, tok, adds, 1, torch.zeros(3, 120, 256, device=DEV))
    with torch.no_grad():
        ev = _run(m.eval(), tok, adds)
    m.train()
    assert torch.equal(out, ev), (out - ev).abs().max().item()


@pytest.mark.parametrize("case", ["midi", "sin"])
def test_golden_reference_gradients(case):
    """p = 0 on the fixture of oracle/gen_golden_fs2enc_train.py: the loss, d_add and the embed_tokens gradient in full,
    and per other parameter the norm and 64 sampled entries of the reference's own fp32 gradients"""
    from conftest import golden
    from oracle import gen_golden_fs2enc_train as G
    from oracle.gen_golden_train import sample_index
    g = golden("fs2enc_train_grad.npz")
    hp = dict({c: h for c, _, h in G.CASES}[case], dropout=0.0)
    enc_sd, tok, adds, tgt = G.case_inputs(case, hp)
    m, _ = model(hp, case == "midi", G.VOCAB, seed=G.SEED)
    m.load_state_dict({k: v.to(DEV) for k, v in enc_sd.items()}, strict=True)
    out, d_add, grads, _ = dsx_step(m, tok.to(DEV), tuple(a.to(DEV) for a in adds), tgt.to(DEV), 1)
    loss = ((out - tgt.to(DEV)) ** 2).mean().item()
    assert abs(loss - float(g[f"{case}.p0.loss"])) <= 1e-3 * abs(float(g[f"{case}.p0.loss"]))
    errs = {"embed_tokens.weight": rel(grads["embed_tokens.weight"].cpu(),
                                       torch.from_numpy(g[f"{case}.p0.grad.embed_tokens.weight"]))}
    if case == "midi":
        errs["d_add"] = rel(d_add.cpu(), torch.from_numpy(g["midi.p0.grad.d_add"]))
    for n, v in grads.items():
        if n == "embed_tokens.weight":
            continue
        flat = v.reshape(-1).cpu()
        ref_norm = float(g[f"{case}.p0.norm.{n}"])
        errs["norm." + n] = abs(flat.norm().item() - ref_norm) / ref_norm
        errs["val." + n] = rel(flat[torch.from_numpy(sample_index(n, flat.numel())).long()],
                               torch.from_numpy(g[f"{case}.p0.val.{n}"]))
    worst = max(errs, key=errs.get)
    print(f"\ngolden {case}: worst {errs[worst]:.2e} ({worst}), median {float(np.median(list(errs.values()))):.2e}")
    assert errs[worst] <= 5e-2, errs


def test_adam_tracks_fp32_autograd():
    """20 Adam steps of the MIDI encoder + Linear(256, 80) + L1, the addends' embeddings training too, p = 0.1 with the
    step's masks in the fp32 run"""
    torch.manual_seed(0)
    m, sd = model(HP)
    B, T = 4, 120
    tok, _, _ = inputs(B, T, (None, 100, None, 31), sd)
    pm = torch.randint(48, 77, (B, T), device=DEV) * (tok > 0)
    md = torch.rand(B, T, device=DEV) * (tok > 0)
    sl = (torch.rand(B, T, device=DEV) < 0.125).long() * (tok > 0)
    emb = {k: sd[k].clone().requires_grad_(True) for k in ("midi_embed.weight", "midi_dur_layer.weight",
                                                           "midi_dur_layer.bias", "is_slur_embed.weight")}
    remb = {k: v.detach().clone().requires_grad_(True) for k, v in emb.items()}
    head, ref_head = torch.nn.Linear(256, 80).to(DEV), torch.nn.Linear(256, 80).to(DEV)
    ref_head.load_state_dict(head.state_dict())
    ref_sd = {n: p.detach().clone().requires_grad_(True) for n, p in m.named_parameters()}
    y = torch.from_numpy(np.random.RandomState(9).standard_normal((B, T, 80)).astype(np.float32)).to(DEV)
    opt = torch.optim.Adam(list(m.parameters()) + list(head.parameters()) + list(emb.values()), lr=3e-4)
    ropt = torch.optim.Adam(list(ref_sd.values()) + list(ref_head.parameters()) + list(remb.values()), lr=3e-4)
    from diffsinger_b200 import fs2enctrain
    orig = fs2enctrain.draw_seed
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    la, lb = [], []
    try:
        for it in range(20):
            seed = 1000 + it
            fs2enctrain.draw_seed = (lambda s: (lambda: s))(seed)
            opt.zero_grad()
            loss = (head(m(tok, *O.midi_addends(emb, pm, md, sl))) - y).abs().mean()
            loss.backward()
            opt.step()
            la.append(loss.item())
            masks = m._dsx_train_step().masks(DEV, seed, 0.1, B, T)
            ropt.zero_grad()
            rl = (ref_head(encoder_train(ref_sd, tok, HP, masks, 0.1, O.midi_addends(remb, pm, md, sl))) - y).abs().mean()
            rl.backward()
            ropt.step()
            lb.append(rl.item())
    finally:
        fs2enctrain.draw_seed = orig
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu
    print("\ndsx  ", " ".join(f"{v:.4f}" for v in la), "\nfp32 ", " ".join(f"{v:.4f}" for v in lb))
    assert la[-1] < la[0] - 0.02
    assert max(abs(a - b) / b for a, b in zip(la, lb)) < 1e-4


def test_chain_encoder_gather_diffnet():
    """dsx MIDI encoder -> mel2ph gather -> dsx DiffNet training step, L1 against the noise: the encoder's and the MIDI
    embeddings' gradients against the fp32 oracle chain, within test_gpu_train.py's bounds for cuDNN's defaults"""
    import diffsinger_b200 as dsx
    from test_gpu_train import BOUND_MEDIAN, BOUND_TENSOR
    m, sd = model(HP)
    B, T = 2, 60
    tok, _, _ = inputs(B, T, (None, 41), sd)
    g = torch.Generator().manual_seed(2)
    pm = (torch.randint(48, 77, (B, T), generator=g).to(DEV)) * (tok > 0)
    md = torch.rand(B, T, generator=g).to(DEV) * (tok > 0)
    sl = (torch.rand(B, T, generator=g) < 0.125).long().to(DEV) * (tok > 0)
    dur = torch.randint(3, 17, (B, T), generator=g).to(DEV) * (tok > 0)
    mel2ph = O.length_regulator(dur, tok == 0)
    Tm = mel2ph.shape[1]
    torch.manual_seed(0)
    net = dsx.DiffNet(80, hparams=dict(hidden_size=256, residual_layers=20, residual_channels=256,
                                       dilation_cycle_length=4), train=True)
    torch.nn.init.normal_(net.output_projection.weight, std=0.02)
    net = net.to(DEV).train()
    spec = torch.randn(B, 1, 80, Tm, generator=g).to(DEV)
    noise = torch.randn(B, 1, 80, Tm, generator=g).to(DEV)
    t = torch.randint(0, 100, (B,), generator=g).to(DEV)
    emb_keys = ("midi_embed.weight", "midi_dur_layer.weight", "midi_dur_layer.bias", "is_slur_embed.weight")

    def chain(path):
        esd = {n: p.detach().clone().requires_grad_(True) for n, p in m.named_parameters()}
        emb = {k: sd[k].clone().requires_grad_(True) for k in emb_keys}
        net.zero_grad(set_to_none=True)
        adds = O.midi_addends(emb, pm, md, sl)
        if path == "dsx":
            from diffsinger_b200 import fs2enctrain
            orig = fs2enctrain.draw_seed
            fs2enctrain.draw_seed = lambda: 21
            try:
                m.zero_grad(set_to_none=True)
                enc = m(tok, *adds)
            finally:
                fs2enctrain.draw_seed = orig
        else:
            masks = m._dsx_train_step().masks(DEV, 21, 0.1, B, T)
            enc = encoder_train(esd, tok, HP, masks, 0.1, adds)
        dec_inp = torch.gather(F.pad(enc, [0, 0, 1, 0]), 1, mel2ph[..., None].repeat([1, 1, 256]))
        cond = (dec_inp * (mel2ph > 0).float()[:, :, None]).transpose(1, 2)
        if path == "dsx":
            eps = net(spec, t, cond)
        else:
            old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
            try:
                eps = net._forward_autograd(spec, t, cond)
            finally:
                torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
        (noise - eps).abs().mean().backward()
        eg = {n: p.grad for n, p in m.named_parameters()} if path == "dsx" else {n: v.grad for n, v in esd.items()}
        return dict(eg, **{k: v.grad for k, v in emb.items()})

    mine, ref = chain("dsx"), chain("fp32")
    per = {n: rel(mine[n], ref[n]) for n in ref}
    med = sorted(per.values())[len(per) // 2]
    print(f"\nchain: worst {max(per.values()):.2e} ({max(per, key=per.get)}), median {med:.2e}")
    assert max(per.values()) <= BOUND_TENSOR and med <= BOUND_MEDIAN, per


# ---- drop-in on a stand-in FastSpeech2MIDI tree whose DurationPredictor trains in eager PyTorch -------------------------
STANDIN_TRAIN = {
    "modules/__init__.py": "",
    "modules/fastspeech/__init__.py": "",
    "modules/fastspeech/tts_modules.py": """
        import torch
        import torch.nn as nn

        class _Ref(nn.Module):
            def __init__(self, *a, **k):
                super().__init__()
                raise RuntimeError(f"stand-in {type(self).__name__}: install_fs2_encoder() should have replaced it")

        class FastspeechEncoder(_Ref):
            pass

        class LengthRegulator(_Ref):
            pass

        class DurationPredictor(nn.Module):
            # an eager stand-in of the reference's: conv, ReLU, linear head, * !padding
            def __init__(self, idim, n_layers=2, n_chans=384, kernel_size=3, dropout_rate=0.1, offset=1.0,
                         padding='SAME'):
                super().__init__()
                self.conv = nn.Conv1d(idim, n_chans, kernel_size, padding=kernel_size // 2)
                self.linear = nn.Linear(n_chans, 1)

            def forward(self, xs, x_masks=None):
                x = torch.relu(self.conv(xs.transpose(1, 2))).transpose(1, 2)
                return self.linear(x).squeeze(-1) * (1 - x_masks.float())
    """,
    "modules/fastspeech/fs2.py": """
        import torch.nn as nn
        from modules.fastspeech.tts_modules import FastspeechEncoder, DurationPredictor, LengthRegulator
        from utils.hparams import hparams

        class FastSpeech2(nn.Module):
            def __init__(self, dictionary):
                super().__init__()
                self.hidden_size = hparams['hidden_size']
                self.encoder_embed_tokens = nn.Embedding(len(dictionary), self.hidden_size, 0)
                self.dur_predictor = DurationPredictor(self.hidden_size, n_chans=64, kernel_size=3)
                self.length_regulator = LengthRegulator()

            def add_dur(self, dur_input, mel2ph, txt_tokens, ret):
                src_padding = txt_tokens == 0
                dur_input = dur_input.detach() + hparams['predictor_grad'] * (dur_input - dur_input.detach())
                ret['dur'] = self.dur_predictor(dur_input, src_padding)
                return mel2ph
    """,
    "modules/diffsinger_midi/__init__.py": "",
    "modules/diffsinger_midi/fs2.py": """
        import torch
        import torch.nn as nn
        import torch.nn.functional as F
        from modules.fastspeech.tts_modules import FastspeechEncoder
        from modules.fastspeech.fs2 import FastSpeech2
        from utils.hparams import hparams

        class FastspeechMIDIEncoder(FastspeechEncoder):
            pass

        FS_ENCODERS = {
            'fft': lambda hp, embed_tokens, d: FastspeechMIDIEncoder(
                embed_tokens, hp['hidden_size'], hp['enc_layers'], hp['enc_ffn_kernel_size'], num_heads=hp['num_heads']),
        }

        class FastSpeech2MIDI(FastSpeech2):
            def __init__(self, dictionary):
                super().__init__(dictionary)
                self.encoder = FS_ENCODERS['fft'](hparams, self.encoder_embed_tokens, dictionary)
                self.midi_embed = nn.Embedding(300, self.hidden_size, 0)
                self.midi_dur_layer = nn.Linear(1, self.hidden_size)
                self.is_slur_embed = nn.Embedding(2, self.hidden_size)

            def forward(self, txt_tokens, mel2ph, **kwargs):
                ret = {}
                midi = self.midi_embed(kwargs['pitch_midi'])
                midi_dur = self.midi_dur_layer(kwargs['midi_dur'][:, :, None])
                slur = self.is_slur_embed(kwargs['is_slur'])
                encoder_out = self.encoder(txt_tokens, midi, midi_dur, slur)
                src_nonpadding = (txt_tokens > 0).float()[:, :, None]
                mel2ph = self.add_dur(encoder_out * src_nonpadding, mel2ph, txt_tokens, ret)
                decoder_inp = F.pad(encoder_out, [0, 0, 1, 0])
                decoder_inp = torch.gather(decoder_inp, 1, mel2ph[..., None].repeat([1, 1, encoder_out.shape[-1]]))
                ret['decoder_inp'] = decoder_inp * (mel2ph > 0).float()[:, :, None]
                return ret
    """,
    "utils/__init__.py": "",
    "utils/hparams.py": "hparams = {}\n",
}


class _Dictionary:
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n


def test_dropin_trains_fastspeech2midi(lib_built, tmp_path, monkeypatch):
    """install_fs2_encoder(duration_predictor=False) under dsx_train: the encoder trains on dsx, the stand-in
    DurationPredictor in eager PyTorch, and 10 Adam steps lower the loss"""
    import sys
    import textwrap
    for rel_, body in STANDIN_TRAIN.items():
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
    import modules.diffsinger_midi.fs2 as mfs2
    import modules.fastspeech.fs2 as fs2
    import diffsinger_b200 as dsx
    import diffsinger_b200.dropin as dropin
    ref_dp = fs2.DurationPredictor
    dropin.install_fs2_encoder(duration_predictor=False)
    try:
        assert fs2.DurationPredictor is ref_dp and mfs2.FastspeechMIDIEncoder is dsx.FastspeechMIDIEncoder
        net = mfs2.FastSpeech2MIDI(_Dictionary(VOCAB))
        assert type(net.encoder) is dsx.FastspeechMIDIEncoder and net.encoder._dsx_train
        assert type(net.dur_predictor) is ref_dp
        torch.manual_seed(0)
        net = net.to(DEV).train()
        B, T = 2, 40
        tok, _, _ = inputs(B, T, (None, 29), {"encoder.embed_tokens.weight": torch.zeros(VOCAB, 256)}, midi=False)
        pm = torch.randint(48, 77, (B, T), device=DEV) * (tok > 0)
        md = torch.rand(B, T, device=DEV) * (tok > 0)
        sl = (torch.rand(B, T, device=DEV) < 0.125).long() * (tok > 0)
        dur = torch.randint(3, 9, (B, T), device=DEV) * (tok > 0)
        mel2ph = O.length_regulator(dur, tok == 0)
        y = torch.randn(B, mel2ph.shape[1], 256, device=DEV)
        head = torch.nn.Linear(256, 256).to(DEV)
        opt = torch.optim.Adam(list(net.parameters()) + list(head.parameters()), lr=1e-3)
        losses = []
        for _ in range(10):
            opt.zero_grad()
            ret = net(tok, mel2ph, pitch_midi=pm, midi_dur=md, is_slur=sl)
            loss = (head(ret['decoder_inp']) - y).abs().mean() + ((ret['dur'] - dur.float().log1p()) ** 2).mean()
            loss.backward()
            for mod in (net.encoder, net.dur_predictor, net.midi_embed):
                assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in mod.parameters())
            assert net.midi_embed.weight.grad.abs().sum() > 0 and net.dur_predictor.conv.weight.grad.abs().sum() > 0
            opt.step()
            losses.append(loss.item())
        print("\nlosses", " ".join(f"{v:.4f}" for v in losses))
        assert losses[-1] < losses[0]
    finally:
        dropin.uninstall_fs2_encoder()
    assert fs2.DurationPredictor is ref_dp and mfs2.FastspeechMIDIEncoder is not dsx.FastspeechMIDIEncoder
    for n in drop():
        del sys.modules[n]
