"""GPU: the FFT denoiser's training step (dsx_fft_train_*, diffsinger_b200.ffttrain) against fp32 autograd of
oracle/fft_train_oracle.py with the masks the step draws (dsx_fs2dec_train_masks of the stack's configuration), and its
exactness properties: scale invariance, determinism, seeds, several forwards before their backwards, the NaN guard of a
(B, T) mismatch, the reference's own gradients, the refusals, a 20-step Adam run and the drop-in end to end.

Errors are per-tensor relative Frobenius norms over eps, d_cond and every parameter gradient.  As in
test_gpu_fs2dec_train.py, the worst tensor must be within 5e-2 and within 1.5 x the worst of TF32 autograd on the same
case, TF32's worst taken as at least FP16_FLOOR = 2^-10 (at the smallest sizes autograd's matmuls run without tensor
cores, so its error says nothing about TF32 rounding).  The one scalar, pos_embed_alpha, is held to 5e-2 only: its
gradient is one sum over every frame with cancellation, so its relative error is not bounded by per-element rounding
(2.2e-3 against TF32's worst tensor of 8e-4 at 3 x 37 with p = 0.1 on an H100; the decoder step computes it unchanged)."""
import numpy as np
import pytest
import torch

from oracle import fft_oracle as O
from oracle.fft_train_oracle import forward_train

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
FP16_FLOOR = 2.0 ** -10
HP = dict(hidden_size=256, dec_layers=4, dec_ffn_kernel_size=9, num_heads=2, ffn_padding='SAME', ffn_act='gelu',
          dropout=0.1, residual_channels=256, audio_num_mel_bins=80, keep_bins=80)


def hp_of(H, heads, k, padding, act, L, dim, p=0.1):
    return dict(HP, hidden_size=H, num_heads=heads, dec_ffn_kernel_size=k, ffn_padding=padding, ffn_act=act,
                dec_layers=L, residual_channels=dim, dropout=p)


def model(hp, seed=3):
    from diffsinger_b200 import FFT
    m = FFT(hparams=dict(hp, dsx_train=True))
    m.load_state_dict(O.random_state_dict(seed, hp), strict=True)
    return m.train().to(DEV)


def inputs(B, T, H, tail=None, seed=5):
    """x_noisy, t, cond (utterance 1 zero from `tail`), target"""
    rs = np.random.RandomState(seed)
    spec = torch.from_numpy(rs.standard_normal((B, 1, 80, T)).astype(np.float32)).to(DEV)
    t = torch.from_numpy(rs.randint(0, 100, B)).long().to(DEV)
    cond = torch.from_numpy(rs.standard_normal((B, H, T)).astype(np.float32))
    if tail is not None and B > 1:
        cond[1, :, tail:] = 0
    tgt = torch.from_numpy(rs.standard_normal((B, 1, 80, T)).astype(np.float32)).to(DEV)
    return spec, t, cond.to(DEV), tgt


def masks_of(m, seed, B, T):
    from diffsinger_b200.fs2train import Fs2DecTrainStep
    return Fs2DecTrainStep(m._fft_cfg.dec).masks(DEV, seed, m.dropout, B, T)


def with_seed(seed, fn):
    from diffsinger_b200 import ffttrain
    orig = ffttrain.draw_seed
    ffttrain.draw_seed = lambda: seed
    try:
        return fn()
    finally:
        ffttrain.draw_seed = orig


def dsx_step(m, spec, t, cond, tgt, seed, loss=lambda e, y: ((e - y) ** 2).mean()):
    """-> eps, d_cond, {name: grad}, the masks of the step"""
    m.zero_grad(set_to_none=True)
    c = cond.clone().requires_grad_(True)

    def run():
        eps = m(spec, t, c)
        loss(eps, tgt).backward()
        return eps
    eps = with_seed(seed, run)
    return eps.detach(), c.grad, {n: p.grad.clone() for n, p in m.named_parameters()}, masks_of(m, seed, *cond.shape[::2])


def ref_step(m, hp, spec, t, cond, tgt, masks, tf32, loss=lambda e, y: ((e - y) ** 2).mean()):
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = tf32
    try:
        sd = {n: p.detach().clone().requires_grad_(True) for n, p in m.named_parameters()}
        c = cond.clone().requires_grad_(True)
        eps = forward_train(sd, spec, t, c, hp, masks, hp['dropout'])
        loss(eps, tgt).backward()
        return eps.detach(), c.grad, {n: v.grad for n, v in sd.items()}
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu


def rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def errors(res, ref):
    e = {"eps": rel(res[0], ref[0]), "d_cond": rel(res[1], ref[1])}
    e.update({n: rel(res[2][n], ref[2][n]) for n in ref[2]})
    return e


def parity(hp, B, T, tail=None, seed=11):
    m = model(hp)
    spec, t, cond, tgt = inputs(B, T, hp['hidden_size'], tail)
    eps, dc, g, masks = dsx_step(m, spec, t, cond, tgt, seed)
    assert len(g) == 13 + 10 * hp['dec_layers']      # 53 for the shipped 4 layers
    ref = ref_step(m, hp, spec, t, cond, tgt, masks, tf32=False)
    tf = ref_step(m, hp, spec, t, cond, tgt, masks, tf32=True)
    e, et = errors((eps, dc, g), ref), errors(tf, ref)
    worst, tworst = max(e.values()), max(et.values())
    print(f"\nB x T = {B} x {T} p = {hp['dropout']}: dsx worst {worst:.2e} ({max(e, key=e.get)}) median "
          f"{float(np.median(list(e.values()))):.2e}; TF32 autograd worst {tworst:.2e} ({max(et, key=et.get)})")
    assert all(np.isfinite(v) for v in e.values()), e
    assert worst <= 5e-2, e
    tensors = {n: v for n, v in e.items() if n != "pos_embed_alpha"}
    assert max(tensors.values()) <= 1.5 * max(tworst, FP16_FLOOR), (tworst, e)


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("B,T,tail", [(2, 1000, 700), (3, 37, None), (1, 4000, None), (1, 1, None)])
def test_parity_shipped(p, B, T, tail):
    parity(dict(HP, dropout=p), B, T, tail)


# dim 16 and 1024, H 64 and 256, head width 64 and 128, LEFT + ReLU, k = 1, one layer
@pytest.mark.parametrize("cfg", [(64, 1, 1, 'SAME', 'gelu', 1, 16), (256, 2, 5, 'LEFT', 'relu', 2, 1024),
                                 (128, 1, 3, 'SAME', 'gelu', 1, 48), (256, 4, 9, 'SAME', 'gelu', 1, 256)])
def test_parity_edges(cfg):
    parity(hp_of(*cfg), 2, 150, tail=90)


def raw_step(m, spec, t, cond, seed, d_eps, want_cond=True):
    """forward and backward through the step without autograd: eps, grads, d_cond"""
    from diffsinger_b200 import ffttrain
    step = m._dsx_train_step()
    named = dict(m.named_parameters())
    params = [named[n].detach() for n in ffttrain.param_names(m.num_layers, m.padding)]
    eps, tape = step.forward(params, spec, t, cond, m.dropout, seed)
    grads, dc = step.backward(params, tape, d_eps, spec.shape[0], spec.shape[3], want_cond)
    return eps, grads, dc


def test_scale_invariance_and_zero():
    m = model(HP)
    spec, t, cond, _ = inputs(2, 300, 256, tail=200)
    g = torch.randn(2, 1, 80, 300, device=DEV) * 1e-4
    _, g1, d1 = raw_step(m, spec, t, cond, 7, g)
    for k in (-20, 13):
        _, g2, d2 = raw_step(m, spec, t, cond, 7, g * 2.0 ** k)
        for a, b in zip(g1 + [d1], g2 + [d2]):
            assert torch.equal(a * 2.0 ** k, b)
    _, g0, d0 = raw_step(m, spec, t, cond, 7, torch.zeros_like(g))
    assert all((v == 0).all() for v in g0 + [d0])


def test_determinism_and_seeds():
    m = model(HP)
    spec, t, cond, _ = inputs(2, 500, 256, tail=321)
    g = torch.randn(2, 1, 80, 500, device=DEV)
    from diffsinger_b200 import ffttrain
    step = m._dsx_train_step()
    named = dict(m.named_parameters())
    params = [named[n].detach() for n in ffttrain.param_names(m.num_layers, m.padding)]
    e1, tape = step.forward(params, spec, t, cond, 0.1, 99)
    ga, da = step.backward(params, tape, g, 2, 500)
    gb, db = step.backward(params, tape, g, 2, 500)
    assert torch.equal(da, db) and all(torch.equal(a, b) for a, b in zip(ga, gb))
    e2, _, _ = raw_step(m, spec, t, cond, 99, g)
    e3, _, _ = raw_step(m, spec, t, cond, 100, g)
    assert torch.equal(e1, e2) and not torch.equal(e1, e3)
    ma, mb = masks_of(m, 99, 2, 500), masks_of(m, 100, 2, 500)
    assert all(not torch.equal(a, b) for a, b in zip(ma, mb))


def test_two_forwards_before_backward():
    m = model(HP)
    from diffsinger_b200 import ffttrain
    step = m._dsx_train_step()
    named = dict(m.named_parameters())
    params = [named[n].detach() for n in ffttrain.param_names(m.num_layers, m.padding)]
    a, b = inputs(2, 200, 256, tail=150, seed=1), inputs(3, 90, 256, seed=2)
    ga, gb = torch.randn(2, 1, 80, 200, device=DEV), torch.randn(3, 1, 80, 90, device=DEV)
    _, ta = step.forward(params, *a[:3], 0.1, 5)
    _, tb = step.forward(params, *b[:3], 0.1, 6)
    rb = step.backward(params, tb, gb, 3, 90)
    ra = step.backward(params, ta, ga, 2, 200)
    _, ea, dca = raw_step(m, *a[:3], 5, ga)
    _, eb, dcb = raw_step(m, *b[:3], 6, gb)
    assert torch.equal(ra[1], dca) and all(torch.equal(x, y) for x, y in zip(ra[0], ea))
    assert torch.equal(rb[1], dcb) and all(torch.equal(x, y) for x, y in zip(rb[0], eb))


def test_backward_with_another_shape_gives_nan():
    m = model(HP)
    from diffsinger_b200 import ffttrain
    step = m._dsx_train_step()
    named = dict(m.named_parameters())
    params = [named[n].detach() for n in ffttrain.param_names(m.num_layers, m.padding)]
    spec, t, cond, _ = inputs(2, 100, 256)
    _, tape = step.forward(params, spec, t, cond, 0.1, 3)
    grads, dc = step.backward(params, tape, torch.randn(2, 1, 80, 99, device=DEV), 2, 99)
    assert torch.isnan(dc).all() and all(torch.isnan(v).all() for v in grads)


def test_golden_reference_gradients():
    """p = 0 at 2 x 24: the L1 loss, d_cond and per parameter the norm and 64 sampled entries of the reference's own
    fp32 gradients"""
    from conftest import golden
    from oracle import gen_golden_fft_train as G
    from oracle.gen_golden_train import sample_index
    g = golden("fft_train_grad.npz")
    hp = dict({k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}, dropout=0.0)
    m = model(hp, seed=int(g["seed"]))
    spec, t, cond, noise = (v.to(DEV) for v in G.inputs(int(hp["hidden_size"])))
    eps, dc, grads, _ = dsx_step(m, spec, t, cond, noise, 1, loss=lambda e, y: (e - y).abs().mean())
    loss = (eps - noise).abs().mean().item()
    assert abs(loss - float(g["loss"])) <= 1e-3 * abs(float(g["loss"]))
    errs = {"d_cond": rel(dc.cpu(), torch.from_numpy(g["d_cond"]))}
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
    spec, t, cond, _ = inputs(1, 50, 256)
    c = cond.clone().requires_grad_(True)
    out = m(spec, t, c)
    with pytest.raises(DsxError, match="double backward"):
        torch.autograd.grad((out ** 2).mean(), c, create_graph=True)
    copy.deepcopy(m)                                                        # handles are not copied
    with pytest.raises(DsxError, match="spec.requires_grad"):
        m(spec.clone().requires_grad_(True), t, cond)
    w = m.layers[0].op.self_attn.in_proj_weight
    w.data = w.data.t().contiguous().t()
    with pytest.raises(DsxError, match="contiguous"):
        m(spec, t, cond)
    m2 = model(HP).double()
    with pytest.raises(DsxError, match="fp32"):
        m2(spec, t, cond)


def test_adam_tracks_fp32_autograd():
    """20 Adam steps of an L1 p_losses-style loss |FFT(x_noisy, t, cond) - noise| on a fixed batch, p = 0.1, with the
    step's masks in the fp32 run"""
    m = model(HP)
    ref_sd = {n: p.detach().clone().requires_grad_(True) for n, p in m.named_parameters()}
    spec, t, cond, noise = inputs(4, 300, 256, tail=250)
    opt = torch.optim.Adam(list(m.parameters()), lr=3e-4)
    ropt = torch.optim.Adam(list(ref_sd.values()), lr=3e-4)
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    la, lb = [], []
    try:
        for it in range(20):
            seed = 1000 + it
            opt.zero_grad()
            loss = with_seed(seed, lambda: (m(spec, t, cond) - noise).abs().mean())
            loss.backward()
            opt.step()
            la.append(loss.item())
            ropt.zero_grad()
            rl = (forward_train(ref_sd, spec, t, cond, HP, masks_of(m, seed, 4, 300), 0.1) - noise).abs().mean()
            rl.backward()
            ropt.step()
            lb.append(rl.item())
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu
    print("\ndsx  ", " ".join(f"{v:.4f}" for v in la), "\nfp32 ", " ".join(f"{v:.4f}" for v in lb))
    assert la[-1] < la[0] - 0.02
    assert max(abs(a - b) / b for a, b in zip(la, lb)) < 5e-3


class _Fs2(torch.nn.Module):
    """stands in for FastSpeech2: decoder_inp from a Linear over fixed features, so its gradient is visible"""

    def __init__(self, src):
        super().__init__()
        self.src = src
        self.enc = torch.nn.Linear(src.shape[-1], 256)

    def forward(self, *a, **k):
        return {"decoder_inp": self.enc(self.src)}


def test_dropin_trains_through_gaussian_diffusion(lib_built, tmp_path, monkeypatch):
    """install() on the stand-in tree with an 'fft' entry and dsx_train set: DIFF_DECODERS['fft'] builds the dsx FFT,
    and GaussianDiffusion's training branch (diff_decoder_type 'fft') gives .grad to the denoiser and to the module that
    produced cond"""
    import sys
    from standin_ref import write_tree
    from test_host_fft_train import FFT_SRC
    import diffsinger_b200 as dsx
    from oracle import diffnet_oracle as N
    write_tree(tmp_path)
    (tmp_path / "usr" / "diff" / "candidate_decoder.py").write_text(FFT_SRC)
    task = tmp_path / "usr" / "diffsinger_task.py"
    task.write_text(task.read_text() + "\nfrom usr.diff.candidate_decoder import FFT\n"
                    "DIFF_DECODERS['fft'] = lambda hp: FFT(hp['hidden_size'], hp['dec_layers'], "
                    "hp['dec_ffn_kernel_size'], hp['num_heads'])\n")
    monkeypatch.syspath_prepend(str(tmp_path))
    for n in [n for n in sys.modules if n.split(".")[0] in ("usr", "utils", "modules", "tasks", "inference")]:
        monkeypatch.delitem(sys.modules, n)
    import usr.diffsinger_task as task_mod
    import utils.hparams
    hp = dict(HP, dsx_train=True, diff_decoder_type='fft')
    utils.hparams.hparams.update(hp)
    import diffsinger_b200.dropin as dropin
    dropin.install()
    try:
        torch.manual_seed(0)
        net = task_mod.DIFF_DECODERS[hp['diff_decoder_type']](hp)
        assert isinstance(net, dsx.FFT) and net._dsx_train
        net.load_state_dict(O.random_state_dict(3, HP), strict=True)
        src = torch.randn(2, 120, 32, device=DEV)
        m = dsx.GaussianDiffusion(None, 80, net, timesteps=100, K_step=100, loss_type="l1",
                                  betas=N.linear_beta_schedule(100, 0.06), spec_min=[-6.0] * 80, spec_max=[0.5] * 80,
                                  fs2=_Fs2(src), hparams=hp).to(DEV).train()
        mel = (torch.rand(2, 120, 80, device=DEV) * 6.5 - 6.0)
        tok = torch.zeros(2, 5, dtype=torch.long, device=DEV)
        opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        losses = []
        for i in range(10):
            opt.zero_grad(set_to_none=True)
            torch.manual_seed(100)            # the same t and noise every step: one fixed batch
            loss = m(tok, ref_mels=mel, infer=False)["diff_loss"]
            loss.backward()
            if i == 0:
                assert m.fs2.enc.weight.grad is not None and m.fs2.enc.weight.grad.abs().sum() > 0
                assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in net.parameters())
            opt.step()
            losses.append(loss.item())
        assert losses[-1] < losses[0]
    finally:
        dropin.uninstall()
