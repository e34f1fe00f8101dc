"""GPU: the SSIM loss (diffsinger_b200.ssim, dsx_ssim_forward / dsx_ssim_backward) against the reference's fp32 values
(tests/golden/ssim.npz), against the float64 oracle side by side with eager fp32 (TF32 off) and eager under PyTorch's
defaults (cuDNN convolutions in TF32), at the edges of the shapes the C ABI accepts, for its bitwise properties, and
through the drop-in in a short Adam run of the dsx decoder with the singing configs' `l1:0.5|ssim:0.5` mel loss.

Accuracy is compared on the map and on both input gradients of sum(d_map * map) for a random d_map.  dsx is "no worse"
than eager fp32 when its mean |error| is at most eager fp32's and its max |error| at most eager fp32's plus SLACK units
of fp32 rounding of the largest reference value (at the rounding floor, random normal images, the two maxima are draws
of the same size)."""
import json

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import ssim_oracle as O
from ssim_standin import drop_tree, install_tree

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
EPS32 = 2.0 ** -24
SLACK = 8


def dsx_map_and_grads(x, y, d_map):
    from diffsinger_b200 import ssim
    xr, yr = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    m = ssim(xr, yr, size_average=False)
    m.backward(d_map)
    return m.detach(), xr.grad, yr.grad


def eager_map_and_grads(x, y, d_map, dtype=None, tf32=False):
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = tf32
    try:
        xr = x.to(dtype or x.dtype).clone().requires_grad_(True)
        yr = y.to(dtype or y.dtype).clone().requires_grad_(True)
        m = O.ssim(xr, yr, size_average=False)
        m.backward(d_map.to(m.dtype))
        torch.cuda.synchronize()
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    return m.detach(), xr.grad, yr.grad


def errors(got, ref):
    return [((g.double() - r).abs().max().item(), (g.double() - r).abs().mean().item()) for g, r in zip(got, ref)]


# ---- the reference's values -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["mel", "cwt"])
def test_golden(lib_built, case):
    from diffsinger_b200 import ssim
    g = golden("ssim.npz")
    f = lambda k: torch.from_numpy(g[f"{case}.{k}"]).to(DEV)
    bias = float(g[f"{case}.bias"])
    out, target = f("decoder_output"), f("target")
    m = ssim(out[:, None] + bias, target[:, None] + bias, size_average=False)
    mean = ssim(out[:, None] + bias, target[:, None] + bias)
    o = out.clone().requires_grad_(True)
    loss = O.ssim_loss(o, target, bias, ssim_fn=ssim)
    loss.backward()
    dm = (m - f("map")).abs().max().item()
    dl = abs(loss.item() - float(g[f"{case}.loss"]))
    dg = (o.grad - f("d_decoder_output")).abs().max().item()
    print(f"golden {case}: map {dm:.2e}, mean {abs(mean.item() - float(g[f'{case}.mean'])):.2e}, loss {dl:.2e}, "
          f"d_decoder_output {dg:.2e}")
    # the reference's own fp32 rounding: float64 lies 8e-4 / 4e-6 / 2e-6 / 9e-8 from its map / mean / loss / gradient
    # (tests/test_oracle_ssim.py); the mean includes the padded frames, where sigma2 = 0 and the rounding is largest
    assert dm <= 2e-3 and dl <= 4e-6 and dg <= 2e-7
    assert abs(mean.item() - float(g[f"{case}.mean"])) <= 2e-5


# ---- accuracy against float64 -----------------------------------------------------------------------------------------
def accuracy_cases():
    gen = torch.Generator().manual_seed(11)
    B, H, W = 8, 400, 80
    z = torch.nn.functional.avg_pool2d(torch.randn(B, 1, H, W, generator=gen), 7, stride=1, padding=3)
    tgt = -2.0 + 3.0 * z
    tgt[1, :, 300:] = 0
    out = tgt + 0.3 * torch.randn(B, 1, H, W, generator=gen)
    return {
        "mel": (out + 6, tgt + 6),
        "constant": (torch.full((B, 1, H, W), 6 - 2.3), torch.full((B, 1, H, W), 6 - 1.9)),
        "normal": (torch.randn(B, 1, H, W, generator=gen), torch.randn(B, 1, H, W, generator=gen)),
    }


@pytest.mark.parametrize("case", ["mel", "constant", "normal"])
def test_accuracy_against_float64(lib_built, case):
    x, y = (t.to(DEV) for t in accuracy_cases()[case])
    d_map = torch.randn(x.shape[0], x.shape[2], x.shape[3], generator=torch.Generator().manual_seed(3)).to(DEV)
    ref = eager_map_and_grads(x, y, d_map, dtype=torch.float64)
    dsx = errors(dsx_map_and_grads(x, y, d_map), ref)
    fp32 = errors(eager_map_and_grads(x, y, d_map), ref)
    dflt = errors(eager_map_and_grads(x, y, d_map, tf32=True), ref)
    names = ("map", "d_x", "d_y")
    print(f"accuracy {case}: " + json.dumps({n: dict(dsx=dsx[i], eager_fp32=fp32[i], eager_defaults=dflt[i])
                                             for i, n in enumerate(names)}))
    for i, n in enumerate(names):
        slack = SLACK * EPS32 * ref[i].abs().max().item()
        assert dsx[i][1] <= fp32[i][1], (n, dsx[i], fp32[i])
        assert dsx[i][0] <= fp32[i][0] + slack, (n, dsx[i], fp32[i], slack)


# ---- edges ------------------------------------------------------------------------------------------------------------
EDGES = [(H, W) for H in (1, 5, 11, 12, 63, 64, 65, 4500) for W in (1, 10, 80, 256)]


@pytest.mark.parametrize("H,W", EDGES, ids=[f"H{H}-W{W}" for H, W in EDGES])
def test_edges(lib_built, H, W):
    B = 64 if H <= 65 else 2
    gen = torch.Generator().manual_seed(H * 1000 + W)
    x = (torch.rand(B, 1, H, W, generator=gen) * 4 + 4).to(DEV)
    y = (x.cpu() + 0.5 * torch.randn(B, 1, H, W, generator=gen)).to(DEV)
    d_map = torch.randn(B, H, W, generator=gen).to(DEV)
    ref = eager_map_and_grads(x, y, d_map, dtype=torch.float64)
    dsx = errors(dsx_map_and_grads(x, y, d_map), ref)
    fp32 = errors(eager_map_and_grads(x, y, d_map), ref)
    for i, n in enumerate(("map", "d_x", "d_y")):
        bound = 2 * fp32[i][0] + 16 * EPS32 * ref[i].abs().max().item()
        assert dsx[i][0] <= bound, (n, dsx[i], fp32[i])


# ---- bitwise properties -----------------------------------------------------------------------------------------------
def test_batch_is_each_image_alone_and_calls_repeat(lib_built):
    x, y = (t[:5, :, :300].to(DEV).contiguous() for t in accuracy_cases()["mel"])
    d_map = torch.randn(5, 300, 80, generator=torch.Generator().manual_seed(4)).to(DEV)
    batch = dsx_map_and_grads(x, y, d_map)
    again = dsx_map_and_grads(x, y, d_map)
    for a, b in zip(batch, again):
        assert torch.equal(a, b)
    for i in range(5):
        alone = dsx_map_and_grads(x[i:i + 1], y[i:i + 1], d_map[i:i + 1])
        for a, b in zip(batch, alone):
            assert torch.equal(a[i:i + 1], b)


def test_gradients_only_where_required(lib_built):
    from diffsinger_b200 import DsxError, ssim
    x, y = (t[:2].to(DEV) for t in accuracy_cases()["mel"])
    xr = x.clone().requires_grad_(True)
    ssim(xr, y).backward()
    assert xr.grad is not None and not y.requires_grad and y.grad is None
    xb, yb = x.clone().requires_grad_(True), y.clone().requires_grad_(True)
    ssim(xb, yb).backward()
    assert torch.equal(xr.grad, xb.grad)
    yr = y.clone().requires_grad_(True)
    ssim(x, yr).backward()
    assert torch.equal(yr.grad, yb.grad)
    with torch.no_grad():
        v = ssim(x, y)
    assert v.dim() == 0 and not v.requires_grad and abs(v.item() - ssim(x, y).item()) == 0
    xr = x.clone().requires_grad_(True)
    with pytest.raises(DsxError, match="double backward"):
        torch.autograd.grad(ssim(xr, y), xr, create_graph=True)


def test_strided_inputs(lib_built):
    from diffsinger_b200 import ssim
    x, y = (t[:2].to(DEV) for t in accuracy_cases()["mel"])
    xt = x.transpose(2, 3).contiguous().transpose(2, 3)
    assert not xt.is_contiguous()
    assert torch.equal(ssim(xt, y, size_average=False), ssim(x, y, size_average=False))


# ---- the drop-in in a training loop -----------------------------------------------------------------------------------
def test_dropin_adam_run_matches_eager_fp32(lib_built, tmp_path, monkeypatch):
    """20 Adam steps of the dsx decoder (dsx_train) + mel_out + the stand-in task's l1:0.5|ssim:0.5 loss on one batch,
    once with the installed dsx ssim and once with eager fp32 (TF32 off); same initialisation and dropout draws"""
    from diffsinger_b200 import FastspeechDecoder
    from oracle import fs2dec_oracle as F
    install_tree(tmp_path, monkeypatch)
    import tasks.tts.fs2 as fs2
    import diffsinger_b200.dropin as dropin
    hp = dict(hidden_size=256, dec_layers=4, dec_ffn_kernel_size=9, num_heads=2, ffn_padding='SAME', ffn_act='gelu',
              dropout=0.1, dsx_train=True)
    B, T = 4, 200
    x = F.fixture_input(1, B, T, 256, tail=150).to(DEV)
    gen = torch.Generator().manual_seed(8)
    target = (torch.nn.functional.avg_pool2d(torch.randn(B, 1, T, 80, generator=gen), 5, 1, 2)[:, 0] * 3 - 2).to(DEV)
    target[1, 150:] = 0

    def run(ssim_fn):
        fs2.ssim = ssim_fn
        torch.manual_seed(0)
        dec = FastspeechDecoder(hparams=hp)
        dec.load_state_dict(F.random_state_dict(0, hp), strict=True)
        dec = dec.to(DEV).train()
        mel_out = torch.nn.Linear(256, 80).to(DEV)
        opt = torch.optim.Adam(list(dec.parameters()) + list(mel_out.parameters()), lr=1e-4)
        task, losses = fs2.MelLossTask("l1:0.5|ssim:0.5"), []
        for _ in range(20):
            opt.zero_grad()
            loss = task.mel_loss(mel_out(dec(x)), target)
            loss.backward()
            opt.step()
            losses.append(loss.item())
        dec.close()
        return losses

    prev = torch.backends.cudnn.allow_tf32
    new = dropin.install_ssim()
    try:
        assert fs2.ssim is new
        got = run(new)
        torch.backends.cudnn.allow_tf32 = False
        ref = run(O.ssim)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
        dropin.uninstall_ssim()
    d = np.abs(np.array(got) - np.array(ref))
    print(f"adam: loss {ref[0]:.5f} -> {ref[-1]:.5f}, max |d loss| over 20 steps {d.max():.2e}")
    assert ref[-1] < ref[0]
    assert d.max() <= 1e-4, d
    drop_tree()
