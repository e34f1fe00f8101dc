"""The launch plan of one evaluation and what follows it, per denoiser, precision and option set, read through the
DSX_INFO_* counters.  In a sampling loop one evaluation is:

  fp32 (SIMT)      input projection, 4 launches per layer, the head (4), then the DDPM or PLMS update kernel
  FFT              its evaluation (5 + 5 per FFTBlock), then the update kernel
  fp16 / fp16x2 /  the stack form (all layers, head, update and next input projection in ONE launch), or with
  fp16s            DSX_OPT_FUSED_HEAD = 0 or DSX_OPT_PROFILE = 2 that launch without the head, then a head launch
  fp16x3, or any   all layers in one launch with the hi / lo weight planes (DSX_OPT_STACK_MODE = 1) or one launch per
  tensor-core      layer (STACK_MODE = 0), then a head launch; DSX_OPT_STACK_KERNEL = 0 puts fp16 / fp16x2 / fp16s here
  precision        too

A tensor-core loop's first evaluation and every dsx_diffnet_forward are preceded by an input-projection launch.
DSX_OPT_PROFILE = 1 brackets the layers of every DiffNet evaluation; 2 brackets the tensor-core head launch of every
evaluation (DDPM, PLMS and forward).
Run on an H100: python -m pytest tests -m gpu"""
import numpy as np
import pytest
import torch

from conftest import GOLDEN, HP, rs_normal
from oracle import diffnet_oracle as N
from oracle import fft_oracle as F

pytestmark = pytest.mark.gpu

L = 4                       # DiffNet residual layers
B, T = 2, 96
EMBED = 2                   # step-table launches of every call (the embedding MLP and its projection)
PLMS_START, PLMS_INTERVAL = 100, 25      # steps t = 75, 50, 25, 0: four steps, five evaluations with the warm-up
PRECISIONS = ["fp32", "fp16", "fp16x2", "fp16x3", "fp16s", "fft"]
OPTIONS = {"default": {}, "separate_head": {"FUSED_HEAD": 0}, "hilo_layers": {"STACK_KERNEL": 0},
           "per_layer": {"STACK_MODE": 0}}


@pytest.fixture(scope="module")
def dsx(lib_built):
    import diffsinger_b200
    assert torch.cuda.is_available()
    return diffsinger_b200


def make_sampler(dsx, prec):
    dev = torch.device("cuda", 0)
    if prec == "fft":
        g = np.load(f"{GOLDEN}/fft_denoiser.npz")
        hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
        m = dsx.FFT(hparams=hp)
        m.load_state_dict(F.random_state_dict(int(g["seed"]), hp), strict=True)
        s = m.eval().to(dev).dsx
        s.ensure_weights(dev)
        return s, dev, hp["hidden_size"], 5 + 5 * hp["dec_layers"]
    torch.manual_seed(0)
    net = dsx.DiffNet(80, hparams=dict(HP, residual_layers=L)).to(dev).eval()
    s = dsx.DsxSampler(net, prec, 1)
    s.ensure_weights(dev)
    return s, dev, 256, None


def plan(prec, opts, profile, fft_eval):
    """Launches of one evaluation in a loop without its update kernel, update kernels per evaluation, input-projection
    launches before a loop or forward, stack-form launches and profile brackets per evaluation."""
    if prec == "fft":
        return dict(eval=fft_eval, update=1, pre=0, stack=0, brackets=0)
    if prec == "fp32":
        return dict(eval=1 + 4 * L + 4, update=1, pre=0, stack=0, brackets=int(profile == 1))
    kernel, mode, fused = opts.get("STACK_KERNEL", 1), opts.get("STACK_MODE", 1), opts.get("FUSED_HEAD", 1)
    stack = prec in ("fp16", "fp16x2", "fp16s") and kernel and mode
    if stack:
        ev = 1 if fused and profile != 2 else 2
    else:
        ev = 2 if mode else L + 1
    return dict(eval=ev, update=0, pre=1, stack=int(stack), brackets=int(profile in (1, 2)))


@pytest.mark.parametrize("profile", [0, 1, 2])
@pytest.mark.parametrize("options", list(OPTIONS))
@pytest.mark.parametrize("prec", PRECISIONS)
def test_launch_plan(dsx, prec, options, profile):
    from diffsinger_b200 import _capi
    opts = OPTIONS[options]
    s, dev, H, fft_eval = make_sampler(dsx, prec)
    s.set_schedule(N.make_schedule(N.linear_beta_schedule(100, 0.06)))
    for k, v in opts.items():
        s.set_option(getattr(_capi, "OPT_" + k), v)
    x, cond = rs_normal(1, (B, 1, 80, T)).to(dev), rs_normal(2, (B, H, T)).to(dev)
    t = torch.tensor([3, 70], device=dev)
    s.diffnet_forward(x, t, cond)                   # packs the conditioner; the calls below re-use it
    s.set_option(_capi.OPT_PROFILE, profile)
    p = plan(prec, opts, profile, fft_eval)
    counters = (_capi.INFO_KERNEL_LAUNCHES, _capi.INFO_STACK_KERNEL_LAUNCHES, _capi.INFO_LAYER_KERNEL_LAUNCHES)

    def delta(call):
        before = [s.info(c) for c in counters]
        call()
        launches, stack, brackets = (s.info(c) - b for c, b in zip(counters, before))
        return launches - EMBED, stack, brackets

    per_eval = (p["eval"], p["stack"], p["brackets"])
    # dsx_diffnet_forward: input projection + one evaluation to eps, no update
    assert delta(lambda: s.diffnet_forward(x, t, cond)) == (p["pre"] + p["eval"],) + per_eval[1:]
    # DDPM: K evaluations, each followed by its update
    for K in (1, 4):
        launches, stack, brackets = delta(lambda: s.sample_ddpm(x, cond, 100, K, seed=1))
        assert (launches - p["pre"]) / K == p["eval"] + p["update"], (K, launches)
        assert (stack, brackets) == (K * p["stack"], K * p["brackets"])
    # PLMS: four steps, the first with the warm-up's second evaluation, each evaluation followed by its update
    n_eval = PLMS_START // PLMS_INTERVAL + 1
    launches, stack, brackets = delta(lambda: s.sample_plms(x, cond, PLMS_START, PLMS_INTERVAL))
    assert launches == p["pre"] + n_eval * (p["eval"] + p["update"]), launches
    assert (stack, brackets) == (n_eval * p["stack"], n_eval * p["brackets"])
    s.close()
