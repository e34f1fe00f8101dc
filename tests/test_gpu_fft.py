"""GPU: the FFT diffusion denoiser of libdsx.so against the reference's outputs (tests/golden/fft_denoiser.npz) and the
oracle (oracle/fft_oracle.py, run here in fp32 with TF32 off), inside the sampler handle's loops.

The entry GEMM (input_projection folded into get_decode_inp) and the cond part use hi+lo fp16 operand pairs, the step
part is fp32, the FFTBlocks stack rounds its GEMM operands to fp16 as the FastSpeech2 decoder does, and get_mel_out
reads the final LayerNorm as fp16.  oracle.fft_oracle.loop_error simulates that rounding on the CPU (H 256, L 4, B 2,
T 200): one evaluation is off by max 2.2e-3 / mean 4.2e-4 in eps (the decoder alone: 1.2e-3 / 1.6e-4), and a K = 51
DDPM infer loop by max 1.05e-2 / mean 5.8e-4 in the denormalised mel (|mel| up to 6).  The bounds below are about 5x
those: eps max 1e-2 / mean 2e-3, mel max 5e-2 / mean 3e-3.  Masked frames must be exactly 0."""
import sys
import textwrap

import numpy as np
import pytest
import torch

from conftest import golden
from oracle import diffnet_oracle as N
from oracle import fft_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
EPS_MAX, EPS_MEAN = 1e-2, 2e-3
MEL_MAX, MEL_MEAN = 5e-2, 3e-3


def fixture():
    g = golden("fft_denoiser.npz")
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    return g, hp, O.random_state_dict(int(g["seed"]), hp)


def model(hp, sd):
    from diffsinger_b200 import FFT
    m = FFT(hparams=hp)
    m.load_state_dict(sd, strict=True)
    return m.eval().to(DEV)


def schedule(g):
    return N.make_schedule(N.linear_beta_schedule(int(g["timesteps"]), float(g["max_beta"])))


def check(out, ref, mx, mean, mask=None):
    out, ref = np.asarray(out.cpu() if torch.is_tensor(out) else out, np.float64), np.asarray(ref, np.float64)
    d = np.abs(out - ref)
    assert np.isfinite(out).all()
    assert d.max() <= mx and d.mean() <= mean, (d.max(), d.mean())
    if mask is not None:
        assert (out[mask] == 0).all()


def sampler(m, g):
    s = m.dsx
    s.ensure_weights(DEV)
    s.set_schedule(schedule(g))
    return s


def infer(s, g, cond, fs2_mel, start, noise=None, mel2ph=None, interval=0):
    t = lambda a: torch.from_numpy(a).to(DEV) if isinstance(a, np.ndarray) else a.to(DEV)
    return s.infer(t(cond), int(g["K_step"]), t(g["spec_min"]), t(g["spec_max"]), fs2_mel=t(fs2_mel),
                   start_noise=t(start), step_noise=None if noise is None else t(noise),
                   mel2ph=None if mel2ph is None else t(mel2ph), pndm_interval=interval)


# ---- the reference's fixture -------------------------------------------------------------------------------------------
def test_reference_evaluations(lib_built):
    g, hp, sd = fixture()
    m = model(hp, sd)
    with torch.no_grad():
        for i, t in enumerate(g["t"]):       # the last row has a different t per utterance
            out = m(torch.from_numpy(g["spec"]).to(DEV), torch.from_numpy(t).to(DEV), torch.from_numpy(g["cond"]).to(DEV))
            check(out, g["eps"][i], EPS_MAX, EPS_MEAN)


def test_reference_ddpm_infer_with_mask(lib_built):
    g, hp, sd = fixture()
    s = sampler(model(hp, sd), g)
    B, _, T = g["cond_loop"].shape
    noise = O.step_noise(int(g["noise_seed"]), int(g["K_step"]), B, T)
    out = infer(s, g, g["cond_loop"], g["fs2_mel"], g["start_noise"], noise, g["mel2ph"])
    check(out, g["mel_ddpm"], MEL_MAX, MEL_MEAN, mask=g["mel2ph"] == 0)


def test_reference_plms_infer(lib_built):
    g, hp, sd = fixture()
    s = sampler(model(hp, sd), g)
    out = infer(s, g, g["cond_plms"], g["fs2_mel_plms"], g["start_noise_plms"], interval=int(g["interval"]))
    check(out, g["mel_plms"], MEL_MAX, MEL_MEAN)


# ---- the oracle ---------------------------------------------------------------------------------------------------
def oracle_gpu(fn):
    mm, cu = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        with torch.no_grad():
            return fn()
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = mm, cu


CASES = {
    "T1": dict(T=1),
    "T37": dict(T=37),
    "T1000": dict(T=1000),
    "T3000": dict(T=3000),
    "H128_heads1": dict(T=300, hp=dict(hidden_size=128, num_heads=1)),
    "H128_heads2": dict(T=130, hp=dict(hidden_size=128, num_heads=2)),
    "residual128_hidden256": dict(T=200, hp=dict(residual_channels=128)),
    "left_k4": dict(T=200, hp=dict(ffn_padding='LEFT', dec_ffn_kernel_size=4)),
    "relu": dict(T=200, hp=dict(ffn_act='relu')),
    "L1": dict(T=200, hp=dict(dec_layers=1)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_against_the_oracle(lib_built, case):
    c = CASES[case]
    hp = dict(O.HPARAMS_POPCS, **c.get("hp", {}))
    sd = O.random_state_dict(51, hp)
    T, B = c["T"], 3
    gen = torch.Generator().manual_seed(52)
    spec = torch.randn(B, 1, 80, T, generator=gen).to(DEV)
    cond = torch.randn(B, hp["hidden_size"], T, generator=gen).to(DEV)
    t = torch.tensor([99, 40, 0], device=DEV)                    # per-utterance t through dsx_diffnet_forward
    with torch.no_grad():
        out = model(hp, sd)(spec, t, cond)
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    ref = oracle_gpu(lambda: O.forward(sdd, spec, t, cond, hp))
    check(out, ref.cpu(), EPS_MAX, EPS_MEAN)


def test_ddpm_loop_against_the_oracle(lib_built):
    hp = O.HPARAMS_POPCS
    sd = O.random_state_dict(53, hp)
    g = golden("fft_denoiser.npz")
    m = model(hp, sd)
    s = sampler(m, g)
    cond, fs2_mel, mel2ph, start = O.fixture_inputs(54, 2, 500, hp)
    noise = O.step_noise(55, 51, 2, 500)
    out = infer(s, g, cond, fs2_mel, start, noise, mel2ph)
    S = {k: v.to(DEV) for k, v in schedule(g).items()}
    sdd = {k: v.to(DEV) for k, v in sd.items()}
    d = lambda a: a.to(DEV)
    ref = oracle_gpu(lambda: O.infer_loop(lambda *a: O.forward(sdd, *a, hp), S, d(cond), 51,
                                          d(torch.from_numpy(g["spec_min"])), d(torch.from_numpy(g["spec_max"])),
                                          fs2_mel=d(fs2_mel), start_noise=d(start), step_noise=d(noise),
                                          mel2ph=d(mel2ph)))
    check(out, ref.cpu(), MEL_MAX, MEL_MEAN, mask=(mel2ph == 0).numpy())


# ---- bit identity ---------------------------------------------------------------------------------------------------
def test_batch_matches_each_utterance_alone(lib_built):
    g, hp, sd = fixture()
    s = sampler(model(hp, sd), g)
    cond, _, _, _ = O.fixture_inputs(56, 3, 150, hp)
    x = torch.randn(3, 1, 80, 150, generator=torch.Generator().manual_seed(57)).to(DEV)
    noise = O.step_noise(58, 6, 3, 150).to(DEV)
    cond = cond.to(DEV)
    out = s.sample_ddpm(x, cond, 51, 6, noise=noise)
    for b in range(3):
        assert torch.equal(out[b:b + 1], s.sample_ddpm(x[b:b + 1], cond[b:b + 1], 51, 6, noise=noise[:, b:b + 1])), b


def test_two_calls_are_identical(lib_built):
    g, hp, sd = fixture()
    s = sampler(model(hp, sd), g)
    cond, fs2_mel, mel2ph, start = O.fixture_inputs(59, 2, 300, hp)
    a = infer(s, g, cond, fs2_mel, start, O.step_noise(60, 51, 2, 300), mel2ph)
    b = infer(s, g, cond, fs2_mel, start, O.step_noise(60, 51, 2, 300), mel2ph)
    assert torch.equal(a, b)


def test_strided_cond_is_bit_identical(lib_built):
    g, hp, sd = fixture()
    m = model(hp, sd)
    cond_bth = torch.randn(2, 120, 256, generator=torch.Generator().manual_seed(61)).to(DEV)   # decoder_inp [B, T, H]
    x = torch.randn(2, 1, 80, 120, generator=torch.Generator().manual_seed(62)).to(DEV)
    t = torch.tensor([30, 31], device=DEV)
    with torch.no_grad():
        a = m(x, t, cond_bth.transpose(1, 2)).clone()
        b = m(x, t, cond_bth.transpose(1, 2).contiguous())
    assert torch.equal(a, b)


def _diffusion(denoise_fn, g):
    from diffsinger_b200 import GaussianDiffusion
    return GaussianDiffusion(None, 80, denoise_fn, timesteps=int(g["timesteps"]), K_step=int(g["K_step"]),
                             betas=N.linear_beta_schedule(int(g["timesteps"]), float(g["max_beta"])),
                             spec_min=list(g["spec_min"].reshape(-1)), spec_max=list(g["spec_max"].reshape(-1)),
                             fs2=torch.nn.Identity(), hparams=dict(keep_bins=80)).to(DEV).eval()


def test_fused_ddpm_matches_per_step_p_sample(lib_built):
    g, hp, sd = fixture()
    gd = _diffusion(model(hp, sd), g)
    cond = torch.randn(2, 256, 90, generator=torch.Generator().manual_seed(63)).to(DEV)
    x0 = torch.randn(2, 1, 80, 90, generator=torch.Generator().manual_seed(64)).to(DEV)
    K = 8
    torch.manual_seed(65)
    x = x0
    for i in reversed(range(K)):
        x = gd.p_sample(x, torch.full((2,), i, device=DEV, dtype=torch.long), cond)
    torch.manual_seed(65)
    noise = torch.cat([torch.randn((1, 2, 1, 80, 90), device=DEV) for _ in range(K)])
    fused = gd._dsx_ready(DEV).sample_ddpm(x0, cond, K, K, noise=noise)
    assert torch.equal(x, fused)


def test_fused_plms_matches_per_step_p_sample_plms(lib_built):
    g, hp, sd = fixture()
    gd = _diffusion(model(hp, sd), g)
    cond = torch.randn(1, 256, 70, generator=torch.Generator().manual_seed(66)).to(DEV)
    x0 = torch.randn(1, 1, 80, 70, generator=torch.Generator().manual_seed(67)).to(DEV)
    K, interval = 51, 10
    gd.noise_list.clear()
    x = x0
    for i in reversed(range(0, K, interval)):
        x = gd.p_sample_plms(x, torch.full((1,), i, device=DEV, dtype=torch.long), interval, cond)
    fused = gd._dsx_ready(DEV).sample_plms(x0, cond, K, interval)
    assert torch.equal(x, fused)


# ---- one handle, two denoisers --------------------------------------------------------------------------------------
def test_handle_switching_diffnet_fft_diffnet(lib_built):
    import diffsinger_b200 as dsx
    from conftest import HP
    g, hp, sd = fixture()
    fft = model(hp, sd)
    torch.manual_seed(0)
    net = dsx.DiffNet(80, hparams=HP)
    torch.nn.init.normal_(net.output_projection.weight, std=0.02)
    net = net.to(DEV).eval()
    cond = torch.randn(2, 256, 100, generator=torch.Generator().manual_seed(68)).to(DEV)
    x = torch.randn(2, 1, 80, 100, generator=torch.Generator().manual_seed(69)).to(DEV)
    noise = O.step_noise(70, 4, 2, 100).to(DEV)
    S = schedule(g)

    def run(s):
        s.ensure_weights(DEV)
        s.set_schedule(S)
        return s.sample_ddpm(x, cond, 51, 4, noise=noise)

    fresh_net, fresh_fft = run(dsx.DsxSampler(net, "fp16s")), run(dsx.DsxSampler(fft))
    dec_ref = _decoder_fixture_output()
    shared = dsx.DsxSampler(net, "fp16s")
    a = run(shared)
    shared.net = fft
    b = run(shared)
    assert shared.info(_capi().INFO_PRECISION) == _capi().PREC_FP16
    shared.net = net
    c = run(shared)
    assert torch.equal(a, fresh_net) and torch.equal(b, fresh_fft) and torch.equal(c, fresh_net)
    assert torch.equal(_decoder_fixture_output(), dec_ref)


def test_diffnet_only_debug_calls_refuse_an_fft_handle(lib_built):
    from diffsinger_b200 import DsxError
    g, hp, sd = fixture()
    s = sampler(model(hp, sd), g)
    for call in (lambda: s.set_layer_limit(2), lambda: s.debug_read(0, 1, 4)):
        with pytest.raises(DsxError, match="FFT"):
            call()
    s.set_option(_capi().OPT_STACK_KERNEL, 0)          # DiffNet-only knobs are accepted and ignored


def _capi():
    from diffsinger_b200 import _capi
    return _capi


def _decoder_fixture_output():
    from diffsinger_b200 import FastspeechDecoder
    from oracle import fs2dec_oracle as D
    d = golden("fs2_decoder.npz")
    hp = {k[3:]: d[k].item() for k in d.files if k.startswith("hp.")}
    dec = FastspeechDecoder(hparams=hp)
    dec.load_state_dict(D.random_state_dict(int(d["seed"]), hp), strict=True)
    with torch.no_grad():
        out = dec.eval().to(DEV)(torch.from_numpy(d["x"]).to(DEV)).cpu()
    dec.close()
    return out


# ---- drop-in ----------------------------------------------------------------------------------------------------------
CANDIDATE = """
    import torch
    import torch.nn as nn
    from diffsinger_b200.fs2dec import TransformerEncoderLayer
    from diffsinger_b200.modules import Conv1d, Mish, SinusoidalPosEmb
    from diffsinger_b200.pitch import SinusoidalPositionalEmbedding
    from utils.hparams import hparams

    class FFT(nn.Module):      # usr/diff/candidate_decoder.py:35-48: the reference's parameters; its forward must not run
        def __init__(self, hidden_size=None, num_layers=None, kernel_size=None, num_heads=None):
            super().__init__()
            H, dim = hidden_size, hparams['residual_channels']
            self.pos_embed_alpha = nn.Parameter(torch.Tensor([1]))
            self.embed_positions = SinusoidalPositionalEmbedding(H, 0)
            self.layers = nn.ModuleList([TransformerEncoderLayer(H, kernel_size, num_heads, hparams['ffn_padding'],
                                                                 hparams['ffn_act']) for _ in range(num_layers)])
            self.layer_norm = nn.LayerNorm(H)
            self.input_projection = Conv1d(hparams['audio_num_mel_bins'], dim, 1)
            self.diffusion_embedding = SinusoidalPosEmb(dim)
            self.mlp = nn.Sequential(nn.Linear(dim, dim * 4), Mish(), nn.Linear(dim * 4, dim))
            self.get_mel_out = nn.Linear(H, 80, bias=True)
            self.get_decode_inp = nn.Linear(H + dim + dim, H)

        def forward(self, *a, **k):
            raise RuntimeError("stand-in FFT.forward: inference must run on dsx")
"""
TASK = """
    from .diff.shallow_diffusion_tts import GaussianDiffusion, OfflineGaussianDiffusion
    from .diff.net import DiffNet
    from .diff.candidate_decoder import FFT

    DIFF_DECODERS = {
        'wavenet': lambda hp: DiffNet(hp['audio_num_mel_bins']),
        'fft': lambda hp: FFT(hp['hidden_size'], hp['dec_layers'], hp['dec_ffn_kernel_size'], hp['num_heads']),
    }
"""


def test_dropin_reference_fft_runs_on_dsx(lib_built, tmp_path, monkeypatch):
    from standin_ref import write_tree
    tree = write_tree(str(tmp_path / "standin"))
    (tmp_path / "standin" / "usr" / "diff" / "candidate_decoder.py").write_text(textwrap.dedent(CANDIDATE).lstrip("\n"))
    (tmp_path / "standin" / "usr" / "diffsinger_task.py").write_text(textwrap.dedent(TASK).lstrip("\n"))
    monkeypatch.syspath_prepend(tree)
    roots = ("usr", "utils")
    drop = lambda: [n for n in sys.modules if n in roots or n.startswith(tuple(r + "." for r in roots))]
    for n in drop():
        monkeypatch.delitem(sys.modules, n)
    g, hp, sd = fixture()
    import utils.hparams
    utils.hparams.hparams.update(hp, keep_bins=80, diff_decoder_type='fft')
    import usr.diffsinger_task as task
    import diffsinger_b200.dropin as dropin
    new_cls = dropin.install()
    try:
        assert task.GaussianDiffusion is new_cls
        net = task.DIFF_DECODERS['fft'](utils.hparams.hparams)
        assert type(net).__module__ == "usr.diff.candidate_decoder"
        net.load_state_dict(sd, strict=True)
        m = task.GaussianDiffusion(None, 80, net, timesteps=int(g["timesteps"]), K_step=int(g["K_step"]),
                                   betas=N.linear_beta_schedule(int(g["timesteps"]), float(g["max_beta"])),
                                   spec_min=list(g["spec_min"].reshape(-1)), spec_max=list(g["spec_max"].reshape(-1)))
        m = m.to(DEV).eval()
        cond = torch.from_numpy(g["cond_loop"]).to(DEV)
        fs2_mel = torch.from_numpy(g["fs2_mel"]).to(DEV)

        class Stub(torch.nn.Module):
            def forward(self, *a, **k):
                return {"decoder_inp": cond.transpose(1, 2).clone(), "mel_out": fs2_mel.clone()}

        m.fs2 = Stub()
        B, _, T = g["cond_loop"].shape
        ret = m(torch.zeros(B, 5, dtype=torch.long, device=DEV), mel2ph=torch.from_numpy(g["mel2ph"]).to(DEV), infer=True,
                dsx_step_noise=O.step_noise(int(g["noise_seed"]), int(g["K_step"]), B, T).to(DEV),
                dsx_start_noise=torch.from_numpy(g["start_noise"]).to(DEV))
        check(ret["mel_out"], g["mel_ddpm"], MEL_MAX, MEL_MEAN, mask=g["mel2ph"] == 0)
        assert torch.equal(ret["fs2_mel"], fs2_mel)
    finally:
        dropin.uninstall()
    for n in drop():
        del sys.modules[n]
