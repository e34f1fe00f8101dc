"""TEST INFRASTRUCTURE ONLY -- pins oracle/fft_oracle.py to the LIVE reference FFT denoiser and its sampling loops (needs a
checkout of the reference: DSX_REFERENCE_ROOT) and writes tests/golden/fft_denoiser.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_fft.py

The reference's FFT (usr/diff/candidate_decoder.py:35-100) and GaussianDiffusion (usr/diff/shallow_diffusion_tts.py) are
imported unmodified (stubs only for librosa / pycwt) under usr/configs/popcs_ds_beta6.yaml (hidden 256, 4 layers, 2 heads,
kernel 9, GELU, 'SAME', residual_channels 256, linear schedule T = 100, max_beta 0.06, K_step 51).  The parameters are
fft_oracle.random_state_dict(SEED), loaded strictly; the oracle must reproduce, bit for bit:
  * three evaluations at different t, with per-utterance t inside one batch;
  * GaussianDiffusion.forward(infer=True) with denoise_fn = FFT: the K = 51 DDPM shallow start with a mel2ph mask (B = 2),
    the step noise injected through noise_like and the start noise through randn_like (as oracle/gen_golden.py does);
  * the same with pndm_speedup = 10 (PLMS) at B = 1, because the reference's PLMS raises at B > 1.
Only per-tensor float64 checksums of the weights are stored; the tests regenerate them, and the step noise, from seeds."""
import os
import sys
from collections import deque

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import diffnet_oracle as N  # noqa: E402
from oracle import fft_oracle as O  # noqa: E402
from oracle import fs2dec_oracle as D  # noqa: E402
from oracle import ref_bridge  # noqa: E402

CONFIG = "usr/configs/popcs_ds_beta6.yaml"
HP_KEYS = ("hidden_size", "dec_layers", "dec_ffn_kernel_size", "num_heads", "ffn_padding", "ffn_act", "dropout",
           "residual_channels", "audio_num_mel_bins")
SEED, EVAL_SEED, LOOP_SEED, NOISE_SEED, PLMS_SEED = 41, 42, 43, 44, 45
B, T, PLMS_T, INTERVAL = 2, 96, 80, 10


def main():
    assert ref_bridge.available(), "set DSX_REFERENCE_ROOT to a checkout of the reference"
    torch.set_num_threads(8)
    ns = ref_bridge.load(CONFIG)
    hparams, sdt = ns.hparams, ns.sdt
    cwd = os.getcwd()
    os.chdir(ref_bridge.REF_ROOT)
    try:
        from usr.diff.candidate_decoder import FFT
    finally:
        os.chdir(cwd)
    hp = {k: hparams[k] for k in HP_KEYS}
    assert (hp["hidden_size"], hp["dec_layers"], hp["num_heads"], hp["dec_ffn_kernel_size"], hp["ffn_act"],
            hp["residual_channels"]) == (256, 4, 2, 9, "gelu", 256), hp
    K_step, timesteps = hparams["K_step"], hparams["timesteps"]
    assert (K_step, timesteps, hparams["schedule_type"], hparams["max_beta"]) == (51, 100, "linear", 0.06)

    net = FFT(hp["hidden_size"], hp["dec_layers"], hp["dec_ffn_kernel_size"], hp["num_heads"]).eval()
    sd = O.random_state_dict(SEED, hp)
    assert list(net.state_dict()) == list(sd), "state-dict names and order"
    assert {k: tuple(v.shape) for k, v in net.state_dict().items()} == {k: tuple(v.shape) for k, v in sd.items()}
    net.load_state_dict(sd, strict=True)
    fn = lambda spec, t, cond: O.forward(sd, spec, t, cond, hp)

    # ---- 1. evaluations ------------------------------------------------------------------------------------------------
    rs = np.random.RandomState(EVAL_SEED)
    spec = torch.from_numpy(rs.standard_normal((B, 1, 80, T)).astype(np.float32))
    cond = torch.from_numpy(rs.standard_normal((B, hp["hidden_size"], T)).astype(np.float32))
    ts = torch.tensor([[99, 99], [0, 0], [50, 7]], dtype=torch.long)          # the last: per-utterance t
    evals = []
    with torch.no_grad():
        for t in ts:
            ref = net(spec, t, cond)
            assert torch.equal(ref, fn(spec, t, cond)), t
            evals.append(ref)
    evals = torch.stack(evals)

    # ---- 2. GaussianDiffusion.forward(infer=True), DDPM K = 51 with a mel2ph mask -----------------------------------------
    enc = ns.TokenTextEncoder(None, vocab_list=["a", "b", "c"], replace_oov=",")
    gd = sdt.GaussianDiffusion(enc, 80, net, timesteps=timesteps, K_step=K_step, loss_type="l1",
                               spec_min=hparams["spec_min"], spec_max=hparams["spec_max"]).eval()
    S = N.make_schedule(N.linear_beta_schedule(timesteps, 0.06))
    for k in N.SCHEDULE_BUFFERS:
        assert torch.equal(getattr(gd, k), S[k]), k
    cond_l, fs2_mel, mel2ph, start = O.fixture_inputs(LOOP_SEED, B, T, hp)
    noise = O.step_noise(NOISE_SEED, K_step, B, T)

    def run(cond_in, fs2_in, m2p, start_in, noise_in, pndm):
        feed = {"i": 0}

        def fake_noise_like(shape, device, repeat=False):
            n = noise_in[feed["i"]]
            feed["i"] += 1
            assert tuple(shape) == tuple(n.shape)
            return n

        class StubFS2(torch.nn.Module):
            def forward(self, *a, **kw):
                return {"decoder_inp": cond_in.transpose(1, 2).clone(), "mel_out": fs2_in.clone()}

        gd.fs2 = StubFS2()
        gd.noise_list = deque(maxlen=4)
        orig = sdt.noise_like, sdt.torch.randn_like, hparams.get("pndm_speedup")
        sdt.noise_like = fake_noise_like
        sdt.torch.randn_like = lambda x: start_in             # q_sample's default noise (:207)
        hparams["pndm_speedup"] = pndm
        try:
            with torch.no_grad():
                return gd(torch.zeros(cond_in.shape[0], 5, dtype=torch.long), mel2ph=m2p, infer=True)["mel_out"]
        finally:
            sdt.noise_like, sdt.torch.randn_like = orig[0], orig[1]
            hparams["pndm_speedup"] = orig[2]

    smin, smax = gd.spec_min, gd.spec_max
    ddpm = run(cond_l, fs2_mel, mel2ph, start, noise, 0)
    with torch.no_grad():
        mo = O.infer_loop(fn, S, cond_l, K_step, smin, smax, fs2_mel=fs2_mel, start_noise=start, step_noise=noise,
                          mel2ph=mel2ph)
    print(f"DDPM K={K_step}: oracle vs live reference max |d| = {(ddpm - mo).abs().max().item():.3e}")
    assert torch.equal(ddpm, mo), "the oracle's DDPM loop must reproduce the reference bit for bit"
    assert (ddpm[1, 3 * T // 4:] == 0).all()

    # ---- 3. PLMS (pndm_speedup = 10) at B = 1 ------------------------------------------------------------------------
    cond_p, fs2_p, _, start_p = O.fixture_inputs(PLMS_SEED, 1, PLMS_T, hp)
    plms = run(cond_p, fs2_p, None, start_p, None, INTERVAL)
    with torch.no_grad():
        po = O.infer_loop(fn, S, cond_p, K_step, smin, smax, fs2_mel=fs2_p, start_noise=start_p, pndm_speedup=INTERVAL)
    print(f"PLMS interval {INTERVAL}: oracle vs live reference max |d| = {(plms - po).abs().max().item():.3e}")
    assert torch.equal(plms, po), "the oracle's PLMS loop must reproduce the reference bit for bit"

    out = os.path.join(ROOT, "tests", "golden", "fft_denoiser.npz")
    np.savez_compressed(
        out, seed=np.int64(SEED), spec=spec.numpy(), cond=cond.numpy(), t=ts.numpy(), eps=evals.numpy(),
        loop_seed=np.int64(LOOP_SEED), noise_seed=np.int64(NOISE_SEED), K_step=np.int64(K_step),
        timesteps=np.int64(timesteps), max_beta=np.float64(0.06), cond_loop=cond_l.numpy(), fs2_mel=fs2_mel.numpy(),
        mel2ph=mel2ph.numpy(), start_noise=start.numpy(), mel_ddpm=ddpm.numpy(),
        noise_checksum=np.float64(noise.double().sum().item()),
        plms_seed=np.int64(PLMS_SEED), interval=np.int64(INTERVAL), cond_plms=cond_p.numpy(), fs2_mel_plms=fs2_p.numpy(),
        start_noise_plms=start_p.numpy(), mel_plms=plms.numpy(), spec_min=smin.numpy(), spec_max=smax.numpy(),
        **{"hp." + k: np.asarray(v) for k, v in hp.items()},
        **{"cks." + k: v for k, v in D.checksums(sd).items()})
    print("wrote", out, os.path.getsize(out) // 1024, "KB;", len(sd), "state-dict entries")


if __name__ == "__main__":
    main()
