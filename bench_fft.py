"""Sampling loops with the FFT diffusion denoiser on one GPU: ms per loop, ms per evaluation and mel frames per second.

    python bench_fft.py [--iters N] [--kernels]

The denoiser is popcs_ds_beta6's FFT (hidden 256, 4 layers, 2 heads, FFN kernel 9, GELU, 'SAME', residual_channels 256)
with seeded weights (oracle.fft_oracle.random_state_dict).  Three workloads, each a whole dsx_infer call (shallow start
from a seeded fs2 mel, mel2ph mask, injected start and step noise so that every implementation sees the same draws):
  * DDPM K = 51 of the T = 100, max_beta 0.06 schedule (popcs_ds_beta6) at B = 16, T = 1024 and at B = 1, T = 4000;
  * PLMS K = 1000 with interval 40 of the T = 1000, max_beta 0.02 schedule (the ds1000 setting: 26 evaluations) at
    B = 16, T = 1024.
Baselines in the same process, timed the same way: the reference's loop in PyTorch eager (oracle.fft_oracle.infer_loop,
the ATen ops the reference runs) in fp32 with TF32 off, and with the FFTBlocks stack and get_mel_out in .half()
(get_decode_inp stays fp32: the reference's step embedding cannot run in half); and the dsx DiffNet sampler (20 layers,
256 channels, its default precision) on the same loop.  Errors are of the mel against the eager fp32 loop.  Times come
from CUDA events around whole calls after a warm-up call.  --kernels adds the summed device time per kernel name of one
dsx call (torch.profiler).  The card's name, power limit and max SM clock are read once; the SM clock again right after
each dsx loop.  Prints one JSON line; writes nothing.
"""
import argparse
import json

import torch
import torch.nn.functional as F

import diffsinger_b200 as dsx
from bench_pe import gpu_info, kernel_times, timed
from oracle import diffnet_oracle as N
from oracle import fft_oracle as O
from oracle import fs2dec_oracle as D

WORKLOADS = (dict(name="ddpm_k51", B=16, T=1024, K=51, interval=0, timesteps=100, max_beta=0.06),
             dict(name="ddpm_k51", B=1, T=4000, K=51, interval=0, timesteps=100, max_beta=0.06),
             dict(name="plms_k1000_i40", B=16, T=1024, K=1000, interval=40, timesteps=1000, max_beta=0.02))


def evaluations(K, interval):
    return K if not interval else len(range(0, K, interval)) + 1


def run(w, iters, kernels):
    dev = torch.device("cuda", 0)
    B, T, K, interval = w["B"], w["T"], w["K"], w["interval"]
    hp = dict(O.HPARAMS_POPCS)
    sd = O.random_state_dict(1, hp)
    net = dsx.FFT(hparams=hp)
    net.load_state_dict(sd, strict=True)
    net = net.eval().to(dev)
    S = N.make_schedule(N.linear_beta_schedule(w["timesteps"], w["max_beta"]))
    s = net.dsx
    s.ensure_weights(dev)
    s.set_schedule(S)
    cond, fs2_mel, mel2ph, start = (v.to(dev) for v in O.fixture_inputs(2, B, T, hp))
    noise = O.step_noise(3, K, B, T).to(dev) if not interval else None
    smin, smax = torch.full((80,), -6.0, device=dev), torch.full((80,), 1.5, device=dev)
    call = lambda smp: smp.infer(cond, K, smin, smax, fs2_mel=fs2_mel, start_noise=start, step_noise=noise, mel2ph=mel2ph,
                                 pndm_interval=interval)
    n_eval = evaluations(K, interval)
    l0 = s.info(dsx._capi.INFO_KERNEL_LAUNCHES)
    call(s)
    launches = (s.info(dsx._capi.INFO_KERNEL_LAUNCHES) - l0)
    t_dsx, out = timed(lambda: call(s), iters)
    sm_clock = gpu_info("clocks.sm")
    res = dict(workload=w["name"], B=B, T=T, K=K, interval=interval, evaluations=n_eval, sm_clock_after_dsx_loop=sm_clock,
               dsx_ms_per_loop=round(t_dsx, 2), dsx_ms_per_eval=round(t_dsx / n_eval, 3),
               dsx_mel_frames_per_s=round(B * T / (t_dsx / 1e3)), dsx_launches_per_call=launches)
    if kernels:
        res["dsx_kernel_ms"] = kernel_times(lambda: call(s))

    Sd = {k: v.to(dev) for k, v in S.items()}
    sd32 = {k: v.to(dev) for k, v in sd.items()}
    sd16 = {k: v.to(dev).half() for k, v in sd.items()}
    smin3, smax3 = smin.view(1, 1, 80), smax.view(1, 1, 80)

    def half_fn(spec, t, c):
        y = D.decoder(sd16, O.decode_inp(sd32, spec, t, c, hp).half(), hp)
        return F.linear(y, sd16["get_mel_out.weight"], sd16["get_mel_out.bias"]).permute([0, 2, 1])[:, None].float()

    eager = lambda fn: O.infer_loop(fn, Sd, cond, K, smin3, smax3, fs2_mel=fs2_mel, start_noise=start, step_noise=noise,
                                    pndm_speedup=interval or None, mel2ph=mel2ph)
    ei = max(1, iters // 3)
    with torch.no_grad():
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = False, False
        t32, ref = timed(lambda: eager(lambda *a: O.forward(sd32, *a, hp)), ei)
        t16, ref16 = timed(lambda: eager(half_fn), ei)
    err = lambda a: [round((a - ref).abs().max().item(), 5), round((a - ref).abs().mean().item(), 6)]
    res.update(eager_fp32_ms_per_loop=round(t32, 1), eager_half_ms_per_loop=round(t16, 1),
               speedup_vs_eager_fp32=round(t32 / t_dsx, 2), speedup_vs_eager_half=round(t16 / t_dsx, 2),
               dsx_err_vs_eager_fp32=err(out), eager_half_err_vs_eager_fp32=err(ref16))

    torch.manual_seed(0)
    dn = dsx.DiffNet(80, hparams=dict(hidden_size=256, residual_layers=20, residual_channels=256,
                                      dilation_cycle_length=1)).to(dev).eval()
    sdn = dsx.DsxSampler(dn, None, 1)
    sdn.ensure_weights(dev)
    sdn.set_schedule(S)
    t_dn, _ = timed(lambda: call(sdn), iters)
    res.update(dsx_diffnet_ms_per_loop=round(t_dn, 2), fft_over_diffnet=round(t_dsx / t_dn, 3))
    sdn.close()
    s.close()
    del sd32, sd16, ref, ref16, out
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=6)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fft.py needs a CUDA device")
    out = dict(metric="fft_denoiser_sampling", hidden_size=256, layers=4, heads=2, ffn_kernel=9, residual_channels=256,
               gpu=gpu_info(), workloads=[run(w, a.iters, a.kernels) for w in WORKLOADS])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
