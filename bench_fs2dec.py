"""Throughput of the FastSpeech2 decoder on one GPU: mel frames per second at the shipped singing size.

    python bench_fs2dec.py [--iters N] [--kernels]

The model is popcs_ds_beta6's decoder (hidden 256, 4 layers, 2 heads, FFN conv kernel 9 and width 1024, GELU, 'SAME')
with seeded weights (oracle.fs2dec_oracle.random_state_dict).  Two sizes: B = 16, T = 1024 (a batch; the second
utterance has a zero-padded tail) and B = 1, T = 4000 (one long sung phrase, where the T^2 attention dominates).  Times
come from CUDA events around whole calls after a warm-up call.  Baselines in the same process: the reference's decoder
(oracle/fs2dec_oracle.py, the ATen ops the reference runs, with the [B * heads, T, T] weights that
F.multi_head_attention_forward materialises) in PyTorch eager -- fp32 with TF32 off, fp32 with cuDNN's defaults (TF32
convolutions), and `.half()`.  Errors are against the eager fp32 TF32-off output.  Share of peak is the FLOP floor
(flops_per_frame at 989 TFLOP/s, the H100 SXM data-sheet dense FP16 rate) over the measured time.  --kernels adds the
summed device time per kernel name of one dsx call (torch.profiler).  The card's name, power limit and max SM clock are
read once; the SM clock again right after each dsx loop.  Prints one JSON line; writes nothing.
"""
import argparse
import json

import torch

import diffsinger_b200 as dsx
from bench_pe import gpu_info, kernel_times, timed
from oracle import fs2dec_oracle as O

PEAK_FLOPS = 989e12
SIZES = ((16, 1024), (1, 4000))


def sampler_k51_ms(B, T, iters):
    from oracle import diffnet_oracle as D
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = dsx.DiffNet(80, hparams=dict(hidden_size=256, residual_layers=20, residual_channels=256,
                                       dilation_cycle_length=1)).to(dev).eval()
    s = dsx.DsxSampler(net, None, 1)
    s.ensure_weights(dev)
    s.set_schedule(D.make_schedule(D.linear_beta_schedule(100, 0.06)))
    g = torch.Generator().manual_seed(3)
    cond = torch.randn(B, T, 256, generator=g).to(dev).transpose(1, 2)
    x = torch.randn(B, 1, 80, T, generator=g).to(dev)
    ms, _ = timed(lambda: s.sample_ddpm(x, cond, 51, 51), max(1, iters // 4))
    s.close()
    return ms


def run_size(B, T, iters, kernels):
    dev = torch.device("cuda", 0)
    hp = dict(O.HPARAMS_POPCS)
    sd = O.random_state_dict(1, hp)
    dec = dsx.FastspeechDecoder(hparams=hp)
    dec.load_state_dict(sd, strict=True)
    dec = dec.eval().to(dev)
    x = O.fixture_input(2, B, T, hp["hidden_size"], tail=T - T // 4 if B > 1 else None).to(dev)
    with torch.no_grad():
        t_dsx, out = timed(lambda: dec(x), iters)
        sm_clock = gpu_info("clocks.sm")      # read right after the timed loop, while the clock is still under load
        sd32 = {k: v.to(dev) for k, v in sd.items()}
        sd16 = {k: v.to(dev).half() for k, v in sd.items()}
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = False, False
        t32, ref = timed(lambda: O.decoder(sd32, x, hp), iters)
        torch.backends.cudnn.allow_tf32 = True                 # cuDNN's default: TF32 convolutions
        t_tf32, ref_tf32 = timed(lambda: O.decoder(sd32, x, hp), iters)
        t16, ref16 = timed(lambda: O.decoder(sd16, x.half(), hp), iters)
        torch.backends.cudnn.allow_tf32 = False
    err = lambda a: [round((a.float() - ref).abs().max().item(), 5), round((a.float() - ref).abs().mean().item(), 6)]
    fps = lambda ms: round(B * T / (ms / 1e3))
    fpf = O.flops_per_frame(T=T)
    res = dict(B=B, T=T, sm_clock_after_dsx_loop=sm_clock, dsx_ms=round(t_dsx, 3), eager_fp32_ms=round(t32, 3),
               eager_cudnn_default_ms=round(t_tf32, 3), eager_fp16_ms=round(t16, 3), mel_frames_per_s=fps(t_dsx),
               eager_fp32_frames_per_s=fps(t32), speedup_vs_eager_fp32=round(t32 / t_dsx, 2),
               speedup_vs_eager_cudnn_default=round(t_tf32 / t_dsx, 2), speedup_vs_eager_fp16=round(t16 / t_dsx, 2),
               flops_per_frame=fpf, floor_ms=round(fpf * B * T / PEAK_FLOPS * 1e3, 4),
               share_of_fp16_peak=round(fpf * B * T / PEAK_FLOPS / (t_dsx / 1e3), 4),
               dsx_err_vs_fp32=err(out), cudnn_default_err_vs_fp32=err(ref_tf32), fp16_err_vs_fp32=err(ref16))
    # what the decoder costs inside a K = 51 shallow-diffusion call (popcs_ds_beta6: 100 steps, K_step 51) whose
    # sampler runs on dsx: the sampler's 51 DDPM steps at the same (B, T), default precision, in-kernel noise
    t_k51 = sampler_k51_ms(B, T, iters)
    res.update(dsx_sampler_k51_ms=round(t_k51, 3),
               eager_fp32_decoder_share_of_k51_call=round(t32 / (t32 + t_k51), 4),
               dsx_decoder_share_of_k51_call=round(t_dsx / (t_dsx + t_k51), 4))
    if kernels:
        with torch.no_grad():
            res["dsx_kernel_ms"] = kernel_times(lambda: dec(x))
    dec.close()
    del sd32, sd16, ref, ref_tf32, ref16, out
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fs2dec.py needs a CUDA device")
    out = dict(metric="fastspeech2_decoder", hidden_size=256, layers=4, heads=2, ffn_kernel=9, gpu=gpu_info(),
               sizes=[run_size(B, T, a.iters, a.kernels) for B, T in SIZES])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
