"""Latency of the FastSpeech2 encoder and duration path on one GPU: txt_tokens (+ MIDI inputs) -> encoder_out ->
durations -> mel2ph.

    python bench_fs2enc.py [--iters N] [--kernels]

The model is the MIDI front end of usr/configs/midi/e2e/opencpop/ds100_adj_rel.yaml (hidden 256, 4 encoder layers,
2 heads, FFN kernel 9, relative positions, a 5-layer duration predictor with k = 3) with seeded weights
(oracle.fs2enc_oracle.random_state_dict) whose duration bias gives about 10 frames per token.  Two sizes: B = 1,
T_txt = 120 (one opencpop phrase) and B = 16, T_txt = 400 (a batch; every other utterance has a padded tail).  The MIDI
embeddings are computed once outside the timed region (they stay eager in FastSpeech2MIDI.forward).  Times come from
CUDA events around the whole chain -- encoder, masking, duration predictor, length regulator -- and around each stage,
after a warm-up call.  Baselines in the same process: the oracle chain (the ATen ops the reference runs) in PyTorch
eager -- fp32 with TF32 off, fp32 with cuDNN's defaults, and `.half()` for the encoder and duration predictor.  Memory:
the peak of torch.cuda.max_memory_allocated above what was allocated before, for the eager length regulator (its
[B, T_txt, T_mel] temporaries) and dsx's.  Errors of encoder_out and xs are against eager fp32; mel2ph is compared
exactly.  --kernels adds the summed device time per kernel name of one dsx chain (torch.profiler).  The card's name,
power limit and max SM clock are read once; the SM clock again after each dsx loop.  Prints one JSON line; writes
nothing.
"""
import argparse
import json

import torch

import diffsinger_b200 as dsx
from bench_pe import gpu_info, kernel_times, timed
from oracle import fs2enc_oracle as O

SIZES = ((1, 120), (16, 400))
VOCAB = 61


def eager_chain(sd, tok, add, hp, half=False):
    c = (lambda t: t.half()) if half else (lambda t: t)
    sdc = {k: c(v) for k, v in sd.items()}
    enc = O.encoder(O.sub(sdc, "encoder."), tok, hp, tuple(c(a) for a in add))
    keep = (tok > 0).to(enc.dtype)[:, :, None]
    xs = O.dur_predictor(O.sub(sdc, "dur_predictor."), enc * keep, tok == 0, hp)
    dur = O.out2dur(xs.float())
    return enc.float(), xs.float(), O.length_regulator(dur, tok == 0)


def peak_mib(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 2), out


def run_size(B, T, iters, kernels):
    dev = torch.device("cuda", 0)
    hp = dict(O.HPARAMS_MIDI)
    H = hp["hidden_size"]
    sd = {k: v.to(dev) for k, v in O.random_state_dict(1, hp, VOCAB, frames_per_token=10.0).items()}
    tails = [None if b % 2 == 0 else T - T // 5 for b in range(B)]
    tok, midi, mdur, slur = (t.to(dev) for t in O.fixture_inputs(2, B, T, tails, VOCAB))
    enc = dsx.FastspeechMIDIEncoder(torch.nn.Embedding(VOCAB, H, 0), H, hp["enc_layers"], hp["enc_ffn_kernel_size"],
                                    num_heads=hp["num_heads"], hparams=hp)
    enc.load_state_dict({k: v.cpu() for k, v in O.sub(sd, "encoder.").items()}, strict=True)
    dp = dsx.DurationPredictor(H, n_chans=O.predictor_hidden(hp), n_layers=hp["dur_predictor_layers"],
                               padding=hp["ffn_padding"], kernel_size=hp["dur_predictor_kernel"], hparams=hp)
    dp.load_state_dict({k: v.cpu() for k, v in O.sub(sd, "dur_predictor.").items()}, strict=True)
    enc, dp, lr = enc.eval().to(dev), dp.eval().to(dev), dsx.LengthRegulator()
    pad = tok == 0
    keep = (~pad).float()[:, :, None]
    with torch.no_grad():
        add = O.midi_addends(sd, midi, mdur, slur)

        def chain():
            out = enc(tok, *add)
            dur, xs = dp.inference(out * keep, pad)
            return out, xs, lr(dur, pad)

        t_dsx, (out, xs, mel2ph) = timed(chain, iters)
        sm_clock = gpu_info("clocks.sm")
        t_enc, out = timed(lambda: enc(tok, *add), iters)
        x = out * keep
        t_dp, (dur, _) = timed(lambda: dp.inference(x, pad), iters)
        t_lr, _ = timed(lambda: lr(dur, pad), iters)
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = False, False
        t32, (ref_enc, ref_xs, ref_m) = timed(lambda: eager_chain(sd, tok, add, hp), iters)
        torch.backends.cudnn.allow_tf32 = True
        t_tf32, (tf_enc, _, _) = timed(lambda: eager_chain(sd, tok, add, hp), iters)
        t16, (h_enc, h_xs, h_m) = timed(lambda: eager_chain(sd, tok, add, hp, half=True), iters)
        torch.backends.cudnn.allow_tf32 = False
        d_ref = O.out2dur(ref_xs)
        mem_eager, _ = peak_mib(lambda: O.length_regulator(d_ref, pad))
        mem_dsx, _ = peak_mib(lambda: lr(d_ref, pad))
    err = lambda a, r: [round((a - r).abs().max().item(), 6), round((a - r).abs().mean().item(), 7)]
    res = dict(B=B, T_txt=T, T_mel=int(mel2ph.shape[1]), sm_clock_after_dsx_loop=sm_clock, dsx_chain_ms=round(t_dsx, 3),
               dsx_encoder_ms=round(t_enc, 3), dsx_duration_predictor_ms=round(t_dp, 3),
               dsx_length_regulator_ms=round(t_lr, 3), eager_fp32_chain_ms=round(t32, 3),
               eager_cudnn_default_chain_ms=round(t_tf32, 3), eager_fp16_chain_ms=round(t16, 3),
               speedup_vs_eager_fp32=round(t32 / t_dsx, 2), speedup_vs_eager_cudnn_default=round(t_tf32 / t_dsx, 2),
               speedup_vs_eager_fp16=round(t16 / t_dsx, 2),
               length_regulator_peak_mib=dict(eager=mem_eager, dsx=mem_dsx),
               dsx_encoder_err_vs_fp32=err(out, ref_enc), dsx_xs_err_vs_fp32=err(xs.squeeze(-1), ref_xs.squeeze(-1)),
               dsx_mel2ph_equal_to_fp32=bool(torch.equal(mel2ph, ref_m)),
               cudnn_default_encoder_err_vs_fp32=err(tf_enc, ref_enc), fp16_encoder_err_vs_fp32=err(h_enc, ref_enc),
               fp16_mel2ph_equal_to_fp32=bool(torch.equal(h_m, ref_m)))
    if kernels:
        with torch.no_grad():
            res["dsx_kernel_ms"] = kernel_times(chain)
    enc.close()
    dp.close()
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fs2enc.py needs a CUDA device")
    out = dict(metric="fastspeech2_encoder_duration_path", hidden_size=256, enc_layers=4, heads=2, ffn_kernel=9,
               dur_predictor_layers=5, gpu=gpu_info(), sizes=[run_size(B, T, a.iters, a.kernels) for B, T in SIZES])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
