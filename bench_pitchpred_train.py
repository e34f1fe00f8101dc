"""Times one pitch predictor training step -- the predictor forward on an input that requires grad, the f0 + uv loss of
FastSpeech2's add_pitch_loss (pitch_loss 'l2', use_uv) over the non-padding frames, backward to every parameter and to
the input -- with the dsx training step (PitchPredictor under dsx_train) against eager PyTorch: fp32 with TF32 off,
PyTorch's defaults (cuDNN convolutions in TF32), TF32 everywhere, and autocast(bfloat16).  The predictor is aux_rel's
frame predictor (256 -> 256, 5 layers, k 5, SAME, odim 2, predictor_dropout 0.5).  Sizes: 16 x 1000 frames (about one
max_frames batch), 64 x 250 and 1 x 120.

The chain is bench_durpred_train.py's DiffSinger MIDI step with the pitch predictor added on the frames: MIDI embeddings
-> dsx encoder -> mel2ph gather (decoder_inp) -> the pitch predictor under predictor_grad 0.1 (fs2.py:199) with the f0 +
uv loss, plus the dsx DiffNet training step (L 20, C 256) on the same decoder_inp and its L1 -> backward through all of
it, once with the predictor on dsx and once eager (defaults), so the predictor's share of the step is measured.  Prints
one JSON line with the card, its power limit and SM clock, per-size times, peak memory above the inputs, and the tape and
workspace sizes.  --kernels adds per-kernel CUDA times from torch.profiler for the dsx step at each size.

    python bench_pitchpred_train.py [--steps 20] [--warmup 5] [--kernels]
"""
import argparse
import json
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.abspath(__file__)))
from bench_fs2dec_train import card  # noqa: E402
from bench_fs2enc_train import CHAIN, dsx_encoder, kernels, measure, set_mode, setup  # noqa: E402
from oracle import fs2enc_oracle as O  # noqa: E402
from oracle.gen_golden_pitchpred_train import random_state_dict  # noqa: E402
from oracle.pitchpred_train_oracle import pitchpred_train  # noqa: E402

CFG = (256, 5, 256, 2, 5)      # idim, n_layers, n_chans, odim, kernel_size
P = 0.5
SIZES = [(16, 1000), (64, 250), (1, 120)]
DEV = torch.device("cuda", 0)


def dsx_predictor():
    from diffsinger_b200 import PitchPredictor
    m = PitchPredictor(CFG[0], CFG[1], CFG[2], CFG[3], CFG[4], P, 'SAME', train=True)
    m.load_state_dict(random_state_dict(0, *CFG))
    return m.to(DEV).train()


def eager_predictor(mode):
    sd = {k: v.to(DEV).requires_grad_(True) for k, v in random_state_dict(0, *CFG).items()
          if k != "embed_positions._float_tensor"}

    def run(x):      # nn.Dropout's own kernel at every site, as the reference runs it
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=(mode == "bf16")):
            return pitchpred_train(sd, x, [None] * CFG[1], P, CFG[4]).float()
    return run


def inputs(B, T):
    g = torch.Generator().manual_seed(B * 1000 + T)
    x = torch.randn(B, T, CFG[0], generator=g)
    for b in range(B):
        if b % 3:
            x[b, T - T // 8 * (b % 3):] = 0
    f0 = torch.randn(B, T, generator=g)
    uv = (torch.rand(B, T, generator=g) > 0.7).float()
    return x.to(DEV).requires_grad_(True), f0.to(DEV), uv.to(DEV)


def f0_uv_loss(out, f0, uv, nonpad):
    """add_pitch_loss (fs2.py) with pitch_loss 'l2' and use_uv: the f0 MSE and the uv BCE over the non-padding frames"""
    l_f0 = (F.mse_loss(out[..., 0], f0, reduction='none') * nonpad).sum() / nonpad.sum()
    l_uv = (F.binary_cross_entropy_with_logits(out[..., 1], uv, reduction='none') * nonpad).sum() / nonpad.sum()
    return l_f0 + l_uv


def chain(pred_path, steps, warmup):
    """MIDI embeddings -> dsx encoder -> gather -> predictor (predictor_grad 0.1) and dsx DiffNet, at CHAIN tokens"""
    import diffsinger_b200 as dsx
    B, T = CHAIN
    sd, inp, emb = setup(B, T)
    tok = inp[0]
    g = torch.Generator().manual_seed(3)
    dur = torch.randint(5, 16, (B, T), generator=g).to(DEV) * (tok > 0)
    mel2ph = O.length_regulator(dur, tok == 0)
    Tm = mel2ph.shape[1]
    torch.manual_seed(0)
    net = dsx.DiffNet(80, hparams=dict(hidden_size=256, residual_layers=20, residual_channels=256,
                                       dilation_cycle_length=4), train=True).to(DEV).train()
    spec = torch.randn(B, 1, 80, Tm, generator=g).to(DEV)
    noise = torch.randn(B, 1, 80, Tm, generator=g).to(DEV)
    t = torch.randint(0, 100, (B,), generator=g).to(DEV)
    f0 = torch.randn(B, Tm, generator=g).to(DEV)
    uv = (torch.rand(B, Tm, generator=g) > 0.7).float().to(DEV)
    enc = dsx_encoder(sd)
    pred = dsx_predictor() if pred_path == "dsx" else eager_predictor("defaults")
    idx = mel2ph[..., None].repeat([1, 1, 256])
    nonpad = (mel2ph > 0).float()

    def step():
        out = enc(tok, *O.midi_addends(emb, *inp[1:]))
        dec_inp = torch.gather(F.pad(out, [0, 0, 1, 0]), 1, idx) * nonpad[:, :, None]
        pitch_inp = dec_inp.detach() + 0.1 * (dec_inp - dec_inp.detach())
        loss = f0_uv_loss(pred(pitch_inp), f0, uv, nonpad)
        ((noise - net(spec, t, dec_inp.transpose(1, 2))).abs().mean() + loss).backward()
    r = {}
    measure(r, "chain", step, steps, warmup)
    return r, Tm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    res = dict(card(), workload="PitchPredictor training step (aux_rel frame: 256 -> 256, 5 layers, k 5, odim 2, p 0.5) "
                                 "+ f0 MSE and uv BCE, backward to the parameters and the input", sizes={})
    set_mode("defaults")
    for B, T in SIZES:
        r = {}
        x, f0, uv = inputs(B, T)
        nonpad = (x.detach().abs().sum(-1) > 0).float()
        m = dsx_predictor()

        def dsx_step():
            f0_uv_loss(m(x), f0, uv, nonpad).backward()
        measure(r, "dsx", dsx_step, a.steps, a.warmup)
        st = m._dsx_train_step()
        r["dsx_tape_mib"] = st.tape_bytes(DEV, B, T) / 2 ** 20
        r["dsx_workspace_mib"] = st.workspace(DEV, B, T).numel() / 2 ** 20
        if a.kernels:
            r["dsx_kernels_ms"] = kernels(dsx_step)
        for mode in ("fp32", "defaults", "tf32", "bf16"):
            set_mode(mode)
            run = eager_predictor(mode)

            def eager_step():
                f0_uv_loss(run(x), f0, uv, nonpad).backward()
            measure(r, f"eager_{mode}", eager_step, a.steps, a.warmup)
        set_mode("defaults")
        res["sizes"][f"{B}x{T}"] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()}
    ch = {}
    for path in ("dsx", "eager"):
        r, Tm = chain(path, a.steps, a.warmup)
        ch[f"predictor_{path}_ms"] = round(r["chain_ms"], 3)
        ch[f"predictor_{path}_peak_mib"] = round(r["chain_peak_mib"], 1)
    res["chain"] = dict(ch, tokens=f"{CHAIN[0]}x{CHAIN[1]}", frames=f"{CHAIN[0]}x{Tm}",
                        what="MIDI embeddings -> dsx encoder -> mel2ph gather -> pitch predictor (predictor_grad 0.1, "
                             "f0 + uv) and dsx DiffNet training step (L 20, C 256) -> L1; the eager predictor with "
                             "PyTorch's defaults")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
