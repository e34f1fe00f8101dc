"""Times one duration predictor training step -- the predictor forward on an input that requires grad, the masked pdur
MSE of DiffSinger's add_dur_loss (dur_loss 'mse'), backward to every parameter and to the input -- with the dsx training
step (DurationPredictor under dsx_train) against eager PyTorch: fp32 with TF32 off, PyTorch's defaults (cuDNN
convolutions in TF32), TF32 everywhere, and autocast(bfloat16).  The predictor is ds100_adj_rel's (256 -> 256, 5 layers,
k 3, SAME, predictor_dropout 0.5).  Sizes: 16 x 250 tokens (about one max_tokens: 40000 batch), 64 x 60 and 1 x 120.

The chain is bench_fs2enc_train.py's DiffSinger MIDI step at 16 x 100 tokens with the predictor added: MIDI embeddings ->
dsx encoder -> the predictor on (encoder_out * nonpadding) under predictor_grad 0.1 (fs2.py:161) with the pdur + wdur +
sdur losses (a word is two tokens here), plus the mel2ph gather into the dsx DiffNet training step (L 20, C 256) and its
L1 -> backward through all of it, once with the predictor on dsx and once eager (defaults), so the predictor's share of
the step is measured.  Prints one JSON line with the card, its power limit and SM clock, per-size times, peak memory
above the inputs, and the tape and workspace sizes.  --kernels adds per-kernel CUDA times from torch.profiler for the
dsx step at each size.

    python bench_durpred_train.py [--steps 20] [--warmup 5] [--kernels]
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
from oracle.durpred_train_oracle import durpred_train  # noqa: E402
from oracle.gen_golden_durpred_train import random_state_dict  # noqa: E402

CFG = (256, 5, 256, 3)      # idim, n_layers, n_chans, kernel_size
P = 0.5
SIZES = [(16, 250), (64, 60), (1, 120)]
DEV = torch.device("cuda", 0)


def dsx_predictor():
    from diffsinger_b200 import DurationPredictor
    m = DurationPredictor(CFG[0], CFG[1], CFG[2], CFG[3], P, hparams=dict(dur_loss='mse'), train=True)
    m.load_state_dict(random_state_dict(0, *CFG))
    return m.to(DEV).train()


def eager_predictor(mode):
    sd = {k: v.to(DEV).requires_grad_(True) for k, v in random_state_dict(0, *CFG).items()}

    def run(x, mask):      # nn.Dropout's own kernel at every site, as the reference runs it
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=(mode == "bf16")):
            return durpred_train(sd, x, mask, [None] * CFG[1], P, CFG[3]).float()
    return run


def inputs(B, T):
    g = torch.Generator().manual_seed(B * 1000 + T)
    x = torch.randn(B, T, CFG[0], generator=g).to(DEV).requires_grad_(True)
    mask = torch.zeros(B, T, dtype=torch.bool)
    for b in range(B):
        if b % 3:
            mask[b, T - T // 8 * (b % 3):] = True
    dur = torch.randint(1, 20, (B, T), generator=g).to(DEV)
    return x, mask.to(DEV), dur


def pdur(xs, dur, mask):
    """add_dur_loss's pdur (dur_loss 'mse'): MSE of xs against log(dur + 1) over the non-padding tokens"""
    nonpad = (~mask).float()
    return (F.mse_loss(xs, torch.log(dur.float() + 1), reduction='none') * nonpad).sum() / nonpad.sum()


def dur_losses(xs, dur, tok):
    """pdur + wdur + sdur of add_dur_loss with words of two tokens (ph2word = (t // 2) + 1 on real tokens)"""
    mask = tok == 0
    B, T = tok.shape
    nonpad = (~mask).float()
    loss = pdur(xs, dur, mask)
    d_pred = (xs.exp() - 1).clamp(min=0) * nonpad
    ph2word = ((torch.arange(T, device=DEV) // 2 + 1)[None, :] * (~mask).long())
    nw = T // 2 + 2
    w_pred = d_pred.new_zeros(B, nw).scatter_add(1, ph2word, d_pred)[:, 1:]
    w_gt = d_pred.new_zeros(B, nw).scatter_add(1, ph2word, dur.float() * nonpad)[:, 1:]
    wn = (w_gt > 0).float()
    loss = loss + (F.mse_loss(torch.log(w_pred + 1), torch.log(w_gt + 1), reduction='none') * wn).sum() / wn.sum()
    s_pred, s_gt = d_pred.sum(-1), (dur.float() * nonpad).sum(-1)
    return loss + F.mse_loss(torch.log(s_pred + 1), torch.log(s_gt + 1))


def chain(pred_path, steps, warmup):
    """MIDI embeddings -> dsx encoder -> predictor (predictor_grad 0.1) + gather -> dsx DiffNet, at CHAIN tokens"""
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
    enc = dsx_encoder(sd)
    pred = dsx_predictor() if pred_path == "dsx" else None
    eager = eager_predictor("defaults")
    idx = mel2ph[..., None].repeat([1, 1, 256])
    nonpad = (mel2ph > 0).float()[:, :, None]
    src_pad = tok == 0

    def step():
        out = enc(tok, *O.midi_addends(emb, *inp[1:]))
        dur_inp = out * (~src_pad).float()[:, :, None]
        dur_inp = dur_inp.detach() + 0.1 * (dur_inp - dur_inp.detach())
        xs = pred(dur_inp, src_pad) if pred is not None else eager(dur_inp, src_pad)
        cond = (torch.gather(F.pad(out, [0, 0, 1, 0]), 1, idx) * nonpad).transpose(1, 2)
        ((noise - net(spec, t, cond)).abs().mean() + dur_losses(xs, dur, tok)).backward()
    r = {}
    measure(r, "chain", step, steps, warmup)
    return r, Tm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    res = dict(card(), workload="DurationPredictor training step (ds100_adj_rel: 256 -> 256, 5 layers, k 3, p 0.5) + "
                                 "masked pdur MSE, backward to the parameters and the input", sizes={})
    set_mode("defaults")
    for B, T in SIZES:
        r = {}
        x, mask, dur = inputs(B, T)
        m = dsx_predictor()

        def dsx_step():
            pdur(m(x, mask), dur, mask).backward()
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
                pdur(run(x, mask), dur, mask).backward()
            measure(r, f"eager_{mode}", eager_step, a.steps, a.warmup)
        set_mode("defaults")
        res["sizes"][f"{B}x{T}"] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()}
    ch = {}
    for path in ("dsx", "eager"):
        r, Tm = chain(path, a.steps, a.warmup)
        ch[f"predictor_{path}_ms"] = round(r["chain_ms"], 3)
        ch[f"predictor_{path}_peak_mib"] = round(r["chain_peak_mib"], 1)
    res["chain"] = dict(ch, tokens=f"{CHAIN[0]}x{CHAIN[1]}", frames=f"{CHAIN[0]}x{Tm}",
                        what="MIDI embeddings -> dsx encoder -> predictor (predictor_grad 0.1, pdur + wdur + sdur) + "
                             "mel2ph gather -> dsx DiffNet training step (L 20, C 256) -> L1; the eager predictor with "
                             "PyTorch's defaults")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
