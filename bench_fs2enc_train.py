"""Times one FastSpeech2 encoder training step -- the MIDI embeddings (eager), the encoder forward, an L1 loss on
encoder_out, backward -- with the dsx training step (FastspeechMIDIEncoder under dsx_train) against eager PyTorch: fp32
with TF32 off, PyTorch's defaults (cuDNN convolutions in TF32, matmuls in fp32), TF32 everywhere, and autocast(bfloat16).
The encoder is ds100_adj_rel's (H 256, 4 layers, 2 heads, k 9, rel_pos, the three MIDI addends, dropout 0.1, 61 phoneme
ids).  Sizes: 16 x 250 tokens (about one max_tokens: 40000 batch), 64 x 60 and 1 x 120.

The headline is a chain step of DiffSinger MIDI training at 16 x 100 tokens, about 10 frames per token: MIDI embeddings
-> encoder -> mel2ph gather -> the dsx DiffNet training step (L 20, C 256) -> L1 against the noise -> backward through
all of it, once with the encoder on dsx and once in eager PyTorch (defaults), so the encoder's share of the step is
measured.  Prints one JSON line with the card, its power limit and SM clock, per-size times and peak memory above the
inputs.  --kernels adds per-kernel CUDA times from torch.profiler for the dsx encoder step at each size.

    python bench_fs2enc_train.py [--steps 10] [--warmup 3] [--kernels]
"""
import argparse
import json
import re
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.abspath(__file__)))
from bench_fs2dec_train import card, time_step  # noqa: E402
from oracle import fs2enc_oracle as O  # noqa: E402
from oracle.fs2enc_train_oracle import encoder_train  # noqa: E402

HP = dict(O.HPARAMS_MIDI)
VOCAB = 61
SIZES = [(16, 250), (64, 60), (1, 120)]
CHAIN = (16, 100)
DEV = torch.device("cuda", 0)
EMB = ("midi_embed.weight", "midi_dur_layer.weight", "midi_dur_layer.bias", "is_slur_embed.weight")


def setup(B, T):
    """state dict on the GPU (encoder parameters and MIDI embeddings as leaves), inputs and a target"""
    sd = {k: v.to(DEV) for k, v in O.random_state_dict(0, HP, VOCAB).items()}
    tails = tuple(T - T // 8 * (b % 3) if b % 3 else None for b in range(B))
    tok, midi, mdur, slur = (t.to(DEV) for t in O.fixture_inputs(1, B, T, tails, VOCAB))
    emb = {k: sd[k].clone().requires_grad_(True) for k in EMB}
    return sd, (tok, midi, mdur, slur), emb


def dsx_encoder(sd):
    from diffsinger_b200 import FastspeechMIDIEncoder
    m = FastspeechMIDIEncoder(torch.nn.Embedding(VOCAB, 256, 0), 256, HP['enc_layers'], HP['enc_ffn_kernel_size'],
                              num_heads=HP['num_heads'], hparams=dict(HP, dsx_train=True))
    m.load_state_dict(O.sub(sd, "encoder."), strict=True)
    return m.to(DEV).train()


def eager_encoder(sd, B, T, mode):
    esd = {k: v.clone().requires_grad_(True) for k, v in O.sub(sd, "encoder.").items()}
    p = HP['dropout']

    def run(tok, adds):
        masks = [torch.rand(B, T, 4 * 256 if s > 0 and s % 3 == 2 else 256, device=DEV) >= p
                 for s in range(1 + 3 * HP['enc_layers'])]
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=(mode == "bf16")):
            return encoder_train(esd, tok, HP, masks, p, adds)
    return run


def enc_step(run, inp, emb, y):
    tok, midi, mdur, slur = inp

    def step():
        out = run(tok, O.midi_addends(emb, midi, mdur, slur))
        (out - y).abs().mean().backward()
    return step


def set_mode(mode):
    torch.backends.cuda.matmul.allow_tf32 = mode in ("tf32", "bf16")
    torch.backends.cudnn.allow_tf32 = mode != "fp32"


def measure(r, key, step, steps, warmup):
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    r[key + "_ms"] = time_step(step, steps, warmup)
    r[key + "_peak_mib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20


def kernels(step):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    agg = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            k = re.sub(r"^void |\(anonymous namespace\)::|dsx::|<.*$|\(.*$", "", e.name)
            agg[k] = agg.get(k, 0.0) + e.device_time / 1e3
    return dict(sorted(((k, round(v, 4)) for k, v in agg.items()), key=lambda kv: -kv[1])[:25])


def chain_case(enc_path, steps, warmup):
    """the DiffSinger MIDI training chain at CHAIN tokens: ms per step and peak memory"""
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
    run = dsx_encoder(sd) if enc_path == "dsx" else eager_encoder(sd, B, T, "defaults")
    idx = mel2ph[..., None].repeat([1, 1, 256])
    nonpad = (mel2ph > 0).float()[:, :, None]

    def step():
        out = run(tok, *O.midi_addends(emb, *inp[1:])) if enc_path == "dsx" else \
            run(tok, O.midi_addends(emb, *inp[1:]))
        cond = (torch.gather(F.pad(out, [0, 0, 1, 0]), 1, idx) * nonpad).transpose(1, 2)
        (noise - net(spec, t, cond)).abs().mean().backward()
    r = {}
    measure(r, "chain", step, steps, warmup)
    return r, Tm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--kernels", action="store_true")
    a = ap.parse_args()
    res = dict(card(), workload="FastSpeech2 MIDI encoder training step (ds100_adj_rel: H 256, L 4, heads 2, k 9, "
                                 "rel_pos, 3 MIDI addends, p 0.1) + L1 on encoder_out", sizes={})
    set_mode("defaults")
    for B, T in SIZES:
        r = {}
        sd, inp, emb = setup(B, T)
        y = torch.randn(B, T, 256, device=DEV)
        m = dsx_encoder(sd)
        step = enc_step(lambda tok, adds: m(tok, *adds), inp, emb, y)
        measure(r, "dsx", step, a.steps, a.warmup)
        st = m._dsx_train_step()
        r["dsx_tape_mib"] = st.tape_bytes(DEV, B, T) / 2 ** 20
        r["dsx_workspace_mib"] = st.workspace(DEV, B, T).numel() / 2 ** 20
        if a.kernels:
            r["dsx_kernels_ms"] = kernels(step)
        del step, m
        for mode in ("fp32", "defaults", "tf32", "bf16"):
            set_mode(mode)
            measure(r, f"eager_{mode}", enc_step(eager_encoder(sd, B, T, mode), inp, emb, y), a.steps, a.warmup)
        set_mode("defaults")
        res["sizes"][f"{B}x{T}"] = {k: (round(v, 3) if isinstance(v, float) else v) for k, v in r.items()}
    chain = {}
    for path in ("dsx", "eager"):
        r, Tm = chain_case(path, a.steps, a.warmup)
        chain[f"encoder_{path}_ms"] = round(r["chain_ms"], 3)
        chain[f"encoder_{path}_peak_mib"] = round(r["chain_peak_mib"], 1)
    chain["frames"] = f"{CHAIN[0]}x{Tm}"
    res["chain"] = dict(chain, tokens=f"{CHAIN[0]}x{CHAIN[1]}", what="MIDI embeddings -> encoder -> mel2ph gather -> "
                        "dsx DiffNet training step (L 20, C 256) -> L1; the eager encoder with PyTorch's defaults")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
