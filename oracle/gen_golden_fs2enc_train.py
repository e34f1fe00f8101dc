"""TEST INFRASTRUCTURE ONLY -- pins oracle/fs2enc_train_oracle.py to the LIVE reference FastSpeech2 encoders in training
mode (needs a checkout of the reference: DSX_REFERENCE_ROOT; runs on a CPU) and writes tests/golden/fs2enc_train_grad.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_fs2enc_train.py

The reference modules are loaded as oracle/gen_golden_fs2enc.py loads them (stubs for librosa / pycwt) and built with
oracle.fs2enc_oracle.random_state_dict(SEED) on B = 2, T = 40 tokens (utterance 1 padded from token 29,
oracle.fs2enc_oracle.fixture_inputs), with loss = mean((out - target)^2).  Two encoders:
  midi   FastspeechMIDIEncoder under usr/configs/midi/e2e/opencpop/ds100_adj_rel.yaml (rel_pos, all three addends, which
         are leaves here, so their common gradient d_add is the reference's own);
  sin    FastspeechEncoder under usr/configs/popcs_ds_beta6.yaml (sinusoidal positions).
Each at p = 0 and at p = 0.1 with torch.nn.functional.dropout replaced by seeded keep masks consumed in call order (calls
with p = 0 -- the attention's and RelPositionalEncoding's own -- pass through; each call's p and shape are checked), so
the number, order and placement of the oracle's dropout sites are pinned to the reference's.  The oracle must give the
same bits: output, loss, d_add and every gradient.  Stored per encoder and p: the loss and, per gradient and d_add, its
norm and 64 entries at seeded flat indices (oracle/gen_golden_train.py's sample_index); at p = 0 d_add and the
embed_tokens gradient in full instead."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import fs2enc_oracle as O  # noqa: E402
from oracle.fs2enc_train_oracle import encoder_train  # noqa: E402
from oracle.gen_golden_fs2enc import MIDI_CONFIG, POPCS_CONFIG, load_reference  # noqa: E402
from oracle.gen_golden_train import sample_index  # noqa: E402

SEED, INPUT_SEED, VOCAB, B, T, TAILS, P = 41, 42, 61, 2, 40, (None, 29), 0.1
CASES = (("midi", MIDI_CONFIG, O.HPARAMS_MIDI), ("sin", POPCS_CONFIG, O.HPARAMS_POPCS))


def target(H):
    return torch.from_numpy(np.random.RandomState(INPUT_SEED + 1).standard_normal((B, T, H)).astype(np.float32))


def seeded_masks(hp, p):
    """keep masks [B, T, n] of the 1 + 3 L sites from a fixed generator"""
    g = torch.Generator().manual_seed(INPUT_SEED + 2)
    H, L = int(hp['hidden_size']), int(hp['enc_layers'])
    return [torch.rand(B, T, 4 * H if s > 0 and s % 3 == 2 else H, generator=g) >= p for s in range(1 + 3 * L)]


def inputs(case, sd_full):
    """tokens and, for the MIDI encoder, the three addends (from the model's own embedding weights)"""
    tok, midi, mdur, slur = O.fixture_inputs(INPUT_SEED, B, T, TAILS, VOCAB)
    if case != "midi":
        return tok, ()
    with torch.no_grad():
        return tok, tuple(a.clone() for a in O.midi_addends(sd_full, midi, mdur, slur))


def encoder_sd(case, hp):
    sd_full = O.random_state_dict(SEED, hp, VOCAB, midi=case == "midi")
    return sd_full, O.sub(sd_full, "encoder.")


def run_reference(case, hparams, hp, enc_sd, tok, adds, tgt, p, masks):
    hparams['dropout'] = p
    H = hp['hidden_size']
    if case == "midi":
        from modules.diffsinger_midi.fs2 import FastspeechMIDIEncoder as Enc
    else:
        from modules.fastspeech.tts_modules import FastspeechEncoder as Enc
    enc = Enc(torch.nn.Embedding(VOCAB, H, 0), H, hp['enc_layers'], hp['enc_ffn_kernel_size'], num_heads=hp['num_heads'])
    enc.load_state_dict(enc_sd, strict=True)
    enc.train()
    real = torch.nn.functional.dropout
    queue = list(masks)

    def fake(v, p=0.5, training=True, inplace=False):
        if not training or p == 0:
            return real(v, p, training, inplace)
        assert p == P and queue, (p, len(queue))
        m = queue.pop(0)
        if tuple(v.shape) != tuple(m.shape):          # the layers run [T, B, C]
            m = m.transpose(0, 1)
        assert tuple(v.shape) == tuple(m.shape), (v.shape, m.shape)
        return v * m.to(v.dtype).div_(1 - p)

    torch.nn.functional.dropout = fake
    try:
        ar = [a.clone().requires_grad_(True) for a in adds]
        out = enc(tok, *ar)
        loss = ((out - tgt) ** 2).mean()
        loss.backward()
    finally:
        torch.nn.functional.dropout = real
    assert not queue, f"{len(queue)} masks not consumed"
    if ar:
        assert all(torch.equal(a.grad, ar[0].grad) for a in ar)
    return out.detach(), loss.detach(), ar[0].grad if ar else None, {k: v.grad for k, v in enc.named_parameters()}


def run_oracle(hp, enc_sd, tok, adds, tgt, p, masks):
    """-> out, loss, d_add (or None), {name: gradient}"""
    P_ = {k: v.clone().requires_grad_(True) for k, v in enc_sd.items() if not k.endswith("_float_tensor")}
    ar = [a.clone().requires_grad_(True) for a in adds]
    out = encoder_train(P_, tok, dict(hp, dropout=p), masks, p, tuple(ar))
    loss = ((out - tgt) ** 2).mean()
    loss.backward()
    return out.detach(), loss.detach(), ar[0].grad if ar else None, {k: v.grad for k, v in P_.items()}


def case_inputs(case, hp):
    sd_full, enc_sd = encoder_sd(case, hp)
    tok, adds = inputs(case, sd_full)
    return enc_sd, tok, adds, target(hp['hidden_size'])


def main():
    assert os.environ.get("DSX_REFERENCE_ROOT"), "set DSX_REFERENCE_ROOT to a checkout of the reference"
    hparams, configure = load_reference()
    out = dict(seed=SEED, input_seed=INPUT_SEED, vocab=VOCAB, B=B, T=T, tail=TAILS[1], p=P)
    for case, config, hp0 in CASES:
        hp = configure(config)
        assert hp == hp0, hp
        enc_sd, tok, adds, tgt = case_inputs(case, hp)
        for p in (0.0, P):
            masks = seeded_masks(hp, p)
            ref = run_reference(case, hparams, hp, enc_sd, tok, adds, tgt, p, masks if p > 0 else [])
            mine = run_oracle(hp, enc_sd, tok, adds, tgt, p, masks)
            for name, a, b in (("out", mine[0], ref[0]), ("loss", mine[1], ref[1]), ("d_add", mine[2], ref[2])):
                assert (a is None and b is None) or torch.equal(a, b), (case, p, name, (a - b).abs().max().item())
            assert set(mine[3]) == set(ref[3]), (set(mine[3]) ^ set(ref[3]))
            for k in ref[3]:
                assert torch.equal(mine[3][k], ref[3][k]), (case, p, k, (mine[3][k] - ref[3][k]).abs().max().item())
            print(f"{case} p = {p}: oracle bit-exact to the reference (loss {ref[1].item():.6f})")
            pre = f"{case}.p{int(round(p * 10))}."
            _, loss, d_add, grads = ref
            out[pre + "loss"] = loss.numpy()
            full = {"embed_tokens.weight": grads["embed_tokens.weight"]}
            if d_add is not None:
                full["d_add"] = d_add
            for k, g in dict(grads, **full).items():
                flat = g.reshape(-1)
                if p == 0 and k in full:
                    out[pre + "grad." + k] = g.numpy()
                    continue
                out[pre + "norm." + k] = flat.norm().numpy()
                out[pre + "val." + k] = flat[torch.from_numpy(sample_index(k, flat.numel())).long()].numpy()
        out.update({f"hp.{case}." + k: np.asarray(v) for k, v in hp.items()})
    path = os.path.join(ROOT, "tests", "golden", "fs2enc_train_grad.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
