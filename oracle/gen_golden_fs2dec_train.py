"""TEST INFRASTRUCTURE ONLY -- pins oracle/fs2dec_train_oracle.py to the LIVE reference FastSpeech2 decoder in training mode
(needs a checkout of the reference: DSX_REFERENCE_ROOT) and writes tests/golden/fs2dec_train_grad.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_fs2dec_train.py

The reference's FastspeechDecoder is built as oracle/gen_golden_fs2dec.py builds it (popcs config, hidden 256, 4 layers,
2 heads, kernel 9, GELU, 'SAME'), put in training mode, and run on B = 2, T = 40 (utterance 1 padded from frame 29) with
loss = mean((out - target)^2).  Two cases, each asserted bit-exact against the oracle (output, loss, gradient of x and
of every parameter):
  p = 0          the fixture: the loss, the full d_x and, per parameter, the gradient's norm and 64 entries at seeded
                 flat indices (oracle/gen_golden_train.py's sample_index);
  p = 0.1        torch.nn.functional.dropout replaced by seeded keep masks consumed in call order (calls with p = 0, the
                 attention's, pass through): each call's p and shape are checked, so this pins the number, order and
                 placement of the oracle's dropout sites to the reference's."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import fs2dec_oracle as O  # noqa: E402
from oracle.fs2dec_train_oracle import decoder_train  # noqa: E402
from oracle.gen_golden_fs2dec import HP_KEYS, load_reference  # noqa: E402
from oracle.gen_golden_train import sample_index  # noqa: E402

SEED, INPUT_SEED, B, T, TAIL, P = 17, 18, 2, 40, 29, 0.1


def target():
    return torch.from_numpy(np.random.RandomState(INPUT_SEED + 1).standard_normal((B, T, 256)).astype(np.float32))


def seeded_masks(hp, p):
    """keep masks [B, T, n] of the 1 + 3 L sites from a fixed generator"""
    g = torch.Generator().manual_seed(INPUT_SEED + 2)
    H, L = int(hp['hidden_size']), int(hp['dec_layers'])
    return [torch.rand(B, T, 4 * H if s > 0 and s % 3 == 2 else H, generator=g) >= p for s in range(1 + 3 * L)]


def run_reference(FastspeechDecoder, hparams, sd, x, tgt, p, masks):
    hparams['dropout'] = p
    dec = FastspeechDecoder()
    dec.load_state_dict(sd, strict=True)
    dec.train()
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
        xr = x.clone().requires_grad_(True)
        out = dec(xr)
        loss = ((out - tgt) ** 2).mean()
        loss.backward()
    finally:
        torch.nn.functional.dropout = real
    assert not queue, f"{len(queue)} masks not consumed"
    return out.detach(), loss.detach(), xr.grad, {k: v.grad for k, v in dec.named_parameters()}


def run_oracle(sd, x, tgt, hp, p, masks):
    P_ = {k: v.clone().requires_grad_(True) for k, v in sd.items() if k != "embed_positions._float_tensor"}
    xr = x.clone().requires_grad_(True)
    out = decoder_train(P_, xr, hp, masks, p)
    loss = ((out - tgt) ** 2).mean()
    loss.backward()
    return out.detach(), loss.detach(), xr.grad, {k: v.grad for k, v in P_.items()}


def main():
    assert os.environ.get("DSX_REFERENCE_ROOT"), "set DSX_REFERENCE_ROOT to a checkout of the reference"
    hparams, FastspeechDecoder = load_reference()
    hp = {k: hparams[k] for k in HP_KEYS}
    sd = O.random_state_dict(SEED, hp)
    x = O.fixture_input(INPUT_SEED, B, T, hp["hidden_size"], tail=TAIL)
    tgt = target()
    results = {}
    for p in (0.0, P):
        hpp = dict(hp, dropout=p)
        masks = seeded_masks(hp, p)
        ref = run_reference(FastspeechDecoder, hparams, sd, x, tgt, p, masks if p > 0 else [])
        mine = run_oracle(sd, x, tgt, hpp, p, masks)
        for name, a, b in (("out", mine[0], ref[0]), ("loss", mine[1], ref[1]), ("d_x", mine[2], ref[2])):
            assert torch.equal(a, b), (p, name, (a - b).abs().max().item())
        for k in ref[3]:
            assert torch.equal(mine[3][k], ref[3][k]), (p, k, (mine[3][k] - ref[3][k]).abs().max().item())
        print(f"p = {p}: oracle bit-exact to the reference (loss {ref[1].item():.6f})")
        results[p] = ref

    _, loss, d_x, grads = results[0.0]
    out = dict(seed=SEED, input_seed=INPUT_SEED, B=B, T=T, tail=TAIL, loss=loss.numpy(), d_x=d_x.numpy())
    out.update({"hp." + k: np.asarray(v) for k, v in hp.items() if k != "dropout"})
    for k, g in grads.items():
        flat = g.reshape(-1)
        out["norm." + k] = flat.norm().numpy()
        out["val." + k] = flat[torch.from_numpy(sample_index(k, flat.numel())).long()].numpy()
    path = os.path.join(ROOT, "tests", "golden", "fs2dec_train_grad.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
