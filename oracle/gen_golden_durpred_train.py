"""TEST INFRASTRUCTURE ONLY -- pins oracle/durpred_train_oracle.py to the LIVE reference DurationPredictor in training mode
(needs a checkout of the reference: DSX_REFERENCE_ROOT; runs on a CPU) and writes tests/golden/durpred_train_grad.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_durpred_train.py

The reference's DurationPredictor is built as FastSpeech2.__init__ builds it (fs2.py:45-50) under two configs:
  midi   usr/configs/midi/e2e/opencpop/ds100_adj_rel.yaml (5 layers, k 3, 256 channels, predictor_dropout 0.5);
  tts    usr/configs/popcs_ds_beta6.yaml (2 layers, the TTS / popcs predictor);
with seeded parameters (random_state_dict) on B = 2, T = 40 tokens: utterance 1 is padded from token 29, and the padding
rows of the input are nonzero, so d_x on them (nonzero within the kernel's reach of a real token) is pinned too.  loss =
mean((xs - target)^2).  Each config at p = 0 and at p = 0.5 with torch.nn.functional.dropout replaced by seeded keep
masks consumed in call order (each call's p and shape are checked), so the number, order and placement of the oracle's
dropout sites are pinned to the reference's.  The oracle must give the same bits: xs, loss, d_x and every gradient.
Stored per config and p: xs, the loss and d_x in full, and per gradient its norm and 64 entries at seeded flat indices
(oracle/gen_golden_train.py's sample_index)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.durpred_train_oracle import durpred_train  # noqa: E402
from oracle.gen_golden_fs2enc import MIDI_CONFIG, POPCS_CONFIG, load_reference  # noqa: E402
from oracle.gen_golden_train import sample_index  # noqa: E402

SEED, INPUT_SEED, B, T, TAIL, P = 51, 52, 2, 40, 29, 0.5
# config name, file, (idim, n_layers, n_chans, kernel_size, padding) as FastSpeech2.__init__ derives them
CASES = (("midi", MIDI_CONFIG, (256, 5, 256, 3, 'SAME')), ("tts", POPCS_CONFIG, (256, 2, 256, 3, 'SAME')))


def random_state_dict(seed, idim, L, C, k):
    """conv weights ~ U(+-1 / sqrt(fan_in)) as torch initialises them, LayerNorm affines near (1, 0), a small head"""
    rs = np.random.RandomState(seed)
    sd = {}
    for i in range(L):
        cin = idim if i == 0 else C
        b = 1.0 / np.sqrt(cin * k)
        sd[f"conv.{i}.1.weight"] = rs.uniform(-b, b, (C, cin, k))
        sd[f"conv.{i}.1.bias"] = rs.uniform(-b, b, C)
        sd[f"conv.{i}.3.weight"] = 1.0 + 0.1 * rs.standard_normal(C)
        sd[f"conv.{i}.3.bias"] = 0.1 * rs.standard_normal(C)
    sd["linear.weight"] = rs.uniform(-1, 1, (1, C)) / np.sqrt(C)
    sd["linear.bias"] = np.array([0.5])
    return {n: torch.from_numpy(v.astype(np.float32)) for n, v in sd.items()}


def case_inputs(cfg):
    """x [B, T, idim] (nonzero everywhere), mask [B, T] (True = padding), target [B, T]"""
    idim = cfg[0]
    rs = np.random.RandomState(INPUT_SEED)
    x = torch.from_numpy(rs.standard_normal((B, T, idim)).astype(np.float32))
    mask = torch.zeros(B, T, dtype=torch.bool)
    mask[1, TAIL:] = True
    tgt = torch.from_numpy(rs.standard_normal((B, T)).astype(np.float32))
    return x, mask, tgt


def seeded_masks(cfg, p):
    g = torch.Generator().manual_seed(INPUT_SEED + 2)
    return [torch.rand(B, T, cfg[2], generator=g) >= p for _ in range(cfg[1])]


def run_reference(hparams, cfg, sd, x, mask, tgt, p, masks):
    from modules.fastspeech.tts_modules import DurationPredictor
    idim, L, C, k, padding = cfg
    dp = DurationPredictor(idim, n_chans=C, n_layers=L, dropout_rate=p, padding=padding, kernel_size=k)
    dp.load_state_dict(sd, strict=True)
    dp.train()
    real = torch.nn.functional.dropout
    queue = list(masks)

    def fake(v, p_=0.5, training=True, inplace=False):
        if not training or p_ == 0:
            return real(v, p_, training, inplace)
        assert p_ == P and queue, (p_, len(queue))
        m = queue.pop(0).transpose(1, 2)            # the layers run [B, C, T]
        assert tuple(v.shape) == tuple(m.shape), (v.shape, m.shape)
        return v * m.to(v.dtype).div_(1 - p_)

    torch.nn.functional.dropout = fake
    try:
        xr = x.clone().requires_grad_(True)
        xs = dp(xr, mask)
        loss = ((xs - tgt) ** 2).mean()
        loss.backward()
    finally:
        torch.nn.functional.dropout = real
    assert not queue, f"{len(queue)} masks not consumed"
    return xs.detach(), loss.detach(), xr.grad, {n: v.grad for n, v in dp.named_parameters()}


def run_oracle(cfg, sd, x, mask, tgt, p, masks):
    """-> xs, loss, d_x, {name: gradient}"""
    P_ = {n: v.clone().requires_grad_(True) for n, v in sd.items()}
    xr = x.clone().requires_grad_(True)
    xs = durpred_train(P_, xr, mask, masks, p, cfg[3], cfg[4])
    loss = ((xs - tgt) ** 2).mean()
    loss.backward()
    return xs.detach(), loss.detach(), xr.grad, {n: v.grad for n, v in P_.items()}


def main():
    assert os.environ.get("DSX_REFERENCE_ROOT"), "set DSX_REFERENCE_ROOT to a checkout of the reference"
    hparams, configure = load_reference()
    out = dict(seed=SEED, input_seed=INPUT_SEED, B=B, T=T, tail=TAIL, p=P)
    for case, config, cfg in CASES:
        configure(config)
        C = hparams['predictor_hidden'] if hparams['predictor_hidden'] > 0 else hparams['hidden_size']
        assert (hparams['hidden_size'], hparams['dur_predictor_layers'], C, hparams['dur_predictor_kernel'],
                hparams['ffn_padding']) == cfg and hparams['dur_loss'] == 'mse', cfg
        sd = random_state_dict(SEED, *cfg[:4])
        x, mask, tgt = case_inputs(cfg)
        for p in (0.0, P):
            masks = seeded_masks(cfg, p)
            ref = run_reference(hparams, cfg, sd, x, mask, tgt, p, masks if p > 0 else [])
            mine = run_oracle(cfg, sd, x, mask, tgt, p, masks)
            for name, a, b in (("xs", mine[0], ref[0]), ("loss", mine[1], ref[1]), ("d_x", mine[2], ref[2])):
                assert torch.equal(a, b), (case, p, name, (a - b).abs().max().item())
            assert set(mine[3]) == set(ref[3]), set(mine[3]) ^ set(ref[3])
            for n in ref[3]:
                assert torch.equal(mine[3][n], ref[3][n]), (case, p, n, (mine[3][n] - ref[3][n]).abs().max().item())
            assert ref[2][1, TAIL:TAIL + 1].abs().sum() > 0, "d_x of the first padding row is 0"
            print(f"{case} p = {p}: oracle bit-exact to the reference (loss {ref[1].item():.6f})")
            pre = f"{case}.p{int(round(p * 10))}."
            xs, loss, d_x, grads = ref
            out[pre + "xs"], out[pre + "loss"], out[pre + "d_x"] = xs.numpy(), loss.numpy(), d_x.numpy()
            for n, g in grads.items():
                flat = g.reshape(-1)
                out[pre + "norm." + n] = flat.norm().numpy()
                out[pre + "val." + n] = flat[torch.from_numpy(sample_index(n, flat.numel())).long()].numpy()
    path = os.path.join(ROOT, "tests", "golden", "durpred_train_grad.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
