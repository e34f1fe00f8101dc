"""TEST INFRASTRUCTURE ONLY -- pins oracle/fft_train_oracle.py to the LIVE reference FFT denoiser in training mode (needs a
checkout of the reference: DSX_REFERENCE_ROOT) and writes tests/golden/fft_train_grad.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_fft_train.py

The reference's FFT (usr/diff/candidate_decoder.py:35-100) is built as oracle/gen_golden_fft.py builds it
(usr/configs/popcs_ds_beta6.yaml: hidden 256, 4 layers, 2 heads, kernel 9, GELU, 'SAME', residual_channels 256) with
dropout 0, put in training mode and run on B = 2, T = 24 at per-utterance diffusion steps, with p_losses' L1 loss
mean |eps - noise| (usr/diff/shallow_diffusion_tts.py:213-231 with a fixed x_noisy).  The oracle must reproduce the
loss, d_cond and every parameter gradient bit for bit.  The fixture holds the loss, the full d_cond and, per parameter,
the gradient's norm and 64 entries at seeded flat indices (oracle/gen_golden_train.py's sample_index)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import fft_oracle as O  # noqa: E402
from oracle import ref_bridge  # noqa: E402
from oracle.fft_train_oracle import forward_train  # noqa: E402
from oracle.gen_golden_fft import CONFIG, HP_KEYS  # noqa: E402
from oracle.gen_golden_train import sample_index  # noqa: E402

SEED, INPUT_SEED, B, T = 51, 52, 2, 24
STEPS = (5, 60)


def inputs(H):
    """x_noisy [B, 1, 80, T], t [B], cond [B, H, T], noise [B, 1, 80, T]"""
    rs = np.random.RandomState(INPUT_SEED)
    spec = torch.from_numpy(rs.standard_normal((B, 1, 80, T)).astype(np.float32))
    cond = torch.from_numpy(rs.standard_normal((B, H, T)).astype(np.float32))
    noise = torch.from_numpy(rs.standard_normal((B, 1, 80, T)).astype(np.float32))
    return spec, torch.tensor(STEPS, dtype=torch.long), cond, noise


def oracle_grads(sd, hp):
    """loss, {name: grad}, d_cond of the oracle at p = 0"""
    spec, t, cond, noise = inputs(int(hp["hidden_size"]))
    P = {k: v.clone().requires_grad_(True) for k, v in sd.items() if k != "embed_positions._float_tensor"}
    c = cond.clone().requires_grad_(True)
    H, L = int(hp["hidden_size"]), int(hp["dec_layers"])
    masks = [torch.ones(B, T, 4 * H if s > 0 and s % 3 == 2 else H, dtype=torch.bool) for s in range(1 + 3 * L)]
    loss = (forward_train(P, spec, t, c, hp, masks, 0.0) - noise).abs().mean()
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in P.items()}, c.grad


def main():
    assert ref_bridge.available(), "set DSX_REFERENCE_ROOT to a checkout of the reference"
    ns = ref_bridge.load(CONFIG)
    hparams = ns.hparams
    hparams["dropout"] = 0.0
    cwd = os.getcwd()
    os.chdir(ref_bridge.REF_ROOT)
    try:
        from usr.diff.candidate_decoder import FFT
    finally:
        os.chdir(cwd)
    hp = {k: hparams[k] for k in HP_KEYS}
    net = FFT(hp["hidden_size"], hp["dec_layers"], hp["dec_ffn_kernel_size"], hp["num_heads"])
    sd = O.random_state_dict(SEED, hp)
    net.load_state_dict(sd, strict=True)
    net.train()
    spec, t, cond, noise = inputs(hp["hidden_size"])
    c = cond.clone().requires_grad_(True)
    loss = (net(spec, t, c) - noise).abs().mean()
    loss.backward()
    ref = {k: v.grad for k, v in net.named_parameters()}

    mine_loss, mine, d_cond = oracle_grads(sd, hp)
    assert torch.equal(mine_loss, loss.detach()), (mine_loss.item(), loss.item())
    assert torch.equal(d_cond, c.grad), (d_cond - c.grad).abs().max().item()
    assert set(mine) == set(ref), set(mine) ^ set(ref)
    for k in ref:
        assert torch.equal(mine[k], ref[k]), (k, (mine[k] - ref[k]).abs().max().item())
    print(f"oracle bit-exact to the reference (loss {loss.item():.6f}, {len(ref)} parameters)")

    out = dict(seed=SEED, input_seed=INPUT_SEED, B=B, T=T, t=np.asarray(STEPS), loss=loss.detach().numpy(),
               d_cond=c.grad.numpy())
    out.update({"hp." + k: np.asarray(v) for k, v in hp.items() if k != "dropout"})
    for k, g in ref.items():
        flat = g.reshape(-1)
        out["norm." + k] = flat.norm().numpy()
        out["val." + k] = flat[torch.from_numpy(sample_index(k, flat.numel())).long()].numpy()
    path = os.path.join(ROOT, "tests", "golden", "fft_train_grad.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
