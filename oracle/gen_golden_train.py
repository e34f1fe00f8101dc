"""Writes tests/golden/diffnet_train_grad.npz: the reference's own DiffNet + GaussianDiffusion.p_losses (L1) with injected
t and noise, and the gradient of the loss to every DiffNet parameter and to cond, with the oracle pinned bit-exact to it.

    DSX_REFERENCE_ROOT=/path/to/DiffSinger python oracle/gen_golden_train.py

L = 20, dilation cycle 4, B = 2, T = 24, weights from build_state_dict(SEED) (the final projection re-drawn N(0, 0.02):
the reference's zeros would make every other gradient 0).  Full 20-layer gradients are about 58 MB, so the fixture keeps
the loss, the full d_cond and, per parameter, the gradient's norm and 64 entries at seeded flat indices."""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import diffnet_oracle as O  # noqa: E402

SEED, L, CYCLE, B, T, STEPS = 31, 20, 4, 2, 24, 100
N_SAMPLES = 64


def inputs():
    g = torch.Generator().manual_seed(SEED + 1)
    x_start = torch.randn(B, 1, 80, T, generator=g)
    noise = torch.randn(B, 1, 80, T, generator=g)
    cond = torch.randn(B, 256, T, generator=g)
    t = torch.tensor([7, 93], dtype=torch.long)
    return x_start, t, noise, cond


def sample_index(name, numel):
    """The flat indices of parameter `name` stored in the fixture."""
    seed = sum(ord(c) for c in name) * 7919 + numel
    return np.random.RandomState(seed % (2 ** 31)).randint(0, numel, size=N_SAMPLES).astype(np.int32)


def oracle_grads(sd, x_start, t, noise, cond):
    """(loss, {name: grad}, d_cond) of p_losses (L1) through the oracle in fp32 autograd."""
    S = O.make_schedule(O.linear_beta_schedule(STEPS, 0.06))
    P = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    c = cond.clone().requires_grad_(True)
    e = lambda a: a.gather(-1, t).reshape(t.shape[0], 1, 1, 1)      # extract() of shallow_diffusion_tts.py:32-35
    x_noisy = e(S["sqrt_alphas_cumprod"]) * x_start + e(S["sqrt_one_minus_alphas_cumprod"]) * noise
    loss = (noise - O.diffnet_forward(P, x_noisy, t, c, CYCLE)).abs().mean()
    loss.backward()
    return loss.detach(), {k: v.grad for k, v in P.items()}, c.grad


def main():
    from oracle import ref_bridge
    assert ref_bridge.available(), "set DSX_REFERENCE_ROOT to a checkout of the reference"
    ns = ref_bridge.load()
    ns.hparams.update(hidden_size=256, residual_layers=L, residual_channels=256, dilation_cycle_length=CYCLE)
    sd = O.build_state_dict(SEED, residual_layers=L, dilation_cycle_length=CYCLE)
    x_start, t, noise, cond = inputs()

    net = ns.DiffNet(80)
    net.load_state_dict(sd, strict=True)
    S = O.make_schedule(O.linear_beta_schedule(STEPS, 0.06))
    fake = types.SimpleNamespace(denoise_fn=net, loss_type="l1",
                                 sqrt_alphas_cumprod=torch.as_tensor(S["sqrt_alphas_cumprod"]),
                                 sqrt_one_minus_alphas_cumprod=torch.as_tensor(S["sqrt_one_minus_alphas_cumprod"]))
    fake.q_sample = lambda **kw: ns.sdt.GaussianDiffusion.q_sample(fake, **kw)
    c = cond.clone().requires_grad_(True)
    loss = ns.sdt.GaussianDiffusion.p_losses(fake, x_start, t, c, noise=noise)
    loss.backward()
    ref = {k: v.grad for k, v in net.named_parameters()}

    o_loss, o_grads, o_cond = oracle_grads(sd, x_start, t, noise, cond)
    assert torch.equal(o_loss, loss.detach()), (o_loss, loss)
    assert torch.equal(o_cond, c.grad)
    for k in ref:
        assert torch.equal(o_grads[k], ref[k]), k

    # the inputs are regenerated from the seed by inputs(), the sampled indices by sample_index()
    out = dict(seed=SEED, L=L, cycle=CYCLE, steps=STEPS, t=t.numpy(), loss=loss.detach().numpy(), d_cond=c.grad.numpy())
    for k, g in ref.items():
        flat = g.reshape(-1)
        out["norm." + k] = flat.norm().numpy()
        out["val." + k] = flat[torch.from_numpy(sample_index(k, flat.numel())).long()].numpy()
    path = os.path.join(ROOT, "tests", "golden", "diffnet_train_grad.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes): loss {loss.item():.6f}, oracle bit-exact to the reference")


if __name__ == "__main__":
    main()
