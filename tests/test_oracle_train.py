"""CPU: the oracle's fp32 autograd gradients of p_losses (L1) match tests/golden/diffnet_train_grad.npz, which
oracle/gen_golden_train.py wrote from the reference's own DiffNet + p_losses with the oracle pinned bit-exact to it."""
import numpy as np
import torch

from conftest import golden


def test_oracle_gradients_match_the_reference_golden():
    from oracle import diffnet_oracle as O
    from oracle import gen_golden_train as G
    g = golden("diffnet_train_grad.npz")
    sd = O.build_state_dict(int(g["seed"]), residual_layers=int(g["L"]), dilation_cycle_length=int(g["cycle"]))
    x_start, t, noise, cond = G.inputs()
    assert np.array_equal(t.numpy(), g["t"])
    loss, grads, d_cond = G.oracle_grads(sd, x_start, t, noise, cond)
    rel = lambda a, b: float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))
    assert rel(loss.numpy(), g["loss"]) <= 1e-5
    assert rel(d_cond.numpy(), g["d_cond"]) <= 1e-5
    assert set(grads) == {k[4:] for k in g.files if k.startswith("val.")}
    for k, v in grads.items():
        flat = v.reshape(-1)
        assert rel(flat.norm().numpy(), g["norm." + k]) <= 1e-5, k
        assert rel(flat[torch.from_numpy(G.sample_index(k, flat.numel())).long()].numpy(), g["val." + k]) <= 1e-5, k
