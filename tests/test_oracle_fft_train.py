"""CPU: the FFT denoiser's training oracle (oracle/fft_train_oracle.py) reproduces tests/golden/fft_train_grad.npz, which
oracle/gen_golden_fft_train.py wrote from the reference's own FFT in training mode with the oracle pinned bit-exact."""
import numpy as np
import torch

from conftest import golden


def test_oracle_gradients_match_the_reference_golden():
    from oracle import fft_oracle as O
    from oracle import gen_golden_fft_train as G
    from oracle.gen_golden_train import sample_index
    g = golden("fft_train_grad.npz")
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    sd = O.random_state_dict(int(g["seed"]), hp)
    assert np.array_equal(g["t"], np.asarray(G.STEPS))
    loss, grads, d_cond = G.oracle_grads(sd, hp)
    rel = lambda a, b: float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))
    assert rel(loss.numpy(), g["loss"]) <= 1e-5
    assert rel(d_cond.numpy(), g["d_cond"]) <= 1e-5
    assert set(grads) == {k[4:] for k in g.files if k.startswith("val.")} and len(grads) == 53
    for k, v in grads.items():
        flat = v.reshape(-1)
        assert rel(flat.norm().numpy(), g["norm." + k]) <= 1e-5, k
        assert rel(flat[torch.from_numpy(sample_index(k, flat.numel())).long()].numpy(), g["val." + k]) <= 1e-5, k
