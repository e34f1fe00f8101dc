"""CPU: the duration predictor's training oracle (oracle/durpred_train_oracle.py) reproduces
tests/golden/durpred_train_grad.npz bit for bit, for the ds100_adj_rel (5 layers) and TTS (2 layers) predictors, at p = 0
and with the seeded p = 0.5 masks: xs, the loss, d_x (padding rows included) and every gradient.
oracle/gen_golden_durpred_train.py wrote the fixture from the reference's own DurationPredictor in training mode, with
the oracle asserted bit-exact against it."""
import numpy as np
import pytest
import torch

from conftest import golden


@pytest.mark.parametrize("case", ["midi", "tts"])
@pytest.mark.parametrize("p", [0.0, 0.5])
def test_oracle_gradients_match_the_reference_golden(case, p):
    from oracle import gen_golden_durpred_train as G
    from oracle.gen_golden_train import sample_index
    g = golden("durpred_train_grad.npz")
    assert (int(g["seed"]), int(g["input_seed"]), int(g["B"]), int(g["T"]), int(g["tail"])) == (G.SEED, G.INPUT_SEED,
                                                                                                 G.B, G.T, G.TAIL)
    cfg = dict((c, f) for c, _, f in G.CASES)[case]
    sd = G.random_state_dict(G.SEED, *cfg[:4])
    x, mask, tgt = G.case_inputs(cfg)
    xs, loss, d_x, grads = G.run_oracle(cfg, sd, x, mask, tgt, p, G.seeded_masks(cfg, p))
    pre = f"{case}.p{int(round(p * 10))}."
    assert np.array_equal(xs.numpy(), g[pre + "xs"])
    assert np.array_equal(loss.numpy(), g[pre + "loss"])
    assert np.array_equal(d_x.numpy(), g[pre + "d_x"])
    assert np.abs(g[pre + "d_x"][1, G.TAIL]).sum() > 0      # a padding row next to a real token
    for k, v in grads.items():
        flat = v.reshape(-1)
        assert np.array_equal(flat.norm().numpy(), g[pre + "norm." + k]), k
        assert np.array_equal(flat[torch.from_numpy(sample_index(k, flat.numel())).long()].numpy(), g[pre + "val." + k]), k
    assert len([k for k in g.files if k.startswith(pre + "val.")]) == len(grads) == 4 * cfg[1] + 2
