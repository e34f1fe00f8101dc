"""CPU: the pitch predictor's training oracle (oracle/pitchpred_train_oracle.py) reproduces
tests/golden/pitchpred_train_grad.npz bit for bit, for the aux_rel frame predictor, the 2-layer 'ph' predictor, the CWT
predictor (idim 128, odim 11) and a LEFT-padding one, at p = 0 and with the seeded p = 0.5 masks: the output, the loss,
d_x and every gradient, pos_embed_alpha's included.  oracle/gen_golden_pitchpred_train.py wrote the fixture from the
reference's own PitchPredictor in training mode, with the oracle asserted bit-exact against it."""
import numpy as np
import pytest
import torch

from conftest import golden


@pytest.mark.parametrize("case", ["frame", "ph", "cwt", "left"])
@pytest.mark.parametrize("p", [0.0, 0.5])
def test_oracle_gradients_match_the_reference_golden(case, p):
    from oracle import gen_golden_pitchpred_train as G
    from oracle.gen_golden_train import sample_index
    g = golden("pitchpred_train_grad.npz")
    assert (int(g["seed"]), int(g["input_seed"]), int(g["B"]), int(g["T"]), int(g["tail"]),
            int(g["zero_frame"])) == (G.SEED, G.INPUT_SEED, G.B, G.T, G.TAIL, G.ZERO_FRAME)
    cfg = dict((c, f) for c, _, _, f in G.CASES)[case]
    sd = G.random_state_dict(G.SEED, *cfg[:5])
    x, tgt = G.case_inputs(cfg)
    out, loss, d_x, grads = G.run_oracle(cfg, sd, x, tgt, p, G.seeded_masks(cfg, p))
    pre = f"{case}.p{int(round(p * 10))}."
    assert np.array_equal(out.numpy(), g[pre + "out"])
    assert np.array_equal(loss.numpy(), g[pre + "loss"])
    assert np.array_equal(d_x.numpy(), g[pre + "d_x"])
    assert np.abs(g[pre + "d_x"][1, G.TAIL:]).sum() > 0      # padding frames get a gradient: nothing is masked
    for k, v in grads.items():
        flat = v.reshape(-1)
        assert np.array_equal(flat.norm().numpy(), g[pre + "norm." + k]), k
        assert np.array_equal(flat[torch.from_numpy(sample_index(k, flat.numel())).long()].numpy(), g[pre + "val." + k]), k
    assert float(g[pre + "norm.pos_embed_alpha"]) > 0
    assert len([k for k in g.files if k.startswith(pre + "val.")]) == len(grads) == 4 * cfg[1] + 3
