"""CPU: the FastSpeech2 encoder's training oracle (oracle/fs2enc_train_oracle.py) reproduces
tests/golden/fs2enc_train_grad.npz bit for bit, for the MIDI encoder (rel_pos, three addends) and the sinusoidal encoder,
at p = 0 and with the seeded p = 0.1 masks.  oracle/gen_golden_fs2enc_train.py wrote the fixture from the reference's own
encoders in training mode, with the oracle asserted bit-exact against them."""
import numpy as np
import pytest
import torch

from conftest import golden


@pytest.mark.parametrize("case", ["midi", "sin"])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_oracle_gradients_match_the_reference_golden(case, p):
    from oracle import gen_golden_fs2enc_train as G
    from oracle.gen_golden_train import sample_index
    g = golden("fs2enc_train_grad.npz")
    hp = {c: h for c, _, h in G.CASES}[case]
    assert {k: g[f"hp.{case}.{k}"].item() for k in hp} == hp
    assert (int(g["seed"]), int(g["input_seed"]), int(g["vocab"])) == (G.SEED, G.INPUT_SEED, G.VOCAB)
    enc_sd, tok, adds, tgt = G.case_inputs(case, hp)
    _, loss, d_add, grads = G.run_oracle(hp, enc_sd, tok, adds, tgt, p, G.seeded_masks(hp, p))
    pre = f"{case}.p{int(round(p * 10))}."
    assert np.array_equal(loss.numpy(), g[pre + "loss"])
    full = {"embed_tokens.weight": grads["embed_tokens.weight"]}
    if case == "midi":
        full["d_add"] = d_add
    else:
        assert d_add is None
    for k, v in dict(grads, **full).items():
        if p == 0 and k in full:
            assert np.array_equal(v.numpy(), g[pre + "grad." + k]), k
            continue
        flat = v.reshape(-1)
        assert np.array_equal(flat.norm().numpy(), g[pre + "norm." + k]), k
        assert np.array_equal(flat[torch.from_numpy(sample_index(k, flat.numel())).long()].numpy(), g[pre + "val." + k]), k
    assert len([k for k in g.files if k.startswith(pre + "val.") or k.startswith(pre + "grad.")]) == len(grads) + (
        case == "midi")
