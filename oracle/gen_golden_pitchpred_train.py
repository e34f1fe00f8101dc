"""TEST INFRASTRUCTURE ONLY -- pins oracle/pitchpred_train_oracle.py to the LIVE reference PitchPredictor in training mode
(needs a checkout of the reference: DSX_REFERENCE_ROOT; runs on a CPU) and writes tests/golden/pitchpred_train_grad.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_pitchpred_train.py

The reference's PitchPredictor is built as FastSpeech2.__init__ builds it (fs2.py:52-78), with the hparams of:
  frame  usr/configs/midi/cascade/opencs/aux_rel.yaml (256 -> 256, 5 layers, k 5, odim 2: f0 and uv per frame);
  ph     usr/configs/popcs_fs2.yaml with pitch_type 'ph' (2 layers, odim 1: f0 per token);
  cwt    configs/tts/lj/fs2.yaml (the one inside cwt_predictor: idim cwt_hidden_size 128, odim 10 + use_uv = 11);
and one LEFT-padding case (the frame predictor with ffn_padding 'LEFT', 3 layers).  Seeded parameters
(random_state_dict, pos_embed_alpha 0.7) on B = 2, T = 40 frames: utterance 1 is zero from frame 29 (padding frames, as
FastSpeech2 feeds them), and frame 5 of utterance 0 has channel 0 exactly 0, so make_positions skips it.  loss =
mean((out - target)^2).  Each case at p = 0 and at p = 0.5 with torch.nn.functional.dropout replaced by seeded keep masks
consumed in call order, so the number, order and placement of the oracle's dropout sites are pinned to the reference's.
The oracle must give the same bits: the output, the loss, d_x and every gradient.  Stored per case and p: the output,
the loss and d_x in full, and per gradient its norm and 64 entries at seeded flat indices (oracle/gen_golden_train.py's
sample_index)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.gen_golden_fs2enc import load_reference  # noqa: E402
from oracle.gen_golden_train import sample_index  # noqa: E402
from oracle.pitchpred_train_oracle import pitchpred_train  # noqa: E402

SEED, INPUT_SEED, B, T, TAIL, ZERO_FRAME, P = 61, 62, 2, 40, 29, 5, 0.5
AUX_REL = "usr/configs/midi/cascade/opencs/aux_rel.yaml"
POPCS = "usr/configs/popcs_fs2.yaml"
LJ = "configs/tts/lj/fs2.yaml"
# case, config file, hparams overrides, (idim, n_layers, n_chans, odim, kernel_size, padding)
CASES = (("frame", AUX_REL, {}, (256, 5, 256, 2, 5, 'SAME')),
         ("ph", POPCS, {"pitch_type": "ph"}, (256, 2, 256, 1, 5, 'SAME')),
         ("cwt", LJ, {}, (128, 2, 256, 11, 5, 'SAME')),
         ("left", AUX_REL, {"ffn_padding": "LEFT", "predictor_layers": 3}, (256, 3, 256, 2, 5, 'LEFT')))


def random_state_dict(seed, idim, L, C, odim, k):
    """conv weights ~ U(+-1 / sqrt(fan_in)) as torch initialises them, LayerNorm affines near (1, 0), a small head,
    pos_embed_alpha 0.7, and the embedding's _float_tensor buffer"""
    rs = np.random.RandomState(seed)
    sd = {}
    for i in range(L):
        cin = idim if i == 0 else C
        b = 1.0 / np.sqrt(cin * k)
        sd[f"conv.{i}.1.weight"] = rs.uniform(-b, b, (C, cin, k))
        sd[f"conv.{i}.1.bias"] = rs.uniform(-b, b, C)
        sd[f"conv.{i}.3.weight"] = 1.0 + 0.1 * rs.standard_normal(C)
        sd[f"conv.{i}.3.bias"] = 0.1 * rs.standard_normal(C)
    sd["linear.weight"] = rs.uniform(-1, 1, (odim, C)) / np.sqrt(C)
    sd["linear.bias"] = 0.1 * rs.standard_normal(odim)
    sd["pos_embed_alpha"] = np.array([0.7])
    sd["embed_positions._float_tensor"] = np.array([1.0])
    return {n: torch.from_numpy(v.astype(np.float32)) for n, v in sd.items()}


def case_inputs(cfg):
    """x [B, T, idim] (utterance 1 zero from TAIL, channel 0 of frame ZERO_FRAME of utterance 0 zero), target
    [B, T, odim]"""
    idim, odim = cfg[0], cfg[3]
    rs = np.random.RandomState(INPUT_SEED)
    x = torch.from_numpy(rs.standard_normal((B, T, idim)).astype(np.float32))
    x[1, TAIL:] = 0
    x[0, ZERO_FRAME, 0] = 0
    tgt = torch.from_numpy(rs.standard_normal((B, T, odim)).astype(np.float32))
    return x, tgt


def seeded_masks(cfg, p):
    g = torch.Generator().manual_seed(INPUT_SEED + 2)
    return [torch.rand(B, T, cfg[2], generator=g) >= p for _ in range(cfg[1])]


def params(sd):
    return {n: v for n, v in sd.items() if n != "embed_positions._float_tensor"}


def run_reference(cfg, sd, x, tgt, p, masks):
    from modules.fastspeech.tts_modules import PitchPredictor
    idim, L, C, odim, k, padding = cfg
    pp = PitchPredictor(idim, n_chans=C, n_layers=L, dropout_rate=p, odim=odim, padding=padding, kernel_size=k)
    pp.load_state_dict(sd, strict=True)
    pp.train()
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
        out = pp(xr)
        loss = ((out - tgt) ** 2).mean()
        loss.backward()
    finally:
        torch.nn.functional.dropout = real
    assert not queue, f"{len(queue)} masks not consumed"
    return out.detach(), loss.detach(), xr.grad, {n: v.grad for n, v in pp.named_parameters()}


def run_oracle(cfg, sd, x, tgt, p, masks):
    """-> out, loss, d_x, {name: gradient}"""
    P_ = {n: v.clone().requires_grad_(True) for n, v in params(sd).items()}
    xr = x.clone().requires_grad_(True)
    out = pitchpred_train(P_, xr, masks, p, cfg[4], cfg[5])
    loss = ((out - tgt) ** 2).mean()
    loss.backward()
    return out.detach(), loss.detach(), xr.grad, {n: v.grad for n, v in P_.items()}


def main():
    assert os.environ.get("DSX_REFERENCE_ROOT"), "set DSX_REFERENCE_ROOT to a checkout of the reference"
    hparams, configure = load_reference()
    out = dict(seed=SEED, input_seed=INPUT_SEED, B=B, T=T, tail=TAIL, zero_frame=ZERO_FRAME, p=P)
    for case, config, over, cfg in CASES:
        configure(config)
        hparams.update(over)
        C = hparams['predictor_hidden'] if hparams['predictor_hidden'] > 0 else hparams['hidden_size']
        cwt = hparams['pitch_type'] == 'cwt'
        idim = hparams['cwt_hidden_size'] if cwt else hparams['hidden_size']
        odim = (11 if hparams['use_uv'] else 10) if cwt else (2 if hparams['pitch_type'] == 'frame' else 1)
        assert (idim, hparams['predictor_layers'], C, odim, hparams['predictor_kernel'],
                hparams['ffn_padding']) == cfg, (case, cfg)
        assert hparams['predictor_dropout'] == P
        sd = random_state_dict(SEED, *cfg[:5])
        x, tgt = case_inputs(cfg)
        for p in (0.0, P):
            masks = seeded_masks(cfg, p)
            ref = run_reference(cfg, sd, x, tgt, p, masks if p > 0 else [])
            mine = run_oracle(cfg, sd, x, tgt, p, masks)
            for name, a, b in (("out", mine[0], ref[0]), ("loss", mine[1], ref[1]), ("d_x", mine[2], ref[2])):
                assert torch.equal(a, b), (case, p, name, (a - b).abs().max().item())
            assert set(mine[3]) == set(ref[3]), set(mine[3]) ^ set(ref[3])
            for n in ref[3]:
                assert torch.equal(mine[3][n], ref[3][n]), (case, p, n, (mine[3][n] - ref[3][n]).abs().max().item())
            print(f"{case} p = {p}: oracle bit-exact to the reference (loss {ref[1].item():.6f})")
            pre = f"{case}.p{int(round(p * 10))}."
            o, loss, d_x, grads = ref
            out[pre + "out"], out[pre + "loss"], out[pre + "d_x"] = o.numpy(), loss.numpy(), d_x.numpy()
            for n, g in grads.items():
                flat = g.reshape(-1)
                out[pre + "norm." + n] = flat.norm().numpy()
                out[pre + "val." + n] = flat[torch.from_numpy(sample_index(n, flat.numel())).long()].numpy()
    path = os.path.join(ROOT, "tests", "golden", "pitchpred_train_grad.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path)} bytes)")


if __name__ == "__main__":
    main()
