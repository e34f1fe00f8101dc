"""TEST INFRASTRUCTURE ONLY -- the reference's PitchPredictor.forward (modules/fastspeech/tts_modules.py:222-235, and
EnergyPredictor, the same class) in training mode, as differentiable torch with the dropout masks given: ``masks[i]``
([B, T, chans] bool) is the keep mask of layer i's Dropout.  The op order and layouts are the reference's (the layers run
[B, C, T]), so oracle/gen_golden_pitchpred_train.py pins it bit for bit to the reference, gradients included.  It runs
in the dtype of its inputs (fp32 for parity, float64 for the edge tests); the sinusoidal table is built in that dtype,
with at least the reference's init_size of 4096 rows (common_layers.py:127-135).  fp16=True rounds each conv's input and
weight to fp16 as dsx_pitchpred_forward and the training forward round them (see oracle/durpred_train_oracle.py for what
that rounding does to the gradients).  A mask of None draws torch's own dropout (for timing)."""
import torch
import torch.nn.functional as F

from oracle.fs2dec_train_oracle import dropout
from oracle.fs2enc_oracle import DUR_LN_EPS, _param
from oracle.pe_oracle import make_positions, sinusoidal_table

INIT_SIZE = 4096               # PitchPredictor's SinusoidalPositionalEmbedding(idim, 0, init_size=4096)


def pitchpred_train(sd, xs, masks, p, kernel, padding='SAME', fp16=False, table=None):
    """xs [B, T, idim] -> [B, T, odim].  sd: the predictor's parameters (conv.i.1.*, conv.i.3.*, linear.*,
    pos_embed_alpha), n_layers = len(masks).  table: the sinusoidal table to use (at least 1 + T rows), or None for the
    reference's."""
    B, T, idim = xs.shape
    pad = ((kernel - 1) // 2, (kernel - 1) // 2) if padding == 'SAME' else (kernel - 1, 0)
    r = (lambda t: t.half().to(t.dtype)) if fp16 else (lambda t: t)
    if table is None:
        table = sinusoidal_table(max(INIT_SIZE, 1 + T), idim,
                                 dtype=torch.float64 if xs.dtype == torch.float64 else torch.float)
    table = table.to(xs)
    pos = make_positions(xs[..., 0].detach())
    x = xs + sd["pos_embed_alpha"] * table.index_select(0, pos.view(-1)).view(B, T, -1).detach()
    x = x.transpose(1, -1)
    for i, m in enumerate(masks):
        pre = f"conv.{i}."
        x = F.conv1d(F.pad(r(x), pad, value=0.0), r(sd[pre + "1.weight"]), sd[pre + "1.bias"])
        x = torch.relu(x)
        x = F.layer_norm(x.transpose(1, -1), (x.shape[1],), sd[pre + "3.weight"], sd[pre + "3.bias"],
                         DUR_LN_EPS).transpose(1, -1)
        x = F.dropout(x, p, training=True) if m is None else dropout(x, m.transpose(1, 2), p)
    return F.linear(x.transpose(1, -1), _param(sd["linear.weight"]), sd["linear.bias"])
