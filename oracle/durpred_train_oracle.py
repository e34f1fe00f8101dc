"""TEST INFRASTRUCTURE ONLY -- the reference's DurationPredictor._forward (modules/fastspeech/tts_modules.py:106-120,
dur_loss 'mse') in training mode, as differentiable torch with the dropout masks given: ``masks[i]`` ([B, T, chans]
bool) is the keep mask of layer i's Dropout.  The op order and layouts are the reference's (the layers run [B, C, T]),
so oracle/gen_golden_durpred_train.py pins it bit for bit to the reference, gradients included.  It runs in the dtype of
its inputs (fp32 for parity, float64 for the edge tests).  fp16=True rounds each conv's input and weight to fp16 as
dsx_durpred_forward and the training forward round them.  The rounding is t.half().to(t.dtype), which autograd
differentiates as two casts: the gradient that passes back through it is rounded to fp16 too, unscaled (the step's
backward rounds its gradient operands to fp16 after scaling them by a power of two).  On the shipped predictor (5
layers, 256 channels, T 65) this moves the float64 gradients by up to 4.6e-4 (relative) against a straight-through
rounding.  A mask of None draws torch's own dropout (for timing)."""
import torch
import torch.nn.functional as F

from oracle.fs2dec_train_oracle import dropout
from oracle.fs2enc_oracle import DUR_LN_EPS, _param


def durpred_train(sd, xs, mask, masks, p, kernel, padding='SAME', fp16=False):
    """xs [B, T, idim], mask [B, T] (True = padding) -> the log-domain xs [B, T].  sd: the predictor's state dict
    (conv.i.1.*, conv.i.3.*, linear.*), n_layers = len(masks)."""
    pad = ((kernel - 1) // 2, (kernel - 1) // 2) if padding == 'SAME' else (kernel - 1, 0)
    r = (lambda t: t.half().to(t.dtype)) if fp16 else (lambda t: t)
    keep = (1 - mask.float()).to(xs.dtype)
    x = xs.transpose(1, -1)
    for i, m in enumerate(masks):
        pre = f"conv.{i}."
        x = F.conv1d(F.pad(r(x), pad, value=0.0), r(sd[pre + "1.weight"]), sd[pre + "1.bias"])
        x = torch.relu(x)
        x = F.layer_norm(x.transpose(1, -1), (x.shape[1],), sd[pre + "3.weight"], sd[pre + "3.bias"],
                         DUR_LN_EPS).transpose(1, -1)
        x = F.dropout(x, p, training=True) if m is None else dropout(x, m.transpose(1, 2), p)
        x = x * keep[:, None, :]
    x = F.linear(x.transpose(1, -1), _param(sd["linear.weight"]), sd["linear.bias"])
    return (x * keep[:, :, None]).squeeze(-1)
