"""TEST INFRASTRUCTURE ONLY -- the reference's FastSpeech2 decoder (FFTBlocks.forward, modules/fastspeech/tts_modules.py:
282-307, EncSALayer / TransformerFFNLayer of modules/commons/common_layers.py:486-588) in training mode, as
differentiable fp32 torch with the dropout masks given: ``masks[s]`` ([B, T, n] bool) is the keep mask of dropout site s
(0 after x + alpha * positions; per layer i, 1 + 3 i after out_proj, 2 + 3 i after the FFN activation, 3 + 3 i after
ffn_2), and dropout(v) is v * (mask / (1 - p)) as ATen's dropout computes it.  Attention probabilities have no dropout
(attention_dropout = 0).  The graph is oracle.fs2dec_oracle.decoder's (the reference's [T, B, C] layout and op order), so
oracle/gen_golden_fs2dec_train.py pins it bit for bit to the reference, gradients included."""
import torch
import torch.nn.functional as F

from oracle.fs2dec_oracle import LN_EPS, _ffn1_key, padding_mask
from oracle.pe_oracle import make_positions, sinusoidal_table


def dropout(v, mask, p):
    """F.dropout(v, p) with the keep mask given (mask in v's layout)"""
    return v * mask.to(v.dtype).div_(1 - p)


def _ffn(sd, hp, i, x, mask, p):
    """TransformerFFNLayer.forward, common_layers.py:503-522 (x: T x B x C), with its dropout"""
    k = int(hp['dec_ffn_kernel_size'])
    w = _ffn1_key(hp, i)
    y = x.permute(1, 2, 0)
    if hp['ffn_padding'] == 'SAME':
        y = F.conv1d(y, sd[w + "weight"], sd[w + "bias"], padding=k // 2)
    else:
        y = F.conv1d(F.pad(y, (k - 1, 0), value=0.0), sd[w + "weight"], sd[w + "bias"])
    y = y.permute(2, 0, 1)
    y = y * k ** -0.5
    y = F.gelu(y) if hp['ffn_act'] == 'gelu' else F.relu(y)
    y = dropout(y, mask, p)
    p2 = f"layers.{i}.op.ffn.ffn_2."
    w2 = sd[p2 + "weight"]
    return F.linear(y, w2 if w2.requires_grad else torch.nn.Parameter(w2), sd[p2 + "bias"])


def decoder_train(sd, x, hp, masks, p, layer_input=None):
    """x [B, T, H] -> [B, T, H]; a float64 x gets a float64 position table.  ``layer_input(i, x)``, if given, replaces
    the residual stream x ([T, B, H]) entering layer i (an identity autograd Function there can alter its backward)."""
    B, T, H = x.shape
    heads = int(hp['num_heads'])
    tb = lambda s: masks[s].transpose(0, 1)                        # [B, T, n] -> the layers' [T, B, n]
    pad = padding_mask(x)
    nonpad_TB = 1 - pad.transpose(0, 1).to(x.dtype)[:, :, None]
    table = sinusoidal_table(max(2000, 1 + T), H, dtype=torch.float64 if x.dtype == torch.float64 else torch.float).to(x)
    pos = make_positions(x[..., 0])
    x = x + sd["pos_embed_alpha"] * table.index_select(0, pos.view(-1)).view(B, T, -1)
    x = dropout(x, masks[0], p)
    x = x.transpose(0, 1) * nonpad_TB
    keep = (1 - pad.to(x.dtype)).transpose(0, 1)[..., None]
    for i in range(int(hp['dec_layers'])):
        pre = f"layers.{i}.op."
        if layer_input is not None:
            x = layer_input(i, x)
        residual = x
        y = F.layer_norm(x, (H,), sd[pre + "layer_norm1.weight"], sd[pre + "layer_norm1.bias"], LN_EPS)
        y, _ = F.multi_head_attention_forward(y, y, y, H, heads, sd[pre + "self_attn.in_proj_weight"], None, None, None,
                                              False, 0.0, sd[pre + "self_attn.out_proj.weight"], None, training=True,
                                              key_padding_mask=pad, need_weights=True, attn_mask=None)
        x = (residual + dropout(y, tb(1 + 3 * i), p)) * keep
        residual = x
        y = F.layer_norm(x, (H,), sd[pre + "layer_norm2.weight"], sd[pre + "layer_norm2.bias"], LN_EPS)
        x = (residual + dropout(_ffn(sd, hp, i, y, tb(2 + 3 * i), p), tb(3 + 3 * i), p)) * keep
        x = x * nonpad_TB
    x = F.layer_norm(x, (H,), sd["layer_norm.weight"], sd["layer_norm.bias"], LN_EPS) * nonpad_TB
    return x.transpose(0, 1)
