"""TEST INFRASTRUCTURE ONLY -- functional torch-CPU fp32 restatement of the reference's FastSpeech2 decoder
(FastspeechDecoder = FFTBlocks, modules/fastspeech/tts_modules.py:251-357, with EncSALayer / MultiheadAttention /
TransformerFFNLayer of modules/commons/common_layers.py:166-588, the position embedding of :88-143 and
utils/__init__.py:145-157), in eval mode, over a state dict ``sd`` with the reference's names.  ``hp`` holds the hparams
the reference reads: hidden_size, dec_layers, dec_ffn_kernel_size, num_heads, ffn_padding, ffn_act."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.pe_oracle import make_positions, sinusoidal_table

# the shipped singing configuration (usr/configs/popcs_ds_beta6.yaml and its bases)
HPARAMS_POPCS = dict(hidden_size=256, dec_layers=4, dec_ffn_kernel_size=9, num_heads=2, ffn_padding='SAME',
                     ffn_act='gelu', dropout=0.1)
LN_EPS = 1e-5          # common_layers.LayerNorm / nn.LayerNorm defaults


def padding_mask(x):
    """tts_modules.py:288 -- a frame is padding when the sum of |channels| is 0"""
    return x.abs().sum(-1).eq(0)


def _ffn1_key(hp, i):
    return f"layers.{i}.op.ffn.ffn_1." if hp['ffn_padding'] == 'SAME' else f"layers.{i}.op.ffn.ffn_1.1."


def _ffn(sd, hp, i, x):
    """TransformerFFNLayer.forward, common_layers.py:503-522 (x: T x B x C)"""
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
    p = f"layers.{i}.op.ffn.ffn_2."
    # a module's weight requires grad, and ATen's matmul picks how it folds the strided 3-d input by that: the same
    # flag keeps the sums in the reference's order
    w2 = sd[p + "weight"]
    return F.linear(y, w2 if w2.requires_grad else torch.nn.Parameter(w2), sd[p + "bias"])


def decoder(sd, x, hp, table=None):
    """FFTBlocks.forward(x), tts_modules.py:282-307, padding_mask = attn_mask = None: x [B, T, H] -> [B, T, H].
    ``table``: the module's cached sinusoidal table, or None to build it here (its rows do not depend on its size)."""
    B, T, H = x.shape
    heads = int(hp['num_heads'])
    pad = padding_mask(x)
    nonpad_TB = 1 - pad.transpose(0, 1).to(x.dtype)[:, :, None]   # .float() in the reference; x.dtype keeps .half() fp16
    if table is None or table.shape[0] < 1 + T:                    # common_layers.py:127-135
        table = sinusoidal_table(max(2000, 1 + T), H, dtype=torch.float64 if x.dtype == torch.float64 else torch.float)
    table = table.to(x)
    pos = make_positions(x[..., 0])
    x = x + sd["pos_embed_alpha"] * table.index_select(0, pos.view(-1)).view(B, T, -1)
    x = x.transpose(0, 1) * nonpad_TB
    keep = (1 - pad.to(x.dtype)).transpose(0, 1)[..., None]
    for i in range(int(hp['dec_layers'])):
        p = f"layers.{i}.op."
        # EncSALayer.forward, common_layers.py:564-588 (dropout = identity)
        residual = x
        y = F.layer_norm(x, (H,), sd[p + "layer_norm1.weight"], sd[p + "layer_norm1.bias"], LN_EPS)
        y, _ = F.multi_head_attention_forward(y, y, y, H, heads, sd[p + "self_attn.in_proj_weight"], None, None, None,
                                              False, 0.0, sd[p + "self_attn.out_proj.weight"], None, training=False,
                                              key_padding_mask=pad, need_weights=True, attn_mask=None)
        x = (residual + y) * keep
        residual = x
        y = F.layer_norm(x, (H,), sd[p + "layer_norm2.weight"], sd[p + "layer_norm2.bias"], LN_EPS)
        x = (residual + _ffn(sd, hp, i, y)) * keep
        x = x * nonpad_TB                                           # tts_modules.py:298
    x = F.layer_norm(x, (H,), sd["layer_norm.weight"], sd["layer_norm.bias"], LN_EPS) * nonpad_TB
    return x.transpose(0, 1)


def state_dict_shapes(hp):
    """name -> shape of the reference decoder's state dict, in its order"""
    H, k = int(hp['hidden_size']), int(hp['dec_ffn_kernel_size'])
    out = {"pos_embed_alpha": (1,), "embed_positions._float_tensor": (1,)}
    for i in range(int(hp['dec_layers'])):
        p = f"layers.{i}.op."
        out.update({p + "layer_norm1.weight": (H,), p + "layer_norm1.bias": (H,),
                    p + "self_attn.in_proj_weight": (3 * H, H), p + "self_attn.out_proj.weight": (H, H),
                    p + "layer_norm2.weight": (H,), p + "layer_norm2.bias": (H,),
                    _ffn1_key(hp, i) + "weight": (4 * H, H, k), _ffn1_key(hp, i) + "bias": (4 * H,),
                    p + "ffn.ffn_2.weight": (H, 4 * H), p + "ffn.ffn_2.bias": (H,)})
    out.update({"layer_norm.weight": (H,), "layer_norm.bias": (H,)})
    return out


def random_state_dict(seed, hp):
    """Seeded parameters from np.random.RandomState (the same on every machine): Xavier-uniform weights, and non-trivial
    LayerNorm affines (so LN2 of a padding row, beta2, is not 0), biases and pos_embed_alpha."""
    rs = np.random.RandomState(seed)
    out = {}
    for name, shape in state_dict_shapes(hp).items():
        if name.endswith("_float_tensor"):
            v = np.zeros(shape)
        elif name == "pos_embed_alpha":
            v = 0.5 + rs.uniform(0, 1, shape)
        elif "layer_norm" in name:
            v = 1.0 + 0.2 * rs.standard_normal(shape) if name.endswith("weight") else 0.1 * rs.standard_normal(shape)
        elif name.endswith("bias"):
            v = 0.05 * rs.standard_normal(shape)
        else:
            rf = int(np.prod(shape[2:]))
            a = np.sqrt(6.0 / (shape[1] * rf + shape[0] * rf))
            v = rs.uniform(-a, a, shape)
        out[name] = torch.from_numpy(np.asarray(v, np.float32))
    return out


def checksums(sd):
    """name -> (sum, sum of |v|) in float64"""
    return {k: np.array([v.double().sum().item(), v.double().abs().sum().item()]) for k, v in sd.items()}


def fixture_input(seed, B, T, H, tail=None):
    """decoder_inp-like input: seeded normals; utterance 0 has frame T // 5 with only channel 0 zeroed (a position the
    scan skips) and frame T // 2 all zero (a padding key and query inside the utterance); utterance 1 (if any) is zero
    from frame `tail` on."""
    x = torch.from_numpy(np.random.RandomState(seed).standard_normal((B, T, H)).astype(np.float32))
    if T >= 3:
        x[0, T // 5, 0] = 0
        x[0, T // 2] = 0
    if B > 1 and tail is not None:
        x[1, tail:] = 0
    return x


def decoder_fp16_sim(sd, x, hp):
    """The decoder with every GEMM operand rounded to fp16 as the dsx kernels round them (weights, LayerNorm outputs,
    Q scaled in fp32 before rounding, K, V, the softmax numerators P, the attention output, the FFN activations);
    accumulation, the residual stream, LayerNorm statistics and the softmax sums in fp32.  Used to size the GPU tests'
    tolerances."""
    r = lambda t: t.half().float()
    B, T, H = x.shape
    heads = int(hp['num_heads'])
    D = H // heads
    k = int(hp['dec_ffn_kernel_size'])
    pad = padding_mask(x)
    keep = (~pad).float()[..., None]
    table = sinusoidal_table(max(2000, 1 + T), H)
    pos = make_positions(x[..., 0])
    x = (x + sd["pos_embed_alpha"] * table.index_select(0, pos.view(-1)).view(B, T, -1)) * keep
    kbias = torch.zeros(B, 1, 1, T).masked_fill(pad[:, None, None, :], float("-inf"))
    for i in range(int(hp['dec_layers'])):
        p = f"layers.{i}.op."
        y = r(F.layer_norm(x, (H,), sd[p + "layer_norm1.weight"], sd[p + "layer_norm1.bias"], LN_EPS))
        qkv = y @ r(sd[p + "self_attn.in_proj_weight"]).t()
        q, kk, v = qkv.split(H, -1)
        q = r(q * (1.0 / D) ** 0.5).view(B, T, heads, D).transpose(1, 2)
        kk, v = r(kk).view(B, T, heads, D).transpose(1, 2), r(v).view(B, T, heads, D).transpose(1, 2)
        s = q @ kk.transpose(-1, -2) + kbias
        m = s.amax(-1, keepdim=True)
        e = torch.exp(s - torch.where(torch.isinf(m), torch.zeros_like(m), m))
        l = e.sum(-1, keepdim=True)
        o = (r(e) @ v) / l
        o = r(torch.nan_to_num(o, nan=0.0).transpose(1, 2).reshape(B, T, H))
        x = (x + o @ r(sd[p + "self_attn.out_proj.weight"]).t()) * keep
        y = r(F.layer_norm(x, (H,), sd[p + "layer_norm2.weight"], sd[p + "layer_norm2.bias"], LN_EPS))
        w = _ffn1_key(hp, i)
        yc = y.transpose(1, 2)
        yc = F.pad(yc, (k // 2, k // 2) if hp['ffn_padding'] == 'SAME' else (k - 1, 0))
        h1 = (F.conv1d(yc, r(sd[w + "weight"])) + sd[w + "bias"][:, None]).transpose(1, 2) * k ** -0.5
        h1 = r(F.gelu(h1) if hp['ffn_act'] == 'gelu' else F.relu(h1))
        x = (x + (h1 @ r(sd[p + "ffn.ffn_2.weight"]).t() + sd[p + "ffn.ffn_2.bias"])) * keep
    return F.layer_norm(x, (H,), sd["layer_norm.weight"], sd["layer_norm.bias"], LN_EPS) * keep


def flops_per_frame(H=256, L=4, k=9, T=1024):
    """2 x multiply-adds per frame: in_proj 3H^2, out_proj H^2, ffn_1 4kH^2, ffn_2 4H^2 and the attention 2TH per layer"""
    return 2 * L * (8 * H * H + 4 * k * H * H + 2 * T * H)
