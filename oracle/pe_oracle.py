"""TEST INFRASTRUCTURE ONLY -- functional torch-CPU fp32 restatement of the reference's pitch extractor
(modules/fastspeech/pe.py:7-149 with modules/fastspeech/tts_modules.py:192-235, modules/commons/common_layers.py:88-143,
utils/__init__.py:145-157 and utils/pitch_utils.py:63-76), in eval mode, over a state dict ``sd`` with the reference's
names.  ``hp`` holds the hparams the reference reads: hidden_size, predictor_hidden, ffn_padding, predictor_kernel,
pitch_type, use_uv, pitch_norm (f0_mean / f0_std for 'standard')."""
import math
import re

import torch
import torch.nn.functional as F

# hparams of the e2e singing configs (usr/configs/midi/e2e/opencpop/ds100_adj_rel.yaml and its bases)
HPARAMS_E2E = dict(hidden_size=256, predictor_hidden=-1, ffn_padding='SAME', predictor_kernel=5, pitch_type='frame',
                   use_uv=True, pitch_norm='log', f0_mean=None, f0_std=None)


def padding_mask(mel):
    """pe.py:29, :143 -- a frame is padding when the sum of |bins| is 0"""
    return mel.abs().sum(-1).eq(0)


def _round(fp16):
    """fp16=True: a GEMM operand as the dsx kernels read it, rounded to fp16 (and back to the tensor's own dtype)"""
    return (lambda t: t.half().to(t.dtype)) if fp16 else (lambda t: t)


def prenet(sd, mel, pre="mel_prenet", fp16=False):
    """Prenet.forward, pe.py:23-41 (strides 1): 3 x [conv k5 pad 2, ReLU, BatchNorm1d eval] * nonpadding, out_proj"""
    r = _round(fp16)
    nonpad = 1 - padding_mask(mel).to(mel.dtype)[:, None, :]   # .float() in the reference; mel.dtype keeps a .half() run in fp16
    x = mel.transpose(1, 2)
    for i in range(3):
        p = f"{pre}.layers.{i}"
        x = F.relu(F.conv1d(r(x), r(sd[f"{p}.0.weight"]), sd[f"{p}.0.bias"], padding=2))
        x = F.batch_norm(x, sd[f"{p}.2.running_mean"], sd[f"{p}.2.running_var"], sd[f"{p}.2.weight"], sd[f"{p}.2.bias"],
                         False, 0.1, 1e-5)
        x = x * nonpad
    x = F.linear(r(x.transpose(1, 2)), r(sd[f"{pre}.out_proj.weight"]), sd[f"{pre}.out_proj.bias"])
    return x * nonpad.transpose(1, 2)


def conv_stacks(sd, x, n_layers, pre="mel_encoder", fp16=False):
    """ConvStacks.forward, pe.py:98-116 (norm 'gn', kernel 5, res): in_proj, x += relu(GroupNorm(conv(x))), out_proj"""
    r = _round(fp16)
    x = F.linear(r(x), r(sd[f"{pre}.in_proj.weight"]), sd[f"{pre}.in_proj.bias"]).transpose(1, -1)
    C = x.shape[1]
    for i in range(n_layers):
        p = f"{pre}.conv.{i}"
        y = F.conv1d(r(x), r(sd[f"{p}.conv.conv.weight"]), sd[f"{p}.conv.conv.bias"], padding=2)   # ConvNorm, common_layers.py:41-59
        y = F.group_norm(y, C // 16, sd[f"{p}.norm.weight"], sd[f"{p}.norm.bias"], 1e-5)     # pe.py:54, :68-75
        x = x + F.relu(y)
    return F.linear(r(x.transpose(1, -1)), r(sd[f"{pre}.out_proj.weight"]), sd[f"{pre}.out_proj.bias"])


def sinusoidal_table(num, dim, padding_idx=0, dtype=torch.float):
    """SinusoidalPositionalEmbedding.get_embedding, common_layers.py:105-122 (the reference's table is fp32; a float64
    ``dtype`` gives a reference-precision table)"""
    half = dim // 2
    emb = math.log(10000) / (half - 1)
    emb = torch.exp(torch.arange(half, dtype=dtype) * -emb)
    emb = torch.arange(num, dtype=dtype).unsqueeze(1) * emb.unsqueeze(0)
    emb = torch.cat([torch.sin(emb), torch.cos(emb)], dim=1).view(num, -1)
    if dim % 2 == 1:
        emb = torch.cat([emb, torch.zeros(num, 1, dtype=dtype)], dim=1)
    emb[padding_idx, :] = 0
    return emb


def make_positions(x, padding_idx=0):
    """utils/__init__.py:145-157"""
    mask = x.ne(padding_idx).int()
    return (torch.cumsum(mask, dim=1).type_as(mask) * mask).long() + padding_idx


def pitch_predictor(sd, xs, hp, pre="pitch_predictor", table=None, fp16=False):
    """PitchPredictor.forward, tts_modules.py:222-235 (dropout = identity).  ``table``: the module's cached
    sinusoidal table (common_layers.py:98-102, init_size 4096), or None to build it here (in float64 for a float64 xs)."""
    r = _round(fp16)
    H = xs.shape[-1]
    k = int(hp['predictor_kernel'])
    T = xs.shape[1]
    if table is None or table.shape[0] < 1 + T:                    # common_layers.py:127-135
        table = sinusoidal_table(max(4096, 0 + 1 + T), H, dtype=torch.float64 if xs.dtype == torch.float64 else torch.float)
    table = table.to(xs)
    pos = make_positions(xs[..., 0])
    xs = xs + sd[f"{pre}.pos_embed_alpha"] * table.index_select(0, pos.view(-1)).view(xs.shape[0], T, -1)
    xs = xs.transpose(1, -1)
    pad = ((k - 1) // 2, (k - 1) // 2) if hp['ffn_padding'] == 'SAME' else (k - 1, 0)
    for i in range(5):
        p = f"{pre}.conv.{i}"
        xs = F.relu(F.conv1d(F.pad(r(xs), pad), r(sd[f"{p}.1.weight"]), sd[f"{p}.1.bias"]))
        xs = F.layer_norm(xs.transpose(1, -1), (xs.shape[1],), sd[f"{p}.3.weight"], sd[f"{p}.3.bias"], 1e-12).transpose(1, -1)
    return F.linear(xs.transpose(1, -1), sd[f"{pre}.linear.weight"], sd[f"{pre}.linear.bias"])


def denorm_f0(f0, uv, hp, pitch_padding=None):
    """utils/pitch_utils.py:63-76 (min / max unused by the pitch extractor)"""
    if hp['pitch_norm'] == 'standard':
        f0 = f0 * hp['f0_std'] + hp['f0_mean']
    if hp['pitch_norm'] == 'log':
        f0 = 2 ** f0
    if uv is not None and hp['use_uv']:
        f0[uv > 0] = 0
    if pitch_padding is not None:
        f0[pitch_padding] = 0
    return f0


def pitch_extractor(sd, mel, hp, conv_layers=2, table=None, fp16=False):
    """PitchExtractor.forward, pe.py:135-149: mel [B, T, 80] -> (pitch_pred [B, T, 2], f0_denorm_pred [B, T]).
    fp16=True: the input and weight of every conv and linear rounded to fp16, as the dsx kernels round them; the
    normalisations, the position term, the head Linear(P, 2) and every sum stay in mel's dtype."""
    h = prenet(sd, mel, fp16=fp16)
    if conv_layers > 0:
        h = conv_stacks(sd, h, conv_layers, fp16=fp16)
    pitch_pred = pitch_predictor(sd, h, hp, table=table, fp16=fp16)
    use_uv = hp['pitch_type'] == 'frame' and hp['use_uv']
    f0 = denorm_f0(pitch_pred[:, :, 0], (pitch_pred[:, :, 1] > 0) if use_uv else None, hp,
                   pitch_padding=padding_mask(mel))
    return pitch_pred, f0


def random_state_dict(sd, seed, log2_f0=math.log2(200.0)):
    """Seeded values for the parameters a fresh module leaves at trivial values (BatchNorm running stats and affine,
    GroupNorm / LayerNorm affine, pos_embed_alpha) and the head bias (bias[0] ~ log2 200 Hz, so f0 is realistic and the
    uv logits straddle 0).  Convolution and linear weights are kept."""
    g = torch.Generator().manual_seed(seed)
    out = {k: v.detach().clone() for k, v in sd.items()}
    for k, v in out.items():
        if v.dtype != torch.float32:
            continue
        if k.endswith("running_mean"):
            out[k] = torch.randn(v.shape, generator=g) * 0.2
        elif k.endswith("running_var"):
            out[k] = torch.rand(v.shape, generator=g) * 0.8 + 0.4
        elif re.search(r"(layers\.\d+\.2|conv\.\d+\.norm|conv\.\d+\.3)\.(weight|bias)$", k):
            out[k] = (1.0 + 0.2 * torch.randn(v.shape, generator=g)) if k.endswith("weight") else 0.1 * torch.randn(v.shape, generator=g)
        elif k.endswith("pos_embed_alpha"):
            out[k] = torch.tensor([0.5 + torch.rand(1, generator=g).item()])
        elif k.endswith("_float_tensor"):            # torch.FloatTensor(1): uninitialised, only carries dtype / device
            out[k] = torch.zeros_like(v)
    lb = out["pitch_predictor.linear.bias"]
    out["pitch_predictor.linear.bias"] = torch.tensor([log2_f0, 0.0], dtype=lb.dtype) + 0.05 * torch.randn(2, generator=g)
    return out


def flops_per_frame(H=256, P=256, k=5, conv_layers=2):
    """multiply-adds x 2 of the convs and linears per mel frame"""
    mac = 80 * H * 5 + 2 * H * H * 5 + H * H                     # prenet
    if conv_layers:
        mac += 2 * H * H + conv_layers * H * H * 5                 # mel_encoder
    mac += H * P * k + 4 * P * P * k + 2 * P                      # pitch predictor
    return 2 * mac
