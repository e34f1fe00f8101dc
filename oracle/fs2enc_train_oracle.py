"""TEST INFRASTRUCTURE ONLY -- the reference's FastSpeech2 encoder (FastspeechEncoder / FastspeechMIDIEncoder,
modules/fastspeech/tts_modules.py:310-347, modules/diffsinger_midi/fs2.py:11-36) in training mode, as differentiable fp32
torch with the dropout masks given: ``masks[s]`` ([B, T, n] bool) is the keep mask of dropout site s (0 after the
embedding and the position term; per layer i, 1 + 3 i after out_proj, 2 + 3 i after the FFN activation, 3 + 3 i after
ffn_2), the decoder step's sites.  The entry is oracle.fs2enc_oracle.embedding, the layers those of
oracle.fs2dec_train_oracle.decoder_train in the reference's [T, B, C] layout and op order, with the padding mask from the
tokens (txt_tokens == 0), not from all-zero rows: midi_dur_layer's bias and the position terms make padding rows of x
non-zero.  oracle/gen_golden_fs2enc_train.py pins it bit for bit to the reference, gradients included."""
import torch
import torch.nn.functional as F

from oracle.fs2dec_oracle import LN_EPS
from oracle.fs2dec_train_oracle import _ffn, dropout
from oracle.fs2enc_oracle import REL_MAX_LEN, embedding, stack_hp


def encoder_train(sd, tokens, hp, masks, p, addends=(), rel_len=REL_MAX_LEN):
    """tokens [B, T] (0 = padding), addends: midi_embedding, midi_dur_embedding, slur_embedding ([B, T, H] or 0) for the
    MIDI encoder -> [B, T, H].  sd: the encoder's state dict (layers.*, layer_norm.*, embed_tokens.weight)."""
    H, heads, shp = int(hp['hidden_size']), int(hp['num_heads']), stack_hp(hp)
    tb = lambda s: masks[s].transpose(0, 1)                        # [B, T, n] -> the layers' [T, B, n]
    pad = tokens.eq(0)
    x = embedding(sd, tokens, hp, addends, rel_len)
    x = dropout(x, masks[0], p)
    nonpad_TB = 1 - pad.transpose(0, 1).float()[:, :, None]       # FFTBlocks.forward, tts_modules.py:288-296
    x = x.transpose(0, 1) * nonpad_TB
    keep = (1 - pad.float()).transpose(0, 1)[..., None]
    for i in range(int(hp['enc_layers'])):
        pre = f"layers.{i}.op."
        residual = x
        y = F.layer_norm(x, (H,), sd[pre + "layer_norm1.weight"], sd[pre + "layer_norm1.bias"], LN_EPS)
        y, _ = F.multi_head_attention_forward(y, y, y, H, heads, sd[pre + "self_attn.in_proj_weight"], None, None, None,
                                              False, 0.0, sd[pre + "self_attn.out_proj.weight"], None, training=True,
                                              key_padding_mask=pad, need_weights=True, attn_mask=None)
        x = (residual + dropout(y, tb(1 + 3 * i), p)) * keep
        residual = x
        y = F.layer_norm(x, (H,), sd[pre + "layer_norm2.weight"], sd[pre + "layer_norm2.bias"], LN_EPS)
        x = (residual + dropout(_ffn(sd, shp, i, y, tb(2 + 3 * i), p), tb(3 + 3 * i), p)) * keep
        x = x * nonpad_TB
    x = F.layer_norm(x, (H,), sd["layer_norm.weight"], sd["layer_norm.bias"], LN_EPS) * nonpad_TB
    return x.transpose(0, 1)
