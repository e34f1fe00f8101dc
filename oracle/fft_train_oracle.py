"""TEST INFRASTRUCTURE ONLY -- the reference's FFT diffusion denoiser (usr/diff/candidate_decoder.py:50-100) in training
mode, as differentiable fp32 torch with the dropout masks of its FFTBlocks stack given: oracle.fft_oracle's entry
(input_projection, the step-embedding MLP, get_decode_inp), oracle.fs2dec_train_oracle.decoder_train (``masks`` as there:
1 + 3 L keep masks [B, T, n] in site order) and get_mel_out.  The entry has no dropout of its own.
oracle/gen_golden_fft_train.py pins it to the reference, gradients included."""
import torch.nn.functional as F

from oracle.fft_oracle import _p, decode_inp
from oracle.fs2dec_train_oracle import decoder_train


def forward_train(sd, spec, t, cond, hp, masks, p, layer_input=None):
    """FFT.forward(spec [B, 1, 80, T], t [B], cond [B, H, T]) in training -> eps [B, 1, 80, T]; ``layer_input`` as in
    decoder_train"""
    x = decoder_train(sd, decode_inp(sd, spec, t, cond, hp), hp, masks, p, layer_input)
    return F.linear(x, _p(sd["get_mel_out.weight"]), sd["get_mel_out.bias"]).permute([0, 2, 1])[:, None, :, :]
