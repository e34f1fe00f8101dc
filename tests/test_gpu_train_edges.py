"""GPU: the three training steps -- the FastSpeech2 decoder (dsx_fs2dec_train_*), the FFT denoiser (dsx_fft_train_*) and
DiffNet (dsx_train_*) -- at the edges of the configurations their *_create functions accept, against float64 autograd
of the oracles with the step's own dropout masks, and two exact properties of their backwards.

Cases.  They put T on both sides of the 64-row blocks of the attention backward (k_attn_bwd_kv / k_attn_bwd_q), the
64-row tiles of the conv core and the 64-frame chunks of k_wgrad (and the FFT's 128-frame column-sum partials), reach
the limits of hidden, heads, kernel, padding, layers, residual_channels and dilation_cycle_length that include/dsx.h
documents, and run batches where a tile, chunk or block straddles two utterances.  Every case has B >= 2 unless its
name says otherwise.

Measures, dsx against float64 and TF32 autograd (fp32 with TF32 matmuls and convolutions) against float64, per tensor:
  rel    ||a - r|| / ||r||;
  frame  for out, d_x, eps and d_cond: the worst non-padding frame's ||a - r|| over the RMS of ||r_frame|| over the
         non-padding frames (over the largest ||r_frame|| for the 64-layer stack, whose frames span a wide range);
  row    for matrices: the worst output row's ||a - r|| over the RMS row norm; for conv weights with k > 1 (ffn_1,
         DiffNet's dilated_conv) the worst tap slice w[:, :, j] over the RMS tap-slice norm.
Vectors get rel only.  The one scalar, pos_embed_alpha, is held to 5e-2 only, as in test_gpu_fft_train.py: its
gradient is one sum over every frame with cancellation, so its relative error is not bounded by per-element rounding.
A case's bound for a measure holds the worst tensor.

Bounds.  BOUNDS[(step, case)] is 3x the worst TF32 error of that measure measured on an H100 (80 GB HBM3, 700 W power
limit), floored at 2^-10 for rel (one fp16 rounding of each GEMM operand; at the smallest sizes cuBLAS runs autograd's
matmuls without tensor cores, so TF32's error there says nothing about 10-bit rounding) and at 2^-8 for frame and row
(a worst frame or row of n is a maximum over n values near rel, about 2-4x it on these cases), and capped at 5e-2.
DiffNet's frame and row bounds are the exception: 2x TF32, uncapped.  Its gradients pass through ReLUs (after
input_projection and skip_projection) whose masks flip wherever a pre-activation lies within rounding of 0, and a flip
changes a unit's gradient by its whole size, so the error goes as the square root of the rounding: on the CPU a 1e-3
relative perturbation of the weights moves float64 DiffNet's d_cond by 3e-2 (rel) and 0.16 (worst frame).  TF32 and
dsx show the same 0.1-0.26 worst frame there; rel still holds DiffNet to 5e-2.  The ReLU decoder case (left_k4) shows
the same effect within the cap.  Measured on that H100, dsx / TF32 / bound:

    step    case                    rel: dsx / TF32 / bound      frame: dsx / TF32 / bound    row: dsx / TF32 / bound
    fs2     H192_h3_T63             6.2e-04 / 5.7e-04 / 1.8e-03  3.0e-04 / 2.9e-04 / 4.0e-03  2.4e-03 / 2.3e-03 / 7.0e-03
    fs2     H192_h3_T64             5.9e-04 / 8.6e-04 / 2.6e-03  2.9e-04 / 2.8e-04 / 4.0e-03  2.2e-03 / 1.8e-03 / 5.5e-03
    fs2     H192_h3_T65             5.6e-04 / 6.0e-04 / 1.9e-03  2.8e-04 / 2.8e-04 / 4.0e-03  2.0e-03 / 1.9e-03 / 5.9e-03
    fs2     H192_h3_T128            6.1e-04 / 8.7e-04 / 2.7e-03  2.8e-04 / 2.7e-04 / 4.0e-03  2.5e-03 / 2.0e-03 / 6.0e-03
    fs2     H192_h3_T129            7.0e-04 / 8.6e-04 / 2.6e-03  2.8e-04 / 2.7e-04 / 4.0e-03  2.5e-03 / 2.6e-03 / 7.7e-03
    fs2     H128_h1_T129            5.5e-04 / 8.6e-04 / 2.6e-03  2.8e-04 / 2.6e-04 / 4.0e-03  2.2e-03 / 2.2e-03 / 6.6e-03
    fs2     H128_h2_T65             6.2e-04 / 6.1e-04 / 1.9e-03  2.9e-04 / 2.8e-04 / 4.0e-03  2.3e-03 / 2.3e-03 / 6.8e-03
    fs2     H256_h4_T65             5.6e-04 / 5.5e-04 / 1.7e-03  2.8e-04 / 2.7e-04 / 4.0e-03  2.1e-03 / 2.8e-03 / 8.3e-03
    fs2     same_k255_H64_T100      5.9e-04 / 5.6e-04 / 1.7e-03  3.3e-04 / 3.5e-04 / 4.0e-03  1.8e-03 / 1.6e-03 / 5.0e-03
    fs2     left_k2_H64_T100        8.8e-04 / 6.6e-04 / 2.0e-03  4.7e-04 / 4.6e-04 / 4.0e-03  2.0e-03 / 1.9e-03 / 5.8e-03
    fs2     left_k4_H64_T100        1.4e-02 / 2.1e-02 / 5.0e-02  1.6e-02 / 2.2e-02 / 5.0e-02  1.9e-02 / 2.6e-02 / 5.0e-02
    fs2     left_k255_H64_T100      6.4e-04 / 6.3e-04 / 1.9e-03  3.1e-04 / 3.0e-04 / 4.0e-03  2.2e-03 / 1.9e-03 / 5.8e-03
    fs2     L64_H64_T80             1.1e-03 / 1.0e-03 / 3.2e-03  6.9e-04 / 6.8e-04 / 4.0e-03  3.9e-03 / 3.9e-03 / 1.2e-02
    fs2     shipped_p05_T300        5.7e-04 / 8.5e-04 / 2.6e-03  2.4e-04 / 2.5e-04 / 4.0e-03  2.2e-03 / 2.1e-03 / 6.2e-03
    fs2     shipped_p09_T300        7.3e-04 / 8.8e-04 / 2.7e-03  5.8e-04 / 5.4e-04 / 4.0e-03  2.3e-03 / 2.4e-03 / 7.2e-03
    fs2     interior_pad_60_70      6.3e-04 / 8.6e-04 / 2.6e-03  2.5e-04 / 2.5e-04 / 4.0e-03  2.5e-03 / 2.6e-03 / 7.8e-03
    fs2     channel0_zero           6.3e-04 / 8.6e-04 / 2.6e-03  2.5e-04 / 2.4e-04 / 4.0e-03  2.6e-03 / 2.5e-03 / 7.4e-03
    fs2     all_padding_utterance   6.2e-04 / 6.1e-04 / 1.9e-03  2.6e-04 / 2.5e-04 / 4.0e-03  2.6e-03 / 2.5e-03 / 7.7e-03
    fs2     B300_T3                 7.3e-04 / 9.1e-04 / 2.8e-03  7.9e-04 / 6.0e-04 / 4.0e-03  1.7e-03 / 1.8e-03 / 5.5e-03
    fs2     B1_T1_p05               6.4e-04 / 3.5e-04 / 1.1e-03  4.4e-04 / 2.6e-05 / 4.0e-03  3.2e-03 / 1.2e-03 / 4.0e-03
    fft     H192_h3_dim16           6.9e-04 / 9.5e-04 / 2.9e-03  5.9e-04 / 6.1e-04 / 4.0e-03  3.0e-03 / 3.2e-03 / 9.6e-03
    fft     H192_h3_dim48           7.5e-04 / 9.6e-04 / 2.9e-03  6.2e-04 / 6.4e-04 / 4.0e-03  3.1e-03 / 2.8e-03 / 8.5e-03
    fft     H192_h3_dim1024         7.3e-04 / 1.0e-03 / 3.2e-03  6.2e-04 / 7.4e-04 / 4.0e-03  2.8e-03 / 3.9e-03 / 1.2e-02
    fft     T63                     6.4e-04 / 7.2e-04 / 2.2e-03  6.6e-04 / 6.5e-04 / 4.0e-03  2.5e-03 / 2.8e-03 / 8.5e-03
    fft     T65                     7.3e-04 / 8.2e-04 / 2.5e-03  6.1e-04 / 6.0e-04 / 4.0e-03  3.1e-03 / 3.2e-03 / 9.7e-03
    fft     T127                    6.8e-04 / 1.0e-03 / 3.0e-03  6.3e-04 / 6.6e-04 / 4.0e-03  3.7e-03 / 3.5e-03 / 1.1e-02
    fft     T128                    6.4e-04 / 9.9e-04 / 3.0e-03  6.1e-04 / 6.8e-04 / 4.0e-03  3.0e-03 / 2.8e-03 / 8.5e-03
    fft     T129                    7.3e-04 / 9.9e-04 / 3.0e-03  6.0e-04 / 6.4e-04 / 4.0e-03  2.9e-03 / 2.5e-03 / 7.7e-03
    fft     t_0_99_repeated         6.8e-04 / 9.7e-04 / 3.0e-03  6.0e-04 / 6.3e-04 / 4.0e-03  3.4e-03 / 3.1e-03 / 9.3e-03
    fft     B300_T3                 7.3e-04 / 1.0e-03 / 3.1e-03  1.0e-03 / 9.6e-04 / 4.0e-03  2.5e-03 / 2.4e-03 / 7.3e-03
    fft     left_k255_H64           8.6e-04 / 8.9e-04 / 2.7e-03  7.0e-04 / 7.9e-04 / 4.0e-03  2.9e-03 / 3.2e-03 / 9.6e-03
    diffnet L1_c1_B1_T1             8.4e-04 / 3.9e-04 / 1.2e-03  7.2e-04 / 3.2e-04 / 4.0e-03  4.1e-03 / 2.1e-03 / 4.3e-03
    diffnet L1_c1_T65               2.9e-02 / 3.2e-02 / 5.0e-02  1.4e-01 / 1.4e-01 / 2.8e-01  2.1e-01 / 2.1e-01 / 4.3e-01
    diffnet L3_T63                  2.4e-02 / 2.4e-02 / 5.0e-02  1.2e-01 / 1.0e-01 / 2.1e-01  2.1e-01 / 2.1e-01 / 4.2e-01
    diffnet L3_T64                  1.6e-02 / 1.5e-02 / 4.5e-02  1.1e-01 / 9.5e-02 / 2.0e-01  1.4e-01 / 1.4e-01 / 2.9e-01
    diffnet L3_T65                  2.2e-02 / 2.2e-02 / 5.0e-02  1.3e-01 / 1.3e-01 / 2.6e-01  1.9e-01 / 1.9e-01 / 3.9e-01
    diffnet L3_T127                 2.5e-02 / 2.5e-02 / 5.0e-02  2.3e-01 / 2.3e-01 / 4.7e-01  2.5e-01 / 2.5e-01 / 5.0e-01
    diffnet L3_T129                 2.6e-02 / 2.4e-02 / 5.0e-02  1.7e-01 / 1.6e-01 / 3.3e-01  1.8e-01 / 1.8e-01 / 3.6e-01
    diffnet L12_c12_T129            2.6e-02 / 3.3e-02 / 5.0e-02  1.5e-01 / 2.1e-01 / 4.2e-01  1.9e-01 / 2.2e-01 / 4.5e-01
    diffnet L12_c12_T1000           2.6e-02 / 2.1e-02 / 5.0e-02  2.2e-01 / 1.9e-01 / 3.8e-01  8.5e-02 / 7.9e-02 / 1.6e-01
    diffnet L24_c24_T40             8.4e-03 / 9.7e-03 / 3.0e-02  4.8e-02 / 6.2e-02 / 1.3e-01  1.0e-01 / 1.1e-01 / 2.3e-01
    diffnet B300_T3                 2.4e-02 / 2.0e-02 / 5.0e-02  2.6e-01 / 2.6e-01 / 5.2e-01  1.4e-01 / 1.4e-01 / 2.8e-01
    diffnet L3_T65_contiguous_cond  2.2e-02 / 2.2e-02 / 5.0e-02  1.3e-01 / 1.3e-01 / 2.6e-01  1.9e-01 / 1.9e-01 / 3.9e-01

The exact properties: a zero cotangent on one utterance gives exactly zero d_x / d_cond rows there (every step, with and
without dropout, at T = 65 and 129 with B = 3, so partial tiles and chunks straddle the utterance); and permuting the
utterances of a batch (t with them) permutes out / eps and d_x / d_cond bit for bit at p = 0, while the weight
gradients, which sum over the batch in another order, stay within the case's bounds."""
import contextlib
import copy

import numpy as np
import pytest
import torch

from oracle import fft_oracle as FO
from oracle import fs2dec_oracle as D
from oracle.fft_train_oracle import forward_train
from oracle.fs2dec_train_oracle import decoder_train

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
CAP = 5e-2
FLOOR = dict(rel=2.0 ** -10, frame=2.0 ** -8, row=2.0 ** -8)
SEED = 11


# ---- the cases -----------------------------------------------------------------------------------------------------
def fs2_hp(H=256, heads=2, k=9, padding='SAME', L=4, p=0.1, act='gelu'):
    return dict(hidden_size=H, dec_layers=L, dec_ffn_kernel_size=k, num_heads=heads, ffn_padding=padding, ffn_act=act,
                dropout=p)


def fft_hp(H=256, heads=2, k=9, padding='SAME', L=4, dim=256, p=0.1, act='gelu'):
    return dict(fs2_hp(H, heads, k, padding, L, p, act), residual_channels=dim, audio_num_mel_bins=80, keep_bins=80)


# B, T; tail: utterance 1 is padding from frame T - T // 4 on; pad: frames [a, b) of every utterance are padding;
# ch0: (utterance, frame) pairs whose channel 0 is exactly 0 (a position make_positions skips); empty: an utterance that
# is padding throughout; lengths: utterance b is padding from frame lengths[b % len] on
FS2 = {
    "H192_h3_T63": dict(hp=fs2_hp(192, 3), B=3, T=63, tail=True),
    "H192_h3_T64": dict(hp=fs2_hp(192, 3), B=3, T=64, tail=True),
    "H192_h3_T65": dict(hp=fs2_hp(192, 3), B=3, T=65, tail=True),
    "H192_h3_T128": dict(hp=fs2_hp(192, 3), B=3, T=128, tail=True),
    "H192_h3_T129": dict(hp=fs2_hp(192, 3), B=3, T=129, tail=True),
    "H128_h1_T129": dict(hp=fs2_hp(128, 1), B=3, T=129, tail=True),
    "H128_h2_T65": dict(hp=fs2_hp(128, 2), B=3, T=65, tail=True),
    "H256_h4_T65": dict(hp=fs2_hp(256, 4), B=3, T=65, tail=True),
    "same_k255_H64_T100": dict(hp=fs2_hp(64, 1, 255), B=2, T=100, tail=True),
    "left_k2_H64_T100": dict(hp=fs2_hp(64, 1, 2, 'LEFT'), B=2, T=100, tail=True),
    "left_k4_H64_T100": dict(hp=fs2_hp(64, 1, 4, 'LEFT', act='relu'), B=2, T=100, tail=True),
    "left_k255_H64_T100": dict(hp=fs2_hp(64, 1, 255, 'LEFT'), B=2, T=100, tail=True),
    "L64_H64_T80": dict(hp=fs2_hp(64, 1, L=64), B=2, T=80, tail=True, peak=True),
    "shipped_p05_T300": dict(hp=fs2_hp(p=0.5), B=2, T=300, tail=True),
    "shipped_p09_T300": dict(hp=fs2_hp(p=0.9), B=2, T=300, tail=True),
    "interior_pad_60_70": dict(hp=fs2_hp(), B=2, T=150, pad=(60, 71)),
    "channel0_zero": dict(hp=fs2_hp(), B=2, T=150, ch0=[(0, 0), (0, 1), (0, 63), (0, 64), (0, 149), (1, 70)]),
    "all_padding_utterance": dict(hp=fs2_hp(), B=3, T=100, empty=1),
    "B300_T3": dict(hp=fs2_hp(), B=300, T=3, lengths=[3, 1, 2]),
    "B1_T1_p05": dict(hp=fs2_hp(p=0.5), B=1, T=1),
}

# t: the diffusion steps, cycled over the batch (default: seeded draws in [0, 100))
FFT = {
    "H192_h3_dim16": dict(hp=fft_hp(192, 3, dim=16), B=3, T=90),
    "H192_h3_dim48": dict(hp=fft_hp(192, 3, dim=48), B=3, T=90),
    "H192_h3_dim1024": dict(hp=fft_hp(192, 3, dim=1024), B=3, T=90),
    "T63": dict(hp=fft_hp(), B=3, T=63),
    "T65": dict(hp=fft_hp(), B=3, T=65),
    "T127": dict(hp=fft_hp(), B=3, T=127),
    "T128": dict(hp=fft_hp(), B=3, T=128),
    "T129": dict(hp=fft_hp(), B=3, T=129),
    "t_0_99_repeated": dict(hp=fft_hp(), B=5, T=100, t=[0, 99, 99, 0, 0]),
    "B300_T3": dict(hp=fft_hp(), B=300, T=3),
    "left_k255_H64": dict(hp=fft_hp(64, 1, 255, 'LEFT'), B=2, T=100),
}

# L, cycle: residual_layers, dilation_cycle_length (dilation 2^(l % cycle)); contiguous: cond as a contiguous [B, H, T]
# instead of the reference's strided view of a [B, T, H] tensor
DIFFNET = {
    "L1_c1_B1_T1": dict(L=1, cycle=1, B=1, T=1),
    "L1_c1_T65": dict(L=1, cycle=1, B=2, T=65),
    "L3_T63": dict(L=3, cycle=3, B=3, T=63),
    "L3_T64": dict(L=3, cycle=3, B=3, T=64),
    "L3_T65": dict(L=3, cycle=3, B=3, T=65),
    "L3_T127": dict(L=3, cycle=3, B=3, T=127),
    "L3_T129": dict(L=3, cycle=3, B=3, T=129),
    "L12_c12_T129": dict(L=12, cycle=12, B=2, T=129),
    "L12_c12_T1000": dict(L=12, cycle=12, B=2, T=1000),
    "L24_c24_T40": dict(L=24, cycle=24, B=2, T=40),
    "B300_T3": dict(L=3, cycle=3, B=300, T=3),
    "L3_T65_contiguous_cond": dict(L=3, cycle=3, B=3, T=65, contiguous=True),
}

CASES = {"fs2": FS2, "fft": FFT, "diffnet": DIFFNET}


def fs2_case(name, seed=SEED):
    """(hp, state dict, x [B, T, H], cotangent of out [B, T, H]) on the CPU, fp32"""
    c = FS2[name]
    hp, B, T = c["hp"], c["B"], c["T"]
    H = hp["hidden_size"]
    rs = np.random.RandomState(seed)
    x = torch.from_numpy(rs.standard_normal((B, T, H)).astype(np.float32))
    if c.get("tail") and B > 1 and T >= 4:
        x[1, T - T // 4:] = 0
    if "pad" in c:
        x[:, c["pad"][0]:c["pad"][1]] = 0
    for b, f in c.get("ch0", []):
        x[b, f, 0] = 0
    if "empty" in c:
        x[c["empty"]] = 0
    if "lengths" in c:
        for b in range(B):
            x[b, c["lengths"][b % len(c["lengths"])]:] = 0
    g = torch.from_numpy(rs.standard_normal((B, T, H)).astype(np.float32))
    return hp, D.random_state_dict(seed + 1, hp), x, g


def fft_case(name, seed=SEED):
    """(hp, state dict, spec [B, 1, 80, T], t [B], cond [B, H, T], cotangent of eps [B, 1, 80, T]) on the CPU"""
    c = FFT[name]
    hp, B, T = c["hp"], c["B"], c["T"]
    rs = np.random.RandomState(seed)
    spec = torch.from_numpy(rs.standard_normal((B, 1, 80, T)).astype(np.float32))
    t = torch.from_numpy(rs.randint(0, 100, B)).long()
    if "t" in c:
        t = torch.tensor([c["t"][b % len(c["t"])] for b in range(B)])
    cond = torch.from_numpy(rs.standard_normal((B, hp["hidden_size"], T)).astype(np.float32))
    g = torch.from_numpy(rs.standard_normal((B, 1, 80, T)).astype(np.float32))
    return hp, FO.random_state_dict(seed + 1, hp), spec, t, cond, g


def diffnet_case(name, seed=SEED):
    """(net: an fp32 CPU DiffNet with train=True, spec, t, cond [B, H, T], cotangent of eps)"""
    return diffnet_inputs(DIFFNET[name], seed)


def diffnet_inputs(c, seed=SEED):
    import diffsinger_b200 as dsx
    B, T = c["B"], c["T"]
    torch.manual_seed(seed)
    net = dsx.DiffNet(80, hparams=dict(hidden_size=256, residual_layers=c["L"], residual_channels=256,
                                       dilation_cycle_length=c["cycle"]), train=True)
    torch.nn.init.normal_(net.output_projection.weight, std=0.02)
    gen = torch.Generator().manual_seed(seed + 1)
    spec = torch.randn(B, 1, 80, T, generator=gen)
    cond = torch.randn(B, T, 256, generator=gen).transpose(1, 2)          # the reference's strided view
    if c.get("contiguous"):
        cond = cond.contiguous()
    t = torch.randint(0, 100, (B,), generator=gen)
    g = torch.randn(B, 1, 80, T, generator=gen)
    return net, spec, t, cond, g


# ---- float64 and TF32 autograd ---------------------------------------------------------------------------------------
@contextlib.contextmanager
def precision(mode):
    """"f64": float64 default dtype (the step embeddings' aranges), TF32 off; "tf32": TF32 matmuls and convolutions;
    "fp32": TF32 off"""
    old = torch.get_default_dtype(), torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.set_default_dtype(torch.float64 if mode == "f64" else torch.float32)
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = mode == "tf32"
    try:
        yield torch.float64 if mode == "f64" else torch.float32
    finally:
        torch.set_default_dtype(old[0])
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old[1], old[2]


def _leaves(sd, dev, dt):
    return {n: v.to(dev, dt).requires_grad_(True) for n, v in sd.items() if not n.endswith("_float_tensor")}


def fs2_ref(hp, sd, x, g, masks, mode, dev, layer_input=None):
    """out, d_x, {name: grad} of sum(out * g) through decoder_train in `mode`"""
    with precision(mode) as dt:
        w = _leaves(sd, dev, dt)
        xr = x.to(dev, dt).requires_grad_(True)
        out = decoder_train(w, xr, hp, [m.to(dev) for m in masks], hp["dropout"], layer_input)
        (out * g.to(dev, dt)).sum().backward()
    return out.detach(), xr.grad, {n: v.grad for n, v in w.items()}


def fft_ref(hp, sd, spec, t, cond, g, masks, mode, dev, layer_input=None):
    """eps, d_cond [B, H, T], {name: grad} of sum(eps * g) through forward_train in `mode`"""
    with precision(mode) as dt:
        w = _leaves(sd, dev, dt)
        c = cond.to(dev, dt).requires_grad_(True)
        eps = forward_train(w, spec.to(dev, dt), t.to(dev), c, hp, [m.to(dev) for m in masks], hp["dropout"],
                            layer_input)
        (eps * g.to(dev, dt)).sum().backward()
    return eps.detach(), c.grad, {n: v.grad for n, v in w.items()}


def diffnet_ref(net, spec, t, cond, g, mode, dev, layer_input=None):
    """eps, d_cond, {name: grad} of sum(eps * g) through DiffNet._forward_autograd in `mode`.  A dilated conv whose
    dilation d exceeds T runs with d = T: either way both outer taps lie wholly outside every utterance, and ATen need
    not pad by up to 2^23 frames."""
    T = spec.shape[-1]
    with precision(mode) as dt:
        m = copy.deepcopy(net).to(dev, dt)
        for layer in m.residual_layers:
            conv = layer.dilated_conv
            if conv.dilation[0] > T:
                conv.dilation, conv.padding = (T,), (T,)
        hooks = [] if layer_input is None else [
            layer.register_forward_pre_hook(lambda mod, a, i=i: (layer_input(i, a[0]),) + tuple(a[1:]))
            for i, layer in enumerate(m.residual_layers)]
        c = cond.to(dev, dt).requires_grad_(True)
        eps = m._forward_autograd(spec.to(dev, dt), t.to(dev), c)
        (eps * g.to(dev, dt)).sum().backward()
        for h in hooks:
            h.remove()
    return eps.detach(), c.grad, {n: p.grad for n, p in m.named_parameters()}


# ---- the measures --------------------------------------------------------------------------------------------------
FRAMES = {"out": "btc", "d_x": "btc", "eps": "bct", "d_cond": "bct"}


def _frames(v, layout):
    """[B, T, C] frame vectors of out / d_x ([B, T, C]), eps ([B, 1, 80, T]) or d_cond ([B, H, T])"""
    return v if layout == "btc" else v.reshape(v.shape[0], -1, v.shape[-1]).transpose(1, 2)


def measure(name, a, r, keep=None, peak=False):
    """{measure: error} of tensor `name`: a against r.  keep: [B, T] bool of the non-padding frames."""
    a, r = a.detach().double().cpu(), r.detach().double().cpu()
    d = a - r
    e = {"rel": (d.norm() / r.norm().clamp_min(1e-300)).item()}
    if name in FRAMES:
        fd, fr = (_frames(v, FRAMES[name]).norm(dim=-1) for v in (d, r))
        if keep is not None:
            fd, fr = fd[keep], fr[keep]
        scale = fr.max() if peak else fr.pow(2).mean().sqrt()
        e["frame"] = (fd.max() / scale.clamp_min(1e-300)).item()
    elif a.dim() >= 2:
        sl = (lambda v: v.permute(2, 0, 1).reshape(v.shape[2], -1)) if a.dim() == 3 and a.shape[2] > 1 else \
            (lambda v: v.reshape(v.shape[0], -1))
        nd, nr = sl(d).norm(dim=1), sl(r).norm(dim=1)
        e["row"] = (nd.max() / nr.pow(2).mean().sqrt().clamp_min(1e-300)).item()
    return e


def errors(res, ref, names, keep=None, peak=False):
    """{tensor: {measure: error}} of (primary, d_input, grads) against the same of the reference"""
    e = {names[0]: measure(names[0], res[0], ref[0], keep, peak), names[1]: measure(names[1], res[1], ref[1], keep, peak)}
    e.update({n: measure(n, res[2][n], ref[2][n]) for n in res[2]})
    return e


def worst(e):
    """{measure: (error, tensor)}: the worst tensor per measure, pos_embed_alpha aside"""
    out = {}
    for n, per in e.items():
        if n == "pos_embed_alpha":
            continue
        for m, v in per.items():
            if m not in out or not v <= out[m][0]:
                out[m] = (v, n)
    return out


# ---- the dsx steps ---------------------------------------------------------------------------------------------------
def with_seed(module, seed, fn):
    orig = module.draw_seed
    module.draw_seed = lambda: seed
    try:
        return fn()
    finally:
        module.draw_seed = orig


def fs2_dsx(hp, sd, x, g, seed=SEED):
    """out, d_x, {name: grad}, masks of one step of FastspeechDecoder under dsx_train"""
    from diffsinger_b200 import FastspeechDecoder, fs2train
    m = FastspeechDecoder(hparams=dict(hp, dsx_train=True))
    m.load_state_dict(sd, strict=True)
    m = m.train().to(DEV)
    xr = x.to(DEV).requires_grad_(True)

    def run():
        out = m(xr)
        (out * g.to(DEV)).sum().backward()
        return out
    out = with_seed(fs2train, seed, run)
    masks = m._dsx_train_step().masks(DEV, seed, hp["dropout"], x.shape[0], x.shape[1])
    return out.detach(), xr.grad, {n: p.grad for n, p in m.named_parameters()}, masks


def fft_dsx(hp, sd, spec, t, cond, g, seed=SEED):
    """eps, d_cond, {name: grad}, masks of one step of FFT under dsx_train"""
    from diffsinger_b200 import FFT as FFTModule, ffttrain
    from diffsinger_b200.fs2train import Fs2DecTrainStep
    m = FFTModule(hparams=dict(hp, dsx_train=True))
    m.load_state_dict(sd, strict=True)
    m = m.train().to(DEV)
    c = cond.to(DEV).requires_grad_(True)

    def run():
        eps = m(spec.to(DEV), t.to(DEV), c)
        (eps * g.to(DEV)).sum().backward()
        return eps
    eps = with_seed(ffttrain, seed, run)
    masks = Fs2DecTrainStep(m._fft_cfg.dec).masks(DEV, seed, hp["dropout"], spec.shape[0], spec.shape[3])
    return eps.detach(), c.grad, {n: p.grad for n, p in m.named_parameters()}, masks


def diffnet_dsx(net, spec, t, cond, g):
    m = copy.deepcopy(net).to(DEV).train()
    c = cond.to(DEV).requires_grad_(True)       # .to keeps the strided view's strides
    eps = m(spec.to(DEV), t.to(DEV), c)
    (eps * g.to(DEV)).sum().backward()
    return eps.detach(), c.grad, {n: p.grad for n, p in m.named_parameters()}


def run_case(step, name):
    """{"dsx": errors, "tf32": errors} of one case, after its exact checks (finite gradients, zero padding rows)"""
    c = CASES[step][name]
    if step == "fs2":
        hp, sd, x, g = fs2_case(name)
        out, dx, grads, masks = fs2_dsx(hp, sd, x, g)
        res = (out, dx, grads)
        pad = D.padding_mask(x).to(DEV)
        assert (dx[pad] == 0).all() and (out[pad] == 0).all()
        idx = [b for b in range(c["B"]) if b != c.get("empty")]
        if "empty" in c:                      # the reference gives NaN there: compare the batch without it
            res = (out[idx], dx[idx], grads)
        sub = lambda v: v[idx]
        refs = {mode: fs2_ref(hp, sd, sub(x), sub(g), [sub(mk) for mk in masks], mode, DEV) for mode in ("f64", "tf32")}
        keep, names = ~D.padding_mask(sub(x)), ("out", "d_x")
    elif step == "fft":
        hp, sd, spec, t, cond, g = fft_case(name)
        eps, dc, grads, masks = fft_dsx(hp, sd, spec, t, cond, g)
        res = (eps, dc, grads)
        refs = {mode: fft_ref(hp, sd, spec, t, cond, g, masks, mode, DEV) for mode in ("f64", "tf32")}
        keep, names = None, ("eps", "d_cond")
    else:
        net, spec, t, cond, g = diffnet_case(name)
        res = diffnet_dsx(net, spec, t, cond, g)
        refs = {mode: diffnet_ref(net, spec, t, cond, g, mode, DEV) for mode in ("f64", "tf32")}
        keep, names = None, ("eps", "d_cond")
    assert all(torch.isfinite(v).all() for v in (res[0], res[1], *res[2].values()))
    peak = c.get("peak", False)
    return {"dsx": errors(res, refs["f64"], names, keep, peak), "tf32": errors(refs["tf32"], refs["f64"], names, keep,
                                                                              peak)}


# ---- the bounds: 3x TF32's worst per measure on an H100, floored and capped (see the docstring) ---------------------
BOUNDS = {
    ("fs2", "H192_h3_T63"): dict(rel=1.8e-03, frame=4.0e-03, row=7.0e-03),
    ("fs2", "H192_h3_T64"): dict(rel=2.6e-03, frame=4.0e-03, row=5.5e-03),
    ("fs2", "H192_h3_T65"): dict(rel=1.9e-03, frame=4.0e-03, row=5.9e-03),
    ("fs2", "H192_h3_T128"): dict(rel=2.7e-03, frame=4.0e-03, row=6.0e-03),
    ("fs2", "H192_h3_T129"): dict(rel=2.6e-03, frame=4.0e-03, row=7.7e-03),
    ("fs2", "H128_h1_T129"): dict(rel=2.6e-03, frame=4.0e-03, row=6.6e-03),
    ("fs2", "H128_h2_T65"): dict(rel=1.9e-03, frame=4.0e-03, row=6.8e-03),
    ("fs2", "H256_h4_T65"): dict(rel=1.7e-03, frame=4.0e-03, row=8.3e-03),
    ("fs2", "same_k255_H64_T100"): dict(rel=1.7e-03, frame=4.0e-03, row=5.0e-03),
    ("fs2", "left_k2_H64_T100"): dict(rel=2.0e-03, frame=4.0e-03, row=5.8e-03),
    ("fs2", "left_k4_H64_T100"): dict(rel=5.0e-02, frame=5.0e-02, row=5.0e-02),
    ("fs2", "left_k255_H64_T100"): dict(rel=1.9e-03, frame=4.0e-03, row=5.8e-03),
    ("fs2", "L64_H64_T80"): dict(rel=3.2e-03, frame=4.0e-03, row=1.2e-02),
    ("fs2", "shipped_p05_T300"): dict(rel=2.6e-03, frame=4.0e-03, row=6.2e-03),
    ("fs2", "shipped_p09_T300"): dict(rel=2.7e-03, frame=4.0e-03, row=7.2e-03),
    ("fs2", "interior_pad_60_70"): dict(rel=2.6e-03, frame=4.0e-03, row=7.8e-03),
    ("fs2", "channel0_zero"): dict(rel=2.6e-03, frame=4.0e-03, row=7.4e-03),
    ("fs2", "all_padding_utterance"): dict(rel=1.9e-03, frame=4.0e-03, row=7.7e-03),
    ("fs2", "B300_T3"): dict(rel=2.8e-03, frame=4.0e-03, row=5.5e-03),
    ("fs2", "B1_T1_p05"): dict(rel=1.1e-03, frame=4.0e-03, row=4.0e-03),
    ("fft", "H192_h3_dim16"): dict(rel=2.9e-03, frame=4.0e-03, row=9.6e-03),
    ("fft", "H192_h3_dim48"): dict(rel=2.9e-03, frame=4.0e-03, row=8.5e-03),
    ("fft", "H192_h3_dim1024"): dict(rel=3.2e-03, frame=4.0e-03, row=1.2e-02),
    ("fft", "T63"): dict(rel=2.2e-03, frame=4.0e-03, row=8.5e-03),
    ("fft", "T65"): dict(rel=2.5e-03, frame=4.0e-03, row=9.7e-03),
    ("fft", "T127"): dict(rel=3.0e-03, frame=4.0e-03, row=1.1e-02),
    ("fft", "T128"): dict(rel=3.0e-03, frame=4.0e-03, row=8.5e-03),
    ("fft", "T129"): dict(rel=3.0e-03, frame=4.0e-03, row=7.7e-03),
    ("fft", "t_0_99_repeated"): dict(rel=3.0e-03, frame=4.0e-03, row=9.3e-03),
    ("fft", "B300_T3"): dict(rel=3.1e-03, frame=4.0e-03, row=7.3e-03),
    ("fft", "left_k255_H64"): dict(rel=2.7e-03, frame=4.0e-03, row=9.6e-03),
    ("diffnet", "L1_c1_B1_T1"): dict(rel=1.2e-03, frame=4.0e-03, row=4.3e-03),
    ("diffnet", "L1_c1_T65"): dict(rel=5.0e-02, frame=2.8e-01, row=4.3e-01),
    ("diffnet", "L3_T63"): dict(rel=5.0e-02, frame=2.1e-01, row=4.2e-01),
    ("diffnet", "L3_T64"): dict(rel=4.5e-02, frame=2.0e-01, row=2.9e-01),
    ("diffnet", "L3_T65"): dict(rel=5.0e-02, frame=2.6e-01, row=3.9e-01),
    ("diffnet", "L3_T127"): dict(rel=5.0e-02, frame=4.7e-01, row=5.0e-01),
    ("diffnet", "L3_T129"): dict(rel=5.0e-02, frame=3.3e-01, row=3.6e-01),
    ("diffnet", "L12_c12_T129"): dict(rel=5.0e-02, frame=4.2e-01, row=4.5e-01),
    ("diffnet", "L12_c12_T1000"): dict(rel=5.0e-02, frame=3.8e-01, row=1.6e-01),
    ("diffnet", "L24_c24_T40"): dict(rel=3.0e-02, frame=1.3e-01, row=2.3e-01),
    ("diffnet", "B300_T3"): dict(rel=5.0e-02, frame=5.2e-01, row=2.8e-01),
    ("diffnet", "L3_T65_contiguous_cond"): dict(rel=5.0e-02, frame=2.6e-01, row=3.9e-01),
}


def report(step, name, e):
    wd, wt = worst(e["dsx"]), worst(e["tf32"])
    b = BOUNDS.get((step, name), {})
    for m in ("rel", "frame", "row"):
        print(f"  {step:8s} {name:26s} {m:6s} dsx {wd[m][0]:.2e} ({wd[m][1]}) TF32 {wt[m][0]:.2e} ({wt[m][1]}) "
              f"bound {b.get(m, float('nan')):.1e} ratio {wd[m][0] / max(wt[m][0], 1e-300):.2f}")
    if "pos_embed_alpha" in e["dsx"]:
        print(f"  {step:8s} {name:26s} pos_embed_alpha rel dsx {e['dsx']['pos_embed_alpha']['rel']:.2e} "
              f"TF32 {e['tf32']['pos_embed_alpha']['rel']:.2e}")
    return wd


def check(step, name, e):
    wd = report(step, name, e)
    assert all(np.isfinite(v) for per in e["dsx"].values() for v in per.values()), e["dsx"]
    for m, bound in BOUNDS[step, name].items():
        assert wd[m][0] <= bound, (m, wd[m], bound)
    if "pos_embed_alpha" in e["dsx"]:
        assert e["dsx"]["pos_embed_alpha"]["rel"] <= CAP


@pytest.mark.parametrize("case", list(FS2))
def test_fs2_decoder_step(lib_built, case):
    check("fs2", case, run_case("fs2", case))


@pytest.mark.parametrize("case", list(FFT))
def test_fft_step(lib_built, case):
    check("fft", case, run_case("fft", case))


@pytest.mark.parametrize("case", list(DIFFNET))
def test_diffnet_step(lib_built, case):
    check("diffnet", case, run_case("diffnet", case))


def test_all_padding_utterance_gets_zero(lib_built):
    """The all-padding utterance of its case: out and d_x exactly 0 there (the kernels' softmax over no key gives 0)."""
    hp, sd, x, g = fs2_case("all_padding_utterance")
    out, dx, grads, _ = fs2_dsx(hp, sd, x, g)
    b = FS2["all_padding_utterance"]["empty"]
    assert (out[b] == 0).all() and (dx[b] == 0).all()
    assert all(torch.isfinite(v).all() for v in grads.values())


# ---- exact properties ----------------------------------------------------------------------------------------------
def _step_run(step, T, p, perm=None, zero=None):
    """One dsx step of a B = 3 batch of `step`'s shipped configuration (L = 12 and cycle 12 for DiffNet, so taps reach
    far past T); perm permutes the utterances (t with them), zero zeroes the cotangent of one utterance.
    -> primary output, d_input, grads"""
    B = 3
    order = list(range(B)) if perm is None else perm
    if step == "fs2":
        hp = fs2_hp(p=p)
        sd = D.random_state_dict(SEED + 1, hp)
        x = D.fixture_input(SEED, B, T, 256, tail=T - T // 4)
        g = torch.from_numpy(np.random.RandomState(SEED + 2).standard_normal((B, T, 256)).astype(np.float32))
        if zero is not None:
            g[zero] = 0
        return fs2_dsx(hp, sd, x[order], g[order])[:3]
    if step == "fft":
        hp = fft_hp(p=p)
        rs = np.random.RandomState(SEED)
        spec = torch.from_numpy(rs.standard_normal((B, 1, 80, T)).astype(np.float32))
        cond = torch.from_numpy(rs.standard_normal((B, 256, T)).astype(np.float32))
        g = torch.from_numpy(rs.standard_normal((B, 1, 80, T)).astype(np.float32))
        t = torch.tensor([7, 99, 0])
        if zero is not None:
            g[zero] = 0
        return fft_dsx(hp, FO.random_state_dict(SEED + 1, hp), spec[order], t[order], cond[order], g[order])[:3]
    net, spec, t, cond, g = diffnet_inputs(dict(L=12, cycle=12, B=B, T=T))
    if zero is not None:
        g[zero] = 0
    return diffnet_dsx(net, spec[order], t[order], cond[order], g[order])


@pytest.mark.parametrize("T", [65, 129])
@pytest.mark.parametrize("step,p", [("fs2", 0.0), ("fs2", 0.1), ("fft", 0.0), ("fft", 0.1), ("diffnet", 0.0)])
def test_utterance_isolation(lib_built, step, p, T):
    """A zero cotangent on utterance 1 of 3: its d_x / d_cond rows are exactly 0, the other utterances' are not."""
    _, d, _ = _step_run(step, T, p, zero=1)
    assert (d[1] == 0).all()
    assert (d[0] != 0).any() and (d[2] != 0).any()


PERM_CASE = {"fs2": "H192_h3_T65", "fft": "T65", "diffnet": "L3_T65"}


@pytest.mark.parametrize("step", ["fs2", "fft", "diffnet"])
def test_permutation_equivariance(lib_built, step):
    """p = 0: permuting the utterances permutes out / eps and d_x / d_cond bit for bit (the gradient scales come from a
    batch amax, which the permutation does not change).  The weight gradients sum over the batch in another order:
    they are held to the parity bounds of PERM_CASE[step] against float64 autograd."""
    name = PERM_CASE[step]
    perm = [2, 0, 1]
    c = CASES[step][name]
    if step == "fs2":
        hp, sd, x, g = fs2_case(name)
        hp = dict(hp, dropout=0.0)
        a, b = fs2_dsx(hp, sd, x, g)[:3], fs2_dsx(hp, sd, x[perm], g[perm])[:3]
        ones = [torch.ones(c["B"], c["T"], n, dtype=torch.bool) for n in
                [hp["hidden_size"]] + [hp["hidden_size"], 4 * hp["hidden_size"], hp["hidden_size"]] * hp["dec_layers"]]
        ref = fs2_ref(hp, sd, x, g, ones, "f64", DEV)
    elif step == "fft":
        hp, sd, spec, t, cond, g = fft_case(name)
        hp = dict(hp, dropout=0.0)
        a = fft_dsx(hp, sd, spec, t, cond, g)[:3]
        b = fft_dsx(hp, sd, spec[perm], t[perm], cond[perm], g[perm])[:3]
        ones = [torch.ones(c["B"], c["T"], n, dtype=torch.bool) for n in
                [hp["hidden_size"]] + [hp["hidden_size"], 4 * hp["hidden_size"], hp["hidden_size"]] * hp["dec_layers"]]
        ref = fft_ref(hp, sd, spec, t, cond, g, ones, "f64", DEV)
    else:
        net, spec, t, cond, g = diffnet_case(name)
        a = diffnet_dsx(net, spec, t, cond, g)
        b = diffnet_dsx(net, spec[perm], t[perm], cond[perm], g[perm])
        ref = diffnet_ref(net, spec, t, cond, g, "f64", DEV)
    for i in (0, 1):
        d = (b[i] - a[i][perm]).abs().reshape(len(perm), -1).amax(1)
        assert torch.equal(b[i], a[i][perm]), (i, d.tolist())
    e = {n: measure(n, b[2][n], ref[2][n]) for n in b[2]}
    wd = worst(e)
    for m, bound in BOUNDS[step, name].items():
        if m in wd:
            assert wd[m][0] <= bound, (m, wd[m], bound)
