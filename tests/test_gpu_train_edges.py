"""GPU: the five training steps -- the FastSpeech2 decoder (dsx_fs2dec_train_*), the FFT denoiser (dsx_fft_train_*),
DiffNet (dsx_train_*), the FastSpeech2 encoder (dsx_fs2enc_train_*) and the duration predictor (dsx_durpred_train_*) --
at the edges of the configurations their *_create functions accept, against float64 autograd of the oracles with the
step's own dropout masks, and exact properties of their backwards.

Cases.  They put T on both sides of the 64-row blocks of the attention backward (k_attn_bwd_kv / k_attn_bwd_q), the
64-row tiles of the conv core and the 64-frame chunks of k_wgrad (and the FFT's 128-frame column-sum partials), reach
the limits of hidden, heads, kernel, padding, layers, residual_channels and dilation_cycle_length that include/dsx.h
documents, and run batches where a tile, chunk or block straddles two utterances.  The encoder's cases also reach its
entry (both position terms, interior padding, T past the sinusoidal table's first 2000 rows and past the relative
table's 5000, rel_len = T, dropout site 0 at p 0.5 and 0.9) and its embedding gradient (a sort of F = 1024 keys in one
CTA, 1025 and 2049 with k_et_sort_step, vocabularies of 2 and 70000 rows).  The duration predictor's reach ragged column
tiles (idim / chans 80, 144, 240), every 4-tap k_wgrad split (k 1, 2, 5, 8, 9, 31), LEFT padding with T < k, L 1 and 16,
several k_dpt_head sweeps (B T up to 64000) and LayerNorm of an all-zero ReLU row (dead_rows_k1, where d_x must be
exactly 0).  Every case has B >= 2 unless its name says otherwise.

Measures, dsx against float64 and TF32 autograd (fp32 with TF32 matmuls and convolutions) against float64, per tensor:
  rel    ||a - r|| / ||r||;
  frame  for out, d_x, d_add, xs ([B, T, 1]), eps and d_cond: the worst non-padding frame's ||a - r|| over the RMS of
         ||r_frame|| over the non-padding frames (over the largest ||r_frame|| for the 64-layer stacks, whose frames
         span a wide range); the duration predictor's d_x over every frame, padding included;
  row    for matrices: the worst output row's ||a - r|| over the RMS row norm (embed_tokens.weight over the rows that
         have a frame); for conv weights with k > 1 (ffn_1, DiffNet's dilated_conv, the duration predictor's convs) the
         worst tap slice w[:, :, j] over the RMS tap-slice norm.
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
the same effect within the cap; the ReLU encoder case (H128_h1_left_k255_relu) shows it above it, so its frame and row
bounds are 3x TF32 uncapped.  The duration predictor's bounds are 3x TF32's worst over four seeds (11, the test's,
and 12, 13, 14), floored, uncapped.  Its reference rounds every conv operand to fp16 as the kernels do, and an fp32
LayerNorm output on one side of an fp16 rounding boundary where the float64 one lies on the other moves a conv output
by an fp16 step, which flips ReLUs and moves whole frames' gradients (oracle/precision_study_durtrain.py); sixteen
layers compound it (L16 at T 130: 0.33 rel for TF32 and dsx alike).  The flips are sparse draws, so one seed's TF32
error is a noisy yardstick: on i64_P64_k31_T130, at seeds 11, 12, 13 and 14, dsx / TF32 rel is 5.3e-2 / 7.7e-3,
2.4e-3 / 3.1e-2, 7.1e-4 / 6.3e-4 and 1.2e-2 / 1.6e-2, and the worst frames of the two lie in different places.  For
the duration predictor the TF32 column below is that worst over the four seeds; dsx is seed 11's.  Measured on an
H100 (80 GB HBM3, 700 W power limit), dsx / TF32 / bound:

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
    fs2enc  midi_T63                5.3e-04 / 5.2e-04 / 1.6e-03  1.8e-05 / 1.8e-05 / 4.0e-03  1.9e-03 / 1.8e-03 / 5.4e-03
    fs2enc  midi_T64                5.0e-04 / 8.3e-04 / 2.5e-03  1.8e-05 / 1.8e-05 / 4.0e-03  1.7e-03 / 2.0e-03 / 6.2e-03
    fs2enc  midi_T65                5.4e-04 / 5.4e-04 / 1.7e-03  1.8e-05 / 1.8e-05 / 4.0e-03  1.7e-03 / 1.9e-03 / 5.9e-03
    fs2enc  midi_T128               4.8e-04 / 8.3e-04 / 2.5e-03  1.7e-05 / 1.8e-05 / 4.0e-03  1.6e-03 / 1.7e-03 / 5.2e-03
    fs2enc  midi_T129               5.1e-04 / 8.3e-04 / 2.5e-03  1.7e-05 / 1.7e-05 / 4.0e-03  1.8e-03 / 1.8e-03 / 5.3e-03
    fs2enc  sin_H192_h3_T65         5.4e-04 / 5.2e-04 / 1.6e-03  2.9e-04 / 3.0e-04 / 4.0e-03  2.2e-03 / 2.2e-03 / 6.5e-03
    fs2enc  sin_interior_pad_60_70  5.6e-04 / 8.5e-04 / 2.6e-03  2.5e-04 / 2.5e-04 / 4.0e-03  2.4e-03 / 2.2e-03 / 6.7e-03
    fs2enc  sin_T2100               5.6e-04 / 8.5e-04 / 2.6e-03  2.3e-04 / 2.3e-04 / 4.0e-03  2.1e-03 / 2.2e-03 / 6.7e-03
    fs2enc  rel_len_T_T65           5.3e-04 / 5.3e-04 / 1.6e-03  1.8e-05 / 1.8e-05 / 4.0e-03  2.0e-03 / 2.1e-03 / 6.4e-03
    fs2enc  rel_B1_T5001_H128_h1_L1 4.3e-04 / 4.3e-04 / 1.3e-03  1.4e-05 / 1.4e-05 / 4.0e-03  1.4e-03 / 1.3e-03 / 4.0e-03
    fs2enc  H64_h1_L1_k1            5.6e-04 / 5.4e-04 / 1.7e-03  5.2e-05 / 5.3e-05 / 4.0e-03  1.7e-03 / 1.7e-03 / 5.0e-03
    fs2enc  H128_h1_left_k255_relu  3.1e-02 / 3.2e-02 / 5.0e-02  9.6e-05 / 9.6e-05 / 4.0e-03  6.0e-02 / 6.3e-02 / 1.9e-01
    fs2enc  H64_h1_L64              7.8e-04 / 7.6e-04 / 2.3e-03  1.4e-04 / 1.4e-04 / 4.0e-03  2.5e-03 / 2.4e-03 / 7.1e-03
    fs2enc  p05_T300                4.9e-04 / 8.3e-04 / 2.5e-03  1.8e-05 / 1.8e-05 / 4.0e-03  2.1e-03 / 1.8e-03 / 5.5e-03
    fs2enc  p09_T300                6.3e-04 / 8.4e-04 / 2.6e-03  5.7e-05 / 5.4e-05 / 4.0e-03  1.7e-03 / 1.8e-03 / 5.6e-03
    fs2enc  B300_T3                 6.3e-04 / 8.3e-04 / 2.5e-03  6.2e-05 / 5.2e-05 / 4.0e-03  1.3e-03 / 1.6e-03 / 4.9e-03
    fs2enc  B1_T1                   4.8e-04 / 3.4e-04 / 1.1e-03  3.8e-05 / 2.2e-06 / 4.0e-03  2.5e-03 / 1.3e-03 / 4.0e-03
    fs2enc  all_padding_utterance   4.9e-04 / 4.7e-04 / 1.5e-03  1.8e-05 / 1.8e-05 / 4.0e-03  2.0e-03 / 2.3e-03 / 6.9e-03
    fs2enc  one_token_utterance     6.0e-04 / 5.3e-04 / 1.6e-03  3.6e-05 / 3.5e-05 / 4.0e-03  1.8e-03 / 1.5e-03 / 4.6e-03
    fs2enc  B1_F1024                6.0e-04 / 8.3e-04 / 2.5e-03  1.6e-05 / 1.6e-05 / 4.0e-03  1.9e-03 / 1.9e-03 / 5.6e-03
    fs2enc  B1_F1025                5.3e-04 / 8.3e-04 / 2.5e-03  1.6e-05 / 1.6e-05 / 4.0e-03  1.8e-03 / 1.7e-03 / 5.1e-03
    fs2enc  B3_T683_F2049           5.8e-04 / 8.3e-04 / 2.6e-03  1.6e-05 / 1.6e-05 / 4.0e-03  1.7e-03 / 1.9e-03 / 5.7e-03
    fs2enc  vocab2                  5.2e-04 / 4.9e-04 / 1.5e-03  3.3e-05 / 3.4e-05 / 4.0e-03  1.8e-03 / 2.0e-03 / 6.2e-03
    fs2enc  vocab70000              5.4e-04 / 8.3e-04 / 2.5e-03  1.4e-05 / 1.5e-05 / 4.0e-03  1.8e-03 / 1.8e-03 / 5.4e-03
    durpred shipped_T63             5.9e-03 / 2.8e-02 / 8.3e-02  3.2e-02 / 1.5e-01 / 4.6e-01  5.9e-03 / 2.8e-02 / 8.3e-02
    durpred shipped_T64             1.2e-02 / 2.8e-02 / 8.4e-02  6.5e-02 / 1.5e-01 / 4.7e-01  1.2e-02 / 2.7e-02 / 8.2e-02
    durpred shipped_T65             7.9e-03 / 1.6e-02 / 4.7e-02  3.8e-02 / 9.2e-02 / 2.8e-01  7.0e-03 / 1.5e-02 / 4.6e-02
    durpred shipped_T128            1.6e-02 / 2.6e-02 / 8.0e-02  8.2e-02 / 2.2e-01 / 6.7e-01  1.4e-02 / 2.7e-02 / 8.0e-02
    durpred shipped_T129            1.3e-02 / 3.3e-02 / 1.0e-01  8.1e-02 / 2.6e-01 / 7.7e-01  1.2e-02 / 3.1e-02 / 9.4e-02
    durpred idim80_P144             6.6e-04 / 1.9e-02 / 5.8e-02  1.6e-03 / 1.6e-01 / 4.8e-01  6.6e-04 / 1.8e-02 / 5.5e-02
    durpred idim144_P48             7.7e-04 / 2.6e-02 / 7.9e-02  1.7e-03 / 2.2e-01 / 6.5e-01  6.7e-04 / 2.2e-02 / 6.7e-02
    durpred idim240_P240            7.3e-03 / 2.5e-02 / 7.7e-02  5.1e-02 / 1.4e-01 / 4.3e-01  6.4e-03 / 2.3e-02 / 6.9e-02
    durpred idim16_P16_k1           7.0e-04 / 2.7e-02 / 8.1e-02  3.9e-03 / 7.3e-02 / 2.3e-01  1.9e-03 / 6.7e-02 / 2.1e-01
    durpred same_k5                 1.7e-03 / 4.1e-02 / 1.3e-01  9.3e-03 / 2.2e-01 / 6.7e-01  1.6e-03 / 4.0e-02 / 1.2e-01
    durpred same_k9                 9.4e-04 / 1.4e-03 / 4.3e-03  1.3e-03 / 3.6e-03 / 1.1e-02  7.2e-04 / 1.1e-03 / 4.0e-03
    durpred left_k8                 2.0e-03 / 5.2e-02 / 1.6e-01  8.1e-03 / 2.1e-01 / 6.3e-01  1.8e-03 / 5.3e-02 / 1.7e-01
    durpred same_k31                1.9e-02 / 4.8e-02 / 1.5e-01  3.6e-02 / 1.2e-01 / 3.8e-01  1.9e-02 / 5.0e-02 / 1.6e-01
    durpred left_k2                 8.3e-04 / 5.6e-04 / 1.7e-03  3.5e-03 / 1.2e-03 / 4.0e-03  6.9e-04 / 5.7e-04 / 4.0e-03
    durpred left_k31_T3             6.1e-04 / 7.8e-04 / 2.4e-03  1.2e-03 / 2.0e-03 / 6.2e-03  3.4e-03 / 4.3e-03 / 1.3e-02
    durpred L1                      2.9e-04 / 5.3e-04 / 1.6e-03  7.1e-04 / 8.6e-04 / 4.0e-03  3.0e-04 / 5.4e-04 / 4.0e-03
    durpred L16_idim32_P32          6.9e-02 / 1.6e-01 / 4.9e-01  2.7e-01 / 8.6e-01 / 2.6e+00  4.6e-02 / 1.2e-01 / 3.7e-01
    durpred L16_idim256_P256        1.3e-01 / 1.2e-01 / 3.8e-01  3.9e-01 / 3.3e-01 / 9.9e-01  1.2e-01 / 1.1e-01 / 3.5e-01
    durpred B16_T250                1.5e-02 / 2.1e-02 / 6.2e-02  2.4e-01 / 3.0e-01 / 8.9e-01  1.3e-02 / 1.9e-02 / 5.6e-02
    durpred B64_T1000               1.6e-02 / 1.9e-02 / 5.8e-02  4.3e-01 / 4.3e-01 / 1.3e+00  1.5e-02 / 1.8e-02 / 5.5e-02
    durpred B300_T3                 1.6e-02 / 3.0e-02 / 9.1e-02  2.2e-01 / 4.8e-01 / 1.5e+00  1.7e-02 / 3.5e-02 / 1.1e-01
    durpred B1_T1                   7.5e-04 / 1.7e-03 / 5.1e-03  7.3e-04 / 1.7e-03 / 5.1e-03  1.3e-03 / 1.5e-03 / 4.4e-03
    durpred all_padding_utterance   1.6e-03 / 3.3e-02 / 9.9e-02  9.2e-03 / 1.9e-01 / 5.8e-01  1.6e-03 / 3.1e-02 / 9.3e-02
    durpred interior_pad_60_70      5.5e-03 / 3.4e-02 / 1.1e-01  3.0e-02 / 1.7e-01 / 5.0e-01  5.2e-03 / 3.0e-02 / 9.0e-02
    durpred p0                      1.9e-02 / 4.2e-02 / 1.3e-01  9.4e-02 / 2.6e-01 / 7.9e-01  1.8e-02 / 3.5e-02 / 1.1e-01
    durpred p09                     7.4e-04 / 4.1e-02 / 1.3e-01  1.9e-03 / 3.6e-01 / 1.1e+00  7.2e-04 / 4.6e-02 / 1.4e-01
    durpred dead_rows_k1            7.4e-04 / 2.2e-04 / 9.8e-04  6.9e-03 / 2.6e-03 / 7.9e-03  1.5e-03 / 7.0e-04 / 4.0e-03
    durpred i16_P16_T65             6.7e-04 / 9.9e-05 / 9.8e-04  2.6e-03 / 3.8e-04 / 4.0e-03  7.2e-04 / 1.2e-04 / 4.0e-03
    durpred L1_i256_P256_T65        3.0e-04 / 3.2e-04 / 9.8e-04  9.9e-04 / 1.0e-03 / 4.0e-03  3.0e-04 / 4.0e-05 / 4.0e-03
    durpred i48_P112_T65            7.5e-04 / 6.2e-02 / 1.9e-01  1.6e-03 / 3.1e-01 / 9.4e-01  7.0e-04 / 5.4e-02 / 1.7e-01
    durpred i16_P256_k1_T65         6.4e-04 / 2.3e-03 / 7.0e-03  3.7e-03 / 3.0e-02 / 9.1e-02  1.7e-03 / 2.0e-02 / 6.2e-02
    durpred i64_P64_k31_T65         1.6e-03 / 9.2e-03 / 2.8e-02  3.7e-03 / 2.2e-02 / 6.8e-02  1.9e-03 / 9.9e-03 / 3.0e-02
    durpred i64_P64_left_k4_T65     6.9e-04 / 5.6e-02 / 1.7e-01  2.3e-03 / 2.4e-01 / 7.2e-01  7.6e-04 / 5.8e-02 / 1.8e-01
    durpred L16_i32_P32_T65         1.2e-02 / 6.8e-02 / 2.1e-01  3.6e-02 / 1.1e-01 / 3.4e-01  9.9e-03 / 5.4e-02 / 1.7e-01
    durpred i128_P128_left_k2_T65   7.0e-04 / 9.1e-04 / 2.8e-03  2.8e-03 / 3.2e-03 / 9.6e-03  6.9e-04 / 9.0e-04 / 4.0e-03
    durpred i16_P16_T130            7.3e-04 / 1.8e-04 / 9.8e-04  2.9e-03 / 9.3e-04 / 4.0e-03  7.1e-04 / 2.0e-04 / 4.0e-03
    durpred L1_i256_P256_T130       2.9e-04 / 5.3e-04 / 1.6e-03  7.5e-04 / 9.7e-04 / 4.0e-03  2.9e-04 / 5.4e-04 / 4.0e-03
    durpred i48_P112_T130           6.7e-04 / 4.5e-03 / 1.4e-02  1.7e-03 / 3.6e-02 / 1.1e-01  6.7e-04 / 4.3e-03 / 1.3e-02
    durpred i16_P256_k1_T130        6.7e-04 / 8.0e-03 / 2.5e-02  4.0e-03 / 1.4e-01 / 4.4e-01  1.5e-03 / 6.6e-02 / 2.0e-01
    durpred i64_P64_k31_T130        5.3e-02 / 3.1e-02 / 9.2e-02  1.1e-01 / 1.0e-01 / 3.1e-01  5.5e-02 / 3.5e-02 / 1.1e-01
    durpred i64_P64_left_k4_T130    7.1e-04 / 1.1e-02 / 3.5e-02  3.6e-03 / 6.5e-02 / 2.0e-01  7.4e-04 / 1.1e-02 / 3.4e-02
    durpred L16_i32_P32_T130        3.3e-01 / 3.3e-01 / 9.8e-01  1.1e+00 / 1.1e+00 / 3.4e+00  1.9e-01 / 1.9e-01 / 5.6e-01
    durpred i128_P128_left_k2_T130  4.1e-02 / 4.4e-02 / 1.4e-01  3.0e-01 / 3.6e-01 / 1.1e+00  3.8e-02 / 4.2e-02 / 1.3e-01

The exact properties: a zero cotangent on one utterance gives exactly zero d_x / d_cond / d_add rows there (every step,
with and without dropout, at T = 65 and 129 with B = 3, so partial tiles and chunks straddle the utterance); permuting
the utterances of a batch (t with them) permutes out / eps / xs and d_x / d_cond / d_add bit for bit at p = 0, while
the weight gradients, which sum over the batch in another order, stay within the case's bounds; the encoder's
embedding gradient is sqrt(H) times the sum of its own d_add per token, to fp32 summation rounding, on token layouts
built for its sort; and the duration predictor's backward without d_x gives the same parameter gradients bit for
bit."""
import contextlib
import copy

import numpy as np
import pytest
import torch

from oracle import fft_oracle as FO
from oracle import fs2dec_oracle as D
from oracle import fs2enc_oracle as EO
from oracle.durpred_train_oracle import durpred_train
from oracle.fft_train_oracle import forward_train
from oracle.fs2dec_train_oracle import decoder_train
from oracle.fs2enc_train_oracle import encoder_train
from oracle.gen_golden_durpred_train import random_state_dict as dur_state_dict

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
CAP = 5e-2
FLOOR = dict(rel=2.0 ** -10, frame=2.0 ** -8, row=2.0 ** -8)
SEED = 11
VOCAB = 61


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



def enc_hp(H=256, heads=2, k=9, padding='SAME', L=4, p=0.1, act='gelu', rel=True):
    return dict(EO.HPARAMS_MIDI, hidden_size=H, enc_layers=L, enc_ffn_kernel_size=k, num_heads=heads,
                ffn_padding=padding, ffn_act=act, rel_pos=rel, dropout=p)


# The MIDI encoder (rel_pos, the addends of fs2enc_oracle.midi_addends) unless midi=False: then FastspeechEncoder with
# the sinusoidal position term and no addends (rel_pos is the MIDI encoder's).  tail, pad, empty, lengths: as in FS2, on
# the tokens; single: an utterance of one token; vocab: rows of embed_tokens (default VOCAB; the ids are drawn from all
# of them); rel_len: "T" sets the module's RelPositionalEncoding length to T before the step (default 5000)
FS2ENC = {
    "midi_T63": dict(hp=enc_hp(), B=3, T=63, tail=True),
    "midi_T64": dict(hp=enc_hp(), B=3, T=64, tail=True),
    "midi_T65": dict(hp=enc_hp(), B=3, T=65, tail=True),
    "midi_T128": dict(hp=enc_hp(), B=3, T=128, tail=True),
    "midi_T129": dict(hp=enc_hp(), B=3, T=129, tail=True),
    "sin_H192_h3_T65": dict(hp=enc_hp(192, 3, rel=False), midi=False, B=3, T=65, tail=True),
    "sin_interior_pad_60_70": dict(hp=enc_hp(rel=False), midi=False, B=2, T=150, tail=True, pad=(60, 71)),
    "sin_T2100": dict(hp=enc_hp(rel=False), midi=False, B=2, T=2100, tail=True),
    "rel_len_T_T65": dict(hp=enc_hp(), B=3, T=65, tail=True, rel_len="T"),
    "rel_B1_T5001_H128_h1_L1": dict(hp=enc_hp(128, 1, L=1), B=1, T=5001),
    "H64_h1_L1_k1": dict(hp=enc_hp(64, 1, 1, L=1), B=2, T=100, tail=True),
    "H128_h1_left_k255_relu": dict(hp=enc_hp(128, 1, 255, 'LEFT', act='relu'), B=2, T=100, tail=True),
    "H64_h1_L64": dict(hp=enc_hp(64, 1, L=64), B=2, T=80, tail=True, peak=True),
    "p05_T300": dict(hp=enc_hp(p=0.5), B=2, T=300, tail=True),
    "p09_T300": dict(hp=enc_hp(p=0.9), B=2, T=300, tail=True),
    "B300_T3": dict(hp=enc_hp(), B=300, T=3, lengths=[3, 1, 2]),
    "B1_T1": dict(hp=enc_hp(), B=1, T=1),
    "all_padding_utterance": dict(hp=enc_hp(), B=3, T=100, tail=True, empty=2),
    "one_token_utterance": dict(hp=enc_hp(), B=3, T=20, tail=True, single=2),
    "B1_F1024": dict(hp=enc_hp(), B=1, T=1024),
    "B1_F1025": dict(hp=enc_hp(), B=1, T=1025),
    "B3_T683_F2049": dict(hp=enc_hp(), B=3, T=683, tail=True),
    "vocab2": dict(hp=enc_hp(), B=3, T=65, tail=True, vocab=2),
    "vocab70000": dict(hp=enc_hp(), B=3, T=300, tail=True, vocab=70000),
}


def dur_hp(idim=256, P=256, L=5, k=3, padding='SAME', p=0.5):
    return dict(idim=idim, P=P, L=L, k=k, padding=padding, p=p)


# tail, pad, empty, lengths: as in FS2, on the mask (x stays non-zero on padding tokens, as in the reference); tails:
# (utterance, first padding token) pairs instead of tail; dead: (utterance, token) pairs where x = 0, with layer 0's bias
# made negative, so that (k = 1) layer 0's ReLU output is an all-zero row there.  The i*_P*_T65 / _T130 cases (B 3, tails
# at T - 20 and 7) are the configurations test_gpu_durpred_train.py checked against float64 before this file did.
DURPRED = {
    "shipped_T63": dict(hp=dur_hp(), B=3, T=63, tail=True),
    "shipped_T64": dict(hp=dur_hp(), B=3, T=64, tail=True),
    "shipped_T65": dict(hp=dur_hp(), B=3, T=65, tail=True),
    "shipped_T128": dict(hp=dur_hp(), B=3, T=128, tail=True),
    "shipped_T129": dict(hp=dur_hp(), B=3, T=129, tail=True),
    "idim80_P144": dict(hp=dur_hp(80, 144), B=3, T=129, tail=True),
    "idim144_P48": dict(hp=dur_hp(144, 48), B=3, T=129, tail=True),
    "idim240_P240": dict(hp=dur_hp(240, 240), B=3, T=129, tail=True),
    "idim16_P16_k1": dict(hp=dur_hp(16, 16, k=1), B=3, T=129, tail=True),
    "same_k5": dict(hp=dur_hp(64, 64, k=5), B=3, T=100, tail=True),
    "same_k9": dict(hp=dur_hp(64, 64, k=9), B=3, T=100, tail=True),
    "left_k8": dict(hp=dur_hp(64, 64, k=8, padding='LEFT'), B=3, T=100, tail=True),
    "same_k31": dict(hp=dur_hp(64, 64, k=31), B=3, T=100, tail=True),
    "left_k2": dict(hp=dur_hp(64, 64, k=2, padding='LEFT'), B=3, T=100, tail=True),
    "left_k31_T3": dict(hp=dur_hp(64, 64, k=31, padding='LEFT'), B=3, T=3, tail=True),
    "L1": dict(hp=dur_hp(L=1), B=3, T=129, tail=True),
    "L16_idim32_P32": dict(hp=dur_hp(32, 32, L=16), B=3, T=129, tail=True),
    "L16_idim256_P256": dict(hp=dur_hp(L=16), B=3, T=129, tail=True),
    "B16_T250": dict(hp=dur_hp(), B=16, T=250, tails=[(b, 250 - 13 * b) for b in range(1, 16)]),
    "B64_T1000": dict(hp=dur_hp(), B=64, T=1000, tails=[(b, 1000 - 13 * b) for b in range(1, 64)]),
    "B300_T3": dict(hp=dur_hp(), B=300, T=3, lengths=[3, 1, 2]),
    "B1_T1": dict(hp=dur_hp(), B=1, T=1),
    "all_padding_utterance": dict(hp=dur_hp(), B=3, T=100, tail=True, empty=2),
    "interior_pad_60_70": dict(hp=dur_hp(), B=2, T=150, tail=True, pad=(60, 71)),
    "p0": dict(hp=dur_hp(p=0.0), B=3, T=129, tail=True),
    "p09": dict(hp=dur_hp(p=0.9), B=3, T=129, tail=True),
    "dead_rows_k1": dict(hp=dur_hp(64, 64, k=1), B=3, T=129, tail=True,
                         dead=[(0, 0), (0, 63), (0, 64), (0, 128), (1, 5), (2, 70)]),
}
for _T in (65, 130):
    for _n, _hp in (("i16_P16", dur_hp(16, 16)), ("L1_i256_P256", dur_hp(L=1)), ("i48_P112", dur_hp(48, 112)),
                    ("i16_P256_k1", dur_hp(16, 256, k=1)), ("i64_P64_k31", dur_hp(64, 64, k=31)),
                    ("i64_P64_left_k4", dur_hp(64, 64, k=4, padding='LEFT')), ("L16_i32_P32", dur_hp(32, 32, L=16)),
                    ("i128_P128_left_k2", dur_hp(128, 128, k=2, padding='LEFT'))):
        DURPRED[f"{_n}_T{_T}"] = dict(hp=_hp, B=3, T=_T, tails=[(1, _T - 20), (2, 7)])

CASES = {"fs2": FS2, "fft": FFT, "diffnet": DIFFNET, "fs2enc": FS2ENC, "durpred": DURPRED}


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


def enc_case(name, seed=SEED):
    """(hp, state dict of the front end (fs2enc_oracle names), tokens [B, T], the three addends [B, T, H] (or ()),
    cotangent of out [B, T, H]) on the CPU, fp32"""
    c = FS2ENC[name]
    hp, B, T, V = c["hp"], c["B"], c["T"], c.get("vocab", VOCAB)
    tails = [None] * B
    if c.get("tail") and B > 1 and T >= 4:
        tails[1] = T - T // 4
    for b in range(B) if "lengths" in c else ():
        tails[b] = c["lengths"][b % len(c["lengths"])]
    for key, at in (("empty", 0), ("single", 1)):
        if key in c:
            tails[c[key]] = at
    tok, pm, md, sl = EO.fixture_inputs(seed, B, T, tails, V)
    if "pad" in c:
        for v in (tok, pm, md, sl):
            v[:, c["pad"][0]:c["pad"][1]] = 0
    midi = c.get("midi", True)
    sd = EO.random_state_dict(seed + 1, hp, V, midi=midi)
    adds = tuple(a.detach() for a in EO.midi_addends(sd, pm, md, sl)) if midi else ()
    g = torch.from_numpy(np.random.RandomState(seed + 2).standard_normal((B, T, hp["hidden_size"])).astype(np.float32))
    return hp, sd, tok, adds, g


def dur_case(name, seed=SEED):
    """(hp, state dict, x [B, T, idim], mask [B, T] (True = padding), cotangent of xs [B, T]) on the CPU, fp32"""
    c = DURPRED[name]
    hp, B, T = c["hp"], c["B"], c["T"]
    sd = dur_state_dict(seed + 1, hp["idim"], hp["L"], hp["P"], hp["k"])
    rs = np.random.RandomState(seed)
    x = torch.from_numpy(rs.standard_normal((B, T, hp["idim"])).astype(np.float32))
    mask = torch.zeros(B, T, dtype=torch.bool)
    if c.get("tail") and B > 1 and T >= 4:
        mask[1, T - T // 4:] = True
    for b, t in c.get("tails", []):
        mask[b, t:] = True
    for b in range(B) if "lengths" in c else ():
        mask[b, c["lengths"][b % len(c["lengths"])]:] = True
    if "empty" in c:
        mask[c["empty"]] = True
    if "pad" in c:
        mask[:, c["pad"][0]:c["pad"][1]] = True
    if "dead" in c:
        sd["conv.0.1.bias"] = -0.05 - sd["conv.0.1.bias"].abs()
        for b, t in c["dead"]:
            x[b, t] = 0
    g = torch.from_numpy(rs.standard_normal((B, T)).astype(np.float32))
    return hp, sd, x, mask, g


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


def enc_ref(hp, sd, tok, adds, g, masks, rel_len, mode, dev):
    """out, d_add (None without addends), {name: grad} of sum(out * g) through encoder_train in `mode`"""
    with precision(mode) as dt:
        w = _leaves(EO.sub(sd, "encoder."), dev, dt)
        ar = [a.to(dev, dt).requires_grad_(True) for a in adds]
        out = encoder_train(w, tok.to(dev), hp, [m.to(dev) for m in masks], hp["dropout"], tuple(ar), rel_len)
        (out * g.to(dev, dt)).sum().backward()
    return out.detach(), ar[0].grad if ar else None, {n: v.grad for n, v in w.items()}


def dur_ref(hp, sd, x, mask, g, masks, mode, dev, fp16=True):
    """xs, d_x, {name: grad} of sum(xs * g) through durpred_train with fp16-rounded conv operands (fp16=True) in
    `mode`"""
    with precision(mode) as dt:
        w = _leaves(sd, dev, dt)
        xr = x.to(dev, dt).requires_grad_(True)
        xs = durpred_train(w, xr, mask.to(dev), [m.to(dev) for m in masks], hp["p"], hp["k"], hp["padding"], fp16=fp16)
        (xs * g.to(dev, dt)).sum().backward()
    return xs.detach(), xr.grad, {n: v.grad for n, v in w.items()}


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
FRAMES = {"out": "btc", "d_x": "btc", "d_add": "btc", "xs": "btc", "eps": "bct", "d_cond": "bct"}


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
    """{tensor: {measure: error}} of (primary, d_input, grads) against the same of the reference.  keep: the frames of
    both, or a pair (the primary's, d_input's); a d_input of None (no addends) is not measured."""
    ks = keep if isinstance(keep, tuple) else (keep, keep)
    e = {n: measure(n, a, r, k, peak) for n, a, r, k in zip(names, res[:2], ref[:2], ks) if r is not None}
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


def fs2enc_dsx(hp, sd, tok, adds, g, rel_len=None, seed=SEED):
    """out, d_add (None without addends), {name: grad}, masks, the module's rel_len of one step of the encoder under
    dsx_train (the MIDI encoder when there are addends)"""
    from diffsinger_b200 import FastspeechEncoder, FastspeechMIDIEncoder, fs2enctrain
    H = hp["hidden_size"]
    cls = FastspeechMIDIEncoder if adds else FastspeechEncoder
    m = cls(torch.nn.Embedding(sd["encoder.embed_tokens.weight"].shape[0], H, 0), H, hp["enc_layers"],
            hp["enc_ffn_kernel_size"], num_heads=hp["num_heads"], hparams=dict(hp, dsx_train=True))
    m.load_state_dict(EO.sub(sd, "encoder."), strict=True)
    m = m.train().to(DEV)
    if rel_len is not None:
        m._rel_len = rel_len
    tk = tok.to(DEV)
    ar = [a.to(DEV).requires_grad_(True) for a in adds]

    def run():
        out = m(tk, *ar) if ar else m(tk)
        (out * g.to(DEV)).sum().backward()
        return out
    out = with_seed(fs2enctrain, seed, run)
    masks = m._dsx_train_step().masks(DEV, seed, hp["dropout"], tok.shape[0], tok.shape[1])
    grads = {n: p.grad for n, p in m.named_parameters()}
    return out.detach(), ar[0].grad if ar else None, grads, masks, m._rel_len


def dur_module(hp, sd):
    from diffsinger_b200 import DurationPredictor
    m = DurationPredictor(hp["idim"], hp["L"], hp["P"], hp["k"], hp["p"], padding=hp["padding"],
                          hparams=dict(dur_loss='mse'), train=True)
    m.load_state_dict(sd, strict=True)
    return m.train().to(DEV)


def dur_dsx(hp, sd, x, mask, g, seed=SEED):
    """xs, d_x, {name: grad}, masks of one step of DurationPredictor under dsx_train"""
    from diffsinger_b200 import durtrain
    m = dur_module(hp, sd)
    xr = x.to(DEV).requires_grad_(True)

    def run():
        xs = m(xr, mask.to(DEV))
        (xs * g.to(DEV)).sum().backward()
        return xs
    xs = with_seed(durtrain, seed, run)
    masks = m._dsx_train_step().masks(DEV, seed, hp["p"], x.shape[0], x.shape[1])
    return xs.detach(), xr.grad, {n: p.grad for n, p in m.named_parameters()}, masks


def used_rows(tok, V):
    """[V] bool: the embedding rows some non-padding token in [1, V) reads"""
    t = tok[(tok > 0) & (tok < V)]
    u = torch.zeros(V, dtype=torch.bool, device=tok.device)
    u[t] = True
    return u


def embed_rows(grads, used):
    """grads with embed_tokens.weight cut to the rows in `used` (its row measure is over the rows that have a frame)"""
    dE = grads["embed_tokens.weight"]
    return dict(grads, **{"embed_tokens.weight": dE[used.to(dE.device)]})


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
    elif step == "fs2enc":
        hp, sd, tok, adds, g = enc_case(name)
        rl = c["T"] if c.get("rel_len") == "T" else None
        out, da, grads, masks, rel_len = fs2enc_dsx(hp, sd, tok, adds, g, rl)
        pad = (tok == 0).to(DEV)
        assert (out[pad] == 0).all() and (da is None or (da[pad] == 0).all())
        used = used_rows(tok, sd["encoder.embed_tokens.weight"].shape[0])
        dE = grads["embed_tokens.weight"]
        assert (dE[0] == 0).all() and (dE[~used.to(DEV)] == 0).all()
        idx = [b for b in range(c["B"]) if b != c.get("empty")]
        if "empty" in c:                      # the reference gives NaN there: compare the batch without it
            assert (out[c["empty"]] == 0).all() and (da[c["empty"]] == 0).all()
        sub = lambda v: v[idx]
        refs = {mode: enc_ref(hp, sd, sub(tok), [sub(a) for a in adds], sub(g), [sub(mk) for mk in masks], rel_len, mode,
                              DEV) for mode in ("f64", "tf32")}
        res = (sub(out), None if da is None else sub(da), embed_rows(grads, used))
        refs = {k: (v[0], v[1], embed_rows(v[2], used)) for k, v in refs.items()}
        keep, names = sub(tok) != 0, ("out", "d_add")
    elif step == "durpred":
        hp, sd, x, mask, g = dur_case(name)
        xs, dx, grads, masks = dur_dsx(hp, sd, x, mask, g)
        assert (xs[mask.to(DEV)] == 0).all()
        for b, t in c.get("dead", []):        # layer 0's ReLU output is an all-zero row there: LayerNorm's rstd is 1e6
            assert (dx[b, t] == 0).all(), (b, t)
        refs = {mode: dur_ref(hp, sd, x, mask, g, masks, mode, DEV) for mode in ("f64", "tf32")}
        for b, t in c.get("dead", []):
            assert (refs["f64"][1][b, t] == 0).all()
        res = (xs[..., None], dx, grads)
        refs = {k: (v[0][..., None], v[1], v[2]) for k, v in refs.items()}
        keep, names = (~mask, None), ("xs", "d_x")           # d_x over every token: padding tokens carry real d_x
    else:
        net, spec, t, cond, g = diffnet_case(name)
        res = diffnet_dsx(net, spec, t, cond, g)
        refs = {mode: diffnet_ref(net, spec, t, cond, g, mode, DEV) for mode in ("f64", "tf32")}
        keep, names = None, ("eps", "d_cond")
    assert all(torch.isfinite(v).all() for v in (res[0], *res[1:2], *res[2].values()) if v is not None)
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
    ("fs2enc", "midi_T63"): dict(rel=1.6e-03, frame=4.0e-03, row=5.4e-03),
    ("fs2enc", "midi_T64"): dict(rel=2.5e-03, frame=4.0e-03, row=6.2e-03),
    ("fs2enc", "midi_T65"): dict(rel=1.7e-03, frame=4.0e-03, row=5.9e-03),
    ("fs2enc", "midi_T128"): dict(rel=2.5e-03, frame=4.0e-03, row=5.2e-03),
    ("fs2enc", "midi_T129"): dict(rel=2.5e-03, frame=4.0e-03, row=5.3e-03),
    ("fs2enc", "sin_H192_h3_T65"): dict(rel=1.6e-03, frame=4.0e-03, row=6.5e-03),
    ("fs2enc", "sin_interior_pad_60_70"): dict(rel=2.6e-03, frame=4.0e-03, row=6.7e-03),
    ("fs2enc", "sin_T2100"): dict(rel=2.6e-03, frame=4.0e-03, row=6.7e-03),
    ("fs2enc", "rel_len_T_T65"): dict(rel=1.6e-03, frame=4.0e-03, row=6.4e-03),
    ("fs2enc", "rel_B1_T5001_H128_h1_L1"): dict(rel=1.3e-03, frame=4.0e-03, row=4.0e-03),
    ("fs2enc", "H64_h1_L1_k1"): dict(rel=1.7e-03, frame=4.0e-03, row=5.0e-03),
    ("fs2enc", "H128_h1_left_k255_relu"): dict(rel=5.0e-02, frame=4.0e-03, row=1.9e-01),
    ("fs2enc", "H64_h1_L64"): dict(rel=2.3e-03, frame=4.0e-03, row=7.1e-03),
    ("fs2enc", "p05_T300"): dict(rel=2.5e-03, frame=4.0e-03, row=5.5e-03),
    ("fs2enc", "p09_T300"): dict(rel=2.6e-03, frame=4.0e-03, row=5.6e-03),
    ("fs2enc", "B300_T3"): dict(rel=2.5e-03, frame=4.0e-03, row=4.9e-03),
    ("fs2enc", "B1_T1"): dict(rel=1.1e-03, frame=4.0e-03, row=4.0e-03),
    ("fs2enc", "all_padding_utterance"): dict(rel=1.5e-03, frame=4.0e-03, row=6.9e-03),
    ("fs2enc", "one_token_utterance"): dict(rel=1.6e-03, frame=4.0e-03, row=4.6e-03),
    ("fs2enc", "B1_F1024"): dict(rel=2.5e-03, frame=4.0e-03, row=5.6e-03),
    ("fs2enc", "B1_F1025"): dict(rel=2.5e-03, frame=4.0e-03, row=5.1e-03),
    ("fs2enc", "B3_T683_F2049"): dict(rel=2.6e-03, frame=4.0e-03, row=5.7e-03),
    ("fs2enc", "vocab2"): dict(rel=1.5e-03, frame=4.0e-03, row=6.2e-03),
    ("fs2enc", "vocab70000"): dict(rel=2.5e-03, frame=4.0e-03, row=5.4e-03),
    ("durpred", "shipped_T63"): dict(rel=8.3e-02, frame=4.6e-01, row=8.3e-02),
    ("durpred", "shipped_T64"): dict(rel=8.4e-02, frame=4.7e-01, row=8.2e-02),
    ("durpred", "shipped_T65"): dict(rel=4.7e-02, frame=2.8e-01, row=4.6e-02),
    ("durpred", "shipped_T128"): dict(rel=8.0e-02, frame=6.7e-01, row=8.0e-02),
    ("durpred", "shipped_T129"): dict(rel=1.0e-01, frame=7.7e-01, row=9.4e-02),
    ("durpred", "idim80_P144"): dict(rel=5.8e-02, frame=4.8e-01, row=5.5e-02),
    ("durpred", "idim144_P48"): dict(rel=7.9e-02, frame=6.5e-01, row=6.7e-02),
    ("durpred", "idim240_P240"): dict(rel=7.7e-02, frame=4.3e-01, row=6.9e-02),
    ("durpred", "idim16_P16_k1"): dict(rel=8.1e-02, frame=2.3e-01, row=2.1e-01),
    ("durpred", "same_k5"): dict(rel=1.3e-01, frame=6.7e-01, row=1.2e-01),
    ("durpred", "same_k9"): dict(rel=4.3e-03, frame=1.1e-02, row=4.0e-03),
    ("durpred", "left_k8"): dict(rel=1.6e-01, frame=6.3e-01, row=1.7e-01),
    ("durpred", "same_k31"): dict(rel=1.5e-01, frame=3.8e-01, row=1.6e-01),
    ("durpred", "left_k2"): dict(rel=1.7e-03, frame=4.0e-03, row=4.0e-03),
    ("durpred", "left_k31_T3"): dict(rel=2.4e-03, frame=6.2e-03, row=1.3e-02),
    ("durpred", "L1"): dict(rel=1.6e-03, frame=4.0e-03, row=4.0e-03),
    ("durpred", "L16_idim32_P32"): dict(rel=4.9e-01, frame=2.6e+00, row=3.7e-01),
    ("durpred", "L16_idim256_P256"): dict(rel=3.8e-01, frame=9.9e-01, row=3.5e-01),
    ("durpred", "B16_T250"): dict(rel=6.2e-02, frame=8.9e-01, row=5.6e-02),
    ("durpred", "B64_T1000"): dict(rel=5.8e-02, frame=1.3e+00, row=5.5e-02),
    ("durpred", "B300_T3"): dict(rel=9.1e-02, frame=1.5e+00, row=1.1e-01),
    ("durpred", "B1_T1"): dict(rel=5.1e-03, frame=5.1e-03, row=4.4e-03),
    ("durpred", "all_padding_utterance"): dict(rel=9.9e-02, frame=5.8e-01, row=9.3e-02),
    ("durpred", "interior_pad_60_70"): dict(rel=1.1e-01, frame=5.0e-01, row=9.0e-02),
    ("durpred", "p0"): dict(rel=1.3e-01, frame=7.9e-01, row=1.1e-01),
    ("durpred", "p09"): dict(rel=1.3e-01, frame=1.1e+00, row=1.4e-01),
    ("durpred", "dead_rows_k1"): dict(rel=9.8e-04, frame=7.9e-03, row=4.0e-03),
    ("durpred", "i16_P16_T65"): dict(rel=9.8e-04, frame=4.0e-03, row=4.0e-03),
    ("durpred", "L1_i256_P256_T65"): dict(rel=9.8e-04, frame=4.0e-03, row=4.0e-03),
    ("durpred", "i48_P112_T65"): dict(rel=1.9e-01, frame=9.4e-01, row=1.7e-01),
    ("durpred", "i16_P256_k1_T65"): dict(rel=7.0e-03, frame=9.1e-02, row=6.2e-02),
    ("durpred", "i64_P64_k31_T65"): dict(rel=2.8e-02, frame=6.8e-02, row=3.0e-02),
    ("durpred", "i64_P64_left_k4_T65"): dict(rel=1.7e-01, frame=7.2e-01, row=1.8e-01),
    ("durpred", "L16_i32_P32_T65"): dict(rel=2.1e-01, frame=3.4e-01, row=1.7e-01),
    ("durpred", "i128_P128_left_k2_T65"): dict(rel=2.8e-03, frame=9.6e-03, row=4.0e-03),
    ("durpred", "i16_P16_T130"): dict(rel=9.8e-04, frame=4.0e-03, row=4.0e-03),
    ("durpred", "L1_i256_P256_T130"): dict(rel=1.6e-03, frame=4.0e-03, row=4.0e-03),
    ("durpred", "i48_P112_T130"): dict(rel=1.4e-02, frame=1.1e-01, row=1.3e-02),
    ("durpred", "i16_P256_k1_T130"): dict(rel=2.5e-02, frame=4.4e-01, row=2.0e-01),
    ("durpred", "i64_P64_k31_T130"): dict(rel=9.2e-02, frame=3.1e-01, row=1.1e-01),
    ("durpred", "i64_P64_left_k4_T130"): dict(rel=3.5e-02, frame=2.0e-01, row=3.4e-02),
    ("durpred", "L16_i32_P32_T130"): dict(rel=9.8e-01, frame=3.4e+00, row=5.6e-01),
    ("durpred", "i128_P128_left_k2_T130"): dict(rel=1.4e-01, frame=1.1e+00, row=1.3e-01),
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


@pytest.mark.parametrize("case", list(FS2ENC))
def test_fs2enc_step(lib_built, case):
    check("fs2enc", case, run_case("fs2enc", case))


@pytest.mark.parametrize("case", list(DURPRED))
def test_durpred_step(lib_built, case):
    check("durpred", case, run_case("durpred", case))


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
    if step == "fs2enc":
        hp = enc_hp(p=p)
        sd = EO.random_state_dict(SEED + 1, hp, VOCAB)
        tok, pm, md, sl = EO.fixture_inputs(SEED, B, T, (None, T - T // 4, None), VOCAB)
        adds = [a.detach()[order] for a in EO.midi_addends(sd, pm, md, sl)]
        g = torch.from_numpy(np.random.RandomState(SEED + 2).standard_normal((B, T, 256)).astype(np.float32))
        if zero is not None:
            g[zero] = 0
        return fs2enc_dsx(hp, sd, tok[order], adds, g[order])[:3]
    if step == "durpred":
        hp = dur_hp(p=p)
        sd = dur_state_dict(SEED + 1, 256, 5, 256, 3)
        rs = np.random.RandomState(SEED)
        x = torch.from_numpy(rs.standard_normal((B, T, 256)).astype(np.float32))
        g = torch.from_numpy(rs.standard_normal((B, T)).astype(np.float32))
        mask = torch.zeros(B, T, dtype=torch.bool)
        mask[1, T - T // 4:] = True
        if zero is not None:
            g[zero] = 0
        return dur_dsx(hp, sd, x[order], mask[order], g[order])[:3]
    net, spec, t, cond, g = diffnet_inputs(dict(L=12, cycle=12, B=B, T=T))
    if zero is not None:
        g[zero] = 0
    return diffnet_dsx(net, spec[order], t[order], cond[order], g[order])


@pytest.mark.parametrize("T", [65, 129])
@pytest.mark.parametrize("step,p", [("fs2", 0.0), ("fs2", 0.1), ("fft", 0.0), ("fft", 0.1), ("diffnet", 0.0),
                                    ("fs2enc", 0.0), ("fs2enc", 0.1), ("durpred", 0.0), ("durpred", 0.5)])
def test_utterance_isolation(lib_built, step, p, T):
    """A zero cotangent on utterance 1 of 3: its d_x / d_cond / d_add rows are exactly 0, the other utterances' are
    not."""
    _, d, _ = _step_run(step, T, p, zero=1)
    assert (d[1] == 0).all()
    assert (d[0] != 0).any() and (d[2] != 0).any()


PERM_CASE = {"fs2": "H192_h3_T65", "fft": "T65", "diffnet": "L3_T65", "fs2enc": "midi_T65", "durpred": "shipped_T65"}


@pytest.mark.parametrize("step", ["fs2", "fft", "diffnet", "fs2enc", "durpred"])
def test_permutation_equivariance(lib_built, step):
    """p = 0: permuting the utterances permutes out / eps / xs and d_x / d_cond / d_add bit for bit (the gradient
    scales come from a batch amax, which the permutation does not change).  The weight gradients (the embedding's
    included) sum over the batch in another order: they are held to the parity bounds of PERM_CASE[step] against
    float64 autograd."""
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
    elif step == "fs2enc":
        hp, sd, tok, adds, g = enc_case(name)
        hp = dict(hp, dropout=0.0)
        a = fs2enc_dsx(hp, sd, tok, adds, g)[:3]
        b = fs2enc_dsx(hp, sd, tok[perm], [v[perm] for v in adds], g[perm])[:3]
        H, L = hp["hidden_size"], hp["enc_layers"]
        ones = [torch.ones(c["B"], c["T"], n, dtype=torch.bool) for n in [H] + [H, 4 * H, H] * L]
        ref = enc_ref(hp, sd, tok, adds, g, ones, EO.REL_MAX_LEN, "f64", DEV)
        used = used_rows(tok, VOCAB)
        b, ref = (b[0], b[1], embed_rows(b[2], used)), (ref[0], ref[1], embed_rows(ref[2], used))
    elif step == "durpred":
        hp, sd, x, mask, g = dur_case(name)
        hp = dict(hp, p=0.0)
        a = dur_dsx(hp, sd, x, mask, g)[:3]
        b = dur_dsx(hp, sd, x[perm], mask[perm], g[perm])[:3]
        ones = [torch.ones(c["B"], c["T"], hp["P"], dtype=torch.bool)] * hp["L"]
        ref = dur_ref(hp, sd, x, mask, g, ones, "f64", DEV)
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


def test_durpred_backward_without_d_x(lib_built):
    """d_x = NULL skips layer 0's repack and data gradient: every parameter gradient stays the same bit for bit, with
    layer 0 straight after the head (L = 1) and under four more layers (L = 5)"""
    from diffsinger_b200 import durtrain
    for L in (1, 5):
        hp = dur_hp(L=L)
        sd = dur_state_dict(SEED, 256, L, 256, 3)
        rs = np.random.RandomState(SEED)
        x = torch.from_numpy(rs.standard_normal((3, 129, 256)).astype(np.float32)).to(DEV)
        g = torch.from_numpy(rs.standard_normal((3, 129)).astype(np.float32)).to(DEV)
        mask = torch.zeros(3, 129, dtype=torch.uint8, device=DEV)
        mask[1, 97:] = 1
        m = dur_module(hp, sd)
        step = m._dsx_train_step()
        params = [dict(m.named_parameters())[n].detach() for n in durtrain.param_names(L)]
        _, tape = step.forward(params, x, mask, 0.5, SEED)
        ga, dxa = step.backward(params, tape, g, 3, 129)
        gb, dxb = step.backward(params, tape, g, 3, 129, want_x=False)
        assert dxb is None and dxa.abs().sum() > 0
        assert all(torch.equal(u, v) for u, v in zip(ga, gb)), L


# ---- the embedding gradient's sort ---------------------------------------------------------------------------------
RUNS = [63, 1, 1, 63, 64, 65, 127, 2, 62, 64]    # sorted run lengths: runs end at 63, 64, 65, 128, 192, 257, 384, ...
SORT_F = {1: (1, 1), 65: (1, 65), 1025: (5, 205), 4097: (17, 241), 2 ** 18 + 1: (481, 545)}     # F: (B, T)


def sort_layout(kind, F, seed=SEED):
    """(tokens [F] int64, vocab): token layouts for the embedding gradient's sort of (token, frame) keys, shuffled over
    the frames so that the sort has work to do.
      one_id        id 7 on every frame (vocab VOCAB);
      distinct      ids 1..F, each on one frame (vocab F + 1);
      runs          runs of RUNS' lengths (cycled) of ids 1, 2, ...: in sorted order, runs end at positions 63, 64, 65
                    and at 64-frame chunk ends (128, 192, 384, ...);
      out_of_range  the runs layout with every fifth frame padding (0), an id at or above vocab, or a negative id, which
                    sort with the padding as token 0."""
    rs = np.random.RandomState(seed)
    if kind == "one_id":
        tok, V = np.full(F, 7), VOCAB
    elif kind == "distinct":
        tok, V = np.arange(1, F + 1), F + 1
    else:
        lengths, n = [], 0
        while n < F:
            lengths.append(min(RUNS[len(lengths) % len(RUNS)], F - n))
            n += lengths[-1]
        tok, V = np.repeat(np.arange(1, len(lengths) + 1), lengths), len(lengths) + 1
        if kind == "out_of_range":
            bad = np.arange(F) % 5 == 4
            tok[bad] = np.array([0, V, V + 1000, -1, -(2 ** 40)])[rs.randint(0, 5, bad.sum())]
    return torch.from_numpy(tok[rs.permutation(F)].astype(np.int64)), V


def sorted_runs(tok, V):
    """(the sorted keys' tokens, the run ends [positions]) of the kernel's sort: ids outside [1, V) count as token 0"""
    key = torch.where((tok > 0) & (tok < V), tok, torch.zeros_like(tok))
    order = torch.argsort(key * tok.numel() + torch.arange(tok.numel()))
    k = key[order]
    ends = (torch.nonzero(k[1:] != k[:-1]).view(-1) + 1).tolist() + [tok.numel()]
    return k, ends


@pytest.mark.parametrize("F", list(SORT_F))
@pytest.mark.parametrize("kind", ["one_id", "distinct", "runs", "out_of_range"])
def test_embedding_gradient_is_the_sum_of_d_add(lib_built, kind, F):
    """dE[v] = sqrt(H) times the sum of the step's own d_add over the frames with token v, against a float64 index_add
    of that d_add, on token layouts built for the bitonic sort (F up to 2^18 + 1 runs every k_et_sort_step stride up to
    2^18).  Each element of a row of n frames is held to (68 + n / 64) 2^-24 times the sum of the |terms|: the
    kernel sums each run's piece of a 64-frame sorted chunk in order, then the row's pieces in chunk order, in fp32.
    Row 0 and rows without a frame are exactly 0; ids outside [0, vocab) add nothing to dE and still get d_add.
    H 64 (sqrt(H) = 8 scales exactly), 1 head, L 1, p 0.1; the relative position term for one_id and distinct, the
    sinusoidal one for runs and out_of_range."""
    import math
    from diffsinger_b200 import FastspeechEncoder, fs2enctrain
    B, T = SORT_F[F]
    tok, V = sort_layout(kind, F)
    tok = tok.view(B, T).to(DEV)
    rel = kind in ("one_id", "distinct")
    hp = enc_hp(64, 1, L=1, rel=rel)
    sd = EO.random_state_dict(SEED + 1, hp, V, midi=False)
    m = FastspeechEncoder(torch.nn.Embedding(V, 64, 0), 64, 1, 9, num_heads=1, hparams=dict(hp, dsx_train=True))
    m.load_state_dict(EO.sub(sd, "encoder."), strict=True)
    m = m.train().to(DEV)
    step = m._dsx_train_step()
    params = [dict(m.named_parameters())[n].detach() for n in fs2enctrain.param_names(1, 'SAME')]
    g = torch.from_numpy(np.random.RandomState(SEED + 2).standard_normal((B, T, 64)).astype(np.float32)).to(DEV)
    _, tape = step.forward(params, tok, [None] * 3, max(T, EO.REL_MAX_LEN), 0.1, SEED)
    grads, d_add = step.backward(params, tape, g, B, T, want_add=True)
    dE = grads[-1].double()
    flat_tok, terms = tok.view(-1), math.sqrt(64) * d_add.double().view(-1, 64)
    ok = (flat_tok > 0) & (flat_tok < V)
    assert (d_add.view(-1, 64)[flat_tok == 0] == 0).all()
    oor = (flat_tok != 0) & ~ok
    assert (d_add.view(-1, 64)[oor].abs().amax(-1) > 0).all()
    rows = flat_tok[ok]
    ref = torch.zeros(V, 64, dtype=torch.float64, device=DEV).index_add_(0, rows, terms[ok])
    absum = torch.zeros(V, 64, dtype=torch.float64, device=DEV).index_add_(0, rows, terms[ok].abs())
    n = torch.bincount(rows, minlength=V).double()[:, None]
    assert (dE[0] == 0).all() and (dE[n[:, 0] == 0] == 0).all()
    err = (dE - ref).abs()
    bound = (68 + n / 64) * 2.0 ** -24 * absum
    worst = (err / bound.clamp_min(1e-300)).max().item()
    print(f"\nembedding gradient {kind} F {F}: {int((n > 0).sum())} rows, worst error / bound {worst:.2e}")
    assert (err <= bound).all(), worst
