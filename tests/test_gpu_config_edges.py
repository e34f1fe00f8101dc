"""GPU: the shared implicit-GEMM conv core (dsx_conv.cuh) and the FastSpeech2 layer stack (dsx_fs2dec.cu) at the edges
of the configurations their front ends' *_create functions accept, against the oracles in float64 on the CPU.

Each case builds the module through its public class from seeded weights and runs a batch of B >= 2 with one padded or
shorter utterance (the sampler denoisers: a different t per utterance).  The edges are where an implicit GEMM goes
wrong: channel counts that leave a partial column tile, taps x cin not a multiple of the 64-wide K chunk, taps that
reach entirely outside the utterance, the vocoder's switch between the chained ResBlock kernel (k_chain) and one k_conv
per conv, one and three attention heads, deep stacks.  The vocoder cases run without f0: the NSF source does not depend
on these edges, and test_gpu_hifigan.py covers it.

Bounds.  Every bound is 3-5x the error of a CPU simulation of the kernels' fp16 operand rounding against the float64
oracle, on the same case (hifigan_oracle.generator(fp16=True), pe_oracle.pitch_extractor(fp16=True),
fs2enc_oracle.dur_predictor(fp16=True), fs2dec_oracle.decoder_fp16_sim, fs2enc_oracle.encoder_fp16_sim,
fft_oracle.forward_fp16_sim).  Simulated max / mean, then the bound (max / mean):

    pitch     H16_one_group               4.7e-03 /  7.4e-04   ->  2.0e-02 / 3.0e-03
    pitch     H48                         4.9e-03 /  7.1e-04   ->  2.0e-02 / 3.0e-03
    pitch     H208                        4.2e-03 /  1.1e-03   ->  2.0e-02 / 4.5e-03
    pitch     P16_under_H256              8.2e-03 /  1.2e-03   ->  3.5e-02 / 5.0e-03
    pitch     kernel1                     3.9e-03 /  1.1e-03   ->  2.0e-02 / 5.0e-03
    pitch     kernel31_T20                4.5e-03 /  1.1e-03   ->  2.0e-02 / 4.5e-03
    pitch     conv_layers16               4.3e-03 /  1.1e-03   ->  2.0e-02 / 4.5e-03
    pitch     left_kernel31               3.8e-03 /  9.5e-04   ->  2.0e-02 / 4.0e-03
    duration idim16_chans256             3.1e-03 /  5.8e-04   ->  1.5e-02 / 2.5e-03
    duration idim256_chans48             2.3e-03 /  2.4e-04   ->  9.5e-03 / 1.0e-03
    duration kernel1                     3.0e-03 /  6.9e-04   ->  1.5e-02 / 3.0e-03
    duration kernel31_same               1.8e-03 /  4.2e-04   ->  7.5e-03 / 2.0e-03
    duration left_k2                     1.5e-03 /  5.1e-04   ->  6.5e-03 / 2.5e-03
    duration layers16                    1.3e-02 /  3.4e-03   ->  5.5e-02 / 1.5e-02
    duration T1                          1.6e-03 /  1.3e-03   ->  7.0e-03 / 5.5e-03
    stack     dec_H64_heads1              1.0e-03 /  1.6e-04   ->  4.5e-03 / 7.0e-04
    stack     dec_H192_heads3_T63         1.1e-03 /  1.6e-04   ->  4.5e-03 / 6.5e-04
    stack     dec_H192_heads3_T64         1.2e-03 /  1.6e-04   ->  5.0e-03 / 6.5e-04
    stack     dec_H192_heads3_T65         1.1e-03 /  1.5e-04   ->  4.5e-03 / 6.5e-04
    stack     dec_H192_heads3_T129        1.1e-03 /  1.4e-04   ->  5.0e-03 / 6.0e-04
    stack     dec_kernel1_same            1.8e-03 /  2.5e-04   ->  7.5e-03 / 1.5e-03
    stack     dec_kernel1_left            1.8e-03 /  2.5e-04   ->  7.5e-03 / 1.5e-03
    stack     dec_kernel255_T100          9.1e-04 /  1.6e-04   ->  4.0e-03 / 6.5e-04
    stack     dec_L64_H64                 7.1e-04 /  1.1e-04   ->  3.0e-03 / 4.5e-04
    stack     enc_H64_heads1              1.3e-03 /  1.6e-04   ->  5.5e-03 / 6.5e-04
    stack     enc_H192_heads3             1.3e-03 /  1.4e-04   ->  5.5e-03 / 6.0e-04
    hifigan   one_stage_u1_k3             6.1e-04 /  1.4e-04   ->  2.5e-03 / 5.5e-04
    hifigan   two_stages_5_3_mel_only     4.4e-04 /  8.9e-05   ->  2.0e-03 / 4.0e-04
    hifigan   hop4096_u64_k128            1.7e-04 /  3.5e-05   ->  7.0e-04 / 1.5e-04
    hifigan   c0_384                      4.3e-04 /  1.1e-04   ->  2.0e-03 / 4.5e-04
    hifigan   c0_2048_T8                  1.6e-04 /  3.6e-05   ->  7.0e-04 / 1.5e-04
    hifigan   c0_16                       3.3e-04 /  1.4e-04   ->  1.5e-03 / 5.5e-04
    hifigan   num_kernels_1               3.8e-04 /  9.2e-05   ->  2.0e-03 / 4.0e-04
    hifigan   num_kernels_2               1.5e-04 /  3.6e-05   ->  6.5e-04 / 1.5e-04
    hifigan   resblock2_k31_d64           5.2e-04 /  1.4e-04   ->  2.5e-03 / 6.0e-04
    hifigan   chain_dil32                 1.3e-04 /  1.9e-05   ->  5.5e-04 / 8.0e-05
    hifigan   per_conv_dil33              1.4e-04 /  1.9e-05   ->  5.5e-04 / 7.5e-05
    hifigan   chain_centre_64             1.3e-04 /  1.9e-05   ->  5.5e-04 / 8.0e-05
    fft       residual16                  2.0e-03 /  4.0e-04   ->  8.0e-03 / 2.0e-03
    fft       residual1024                2.2e-03 /  4.2e-04   ->  9.0e-03 / 2.0e-03
    fft       hidden64                    1.6e-03 /  3.5e-04   ->  7.0e-03 / 1.5e-03
    fft       hidden192                   1.9e-03 /  3.8e-04   ->  8.0e-03 / 2.0e-03

HiFi-GAN errors are relative to the reference's peak |wav|; the pitch extractor's are in log2 Hz (channel 0) and uv
logit (channel 1), the larger of the two; the FS2 stack's and the FFT's are absolute (LayerNorm-scaled outputs up to
about 5, eps up to about 4), except the 64-layer stack, which is relative to its peak output.  The duration predictor
is held as test_gpu_fs2enc.py holds it: max distance to dur_predictor(fp16=True) on the same input (2e-2, the
LayerNorms amplify the remaining summation-order differences on a few tokens) and a mean distance to float64 over the
valid tokens.  DiffNet's tensor-core precisions keep test_diffnet_forward_golden's bounds (fp16x3 2e-4, fp16x2 7.5e-4,
max |eps| error), and its SIMT fp32 path test_error_behaviour_is_loud's 1e-5.  Padding rows and frames must be exactly
0, and uv must agree wherever the reference's |logit| exceeds the max bound."""
import numpy as np
import pytest
import torch

from conftest import HP, rs_normal
from oracle import diffnet_oracle as N
from oracle import fft_oracle as FO
from oracle import fs2dec_oracle as D
from oracle import fs2enc_oracle as E
from oracle import hifigan_oracle as HG
from oracle import pe_oracle as PE

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)


def f64(sd):
    return {k: v.double() for k, v in sd.items()}


def errors(out, ref, scale=1.0):
    d = np.abs(np.asarray(out, np.float64) - np.asarray(ref, np.float64)) / scale
    return d.max(), d.mean()


def within(out, ref, bound, scale=1.0):
    mx, mean = errors(out, ref, scale)
    assert np.isfinite(np.asarray(out)).all()
    assert mx <= bound[0] and mean <= bound[1], (mx, mean, bound)


# ---- HiFi-GAN -----------------------------------------------------------------------------------------------------
def hifigan_hp(**over):
    return dict(HG.HPARAMS_TTS, **over)


RB1_K3 = dict(resblock_kernel_sizes=[3])
HIFIGAN = {
    # one stage: a transposed conv with u = 1 (three taps), one ResBlock kernel; 32 channels on the chain
    "one_stage_u1_k3": dict(h=hifigan_hp(upsample_rates=[1], upsample_kernel_sizes=[3], upsample_initial_channel=64,
                                         resblock_kernel_sizes=[3], resblock_dilation_sizes=[[1, 3, 5]]), T=40),
    # odd rates, the mel-only generator (no noise_convs / m_source); 64 and 32 channels on the chain
    "two_stages_5_3_mel_only": dict(h=hifigan_hp(upsample_rates=[5, 3], upsample_kernel_sizes=[15, 9],
                                                 use_pitch_embed=False), T=30),
    # hop 4096: 128 taps of a u = 64 transposed conv over 16 and 8 channels
    "hop4096_u64_k128": dict(h=hifigan_hp(upsample_rates=[64, 64], upsample_kernel_sizes=[128, 128],
                                          upsample_initial_channel=32), T=6),
    # stages of 192 / 96 / 48 / 24 channels: 96 and 48 run per conv with a partial column tile, 24 pads to 32 on the chain
    "c0_384": dict(h=hifigan_hp(upsample_initial_channel=384), T=12),
    "c0_2048_T8": dict(h=hifigan_hp(upsample_initial_channel=2048, **RB1_K3, resblock_dilation_sizes=[[1, 3, 5]]), T=8),
    # stages of 8 / 4 / 2 / 1 channels: every stage pads to 16, the last stage has one real channel
    "c0_16": dict(h=hifigan_hp(upsample_initial_channel=16), T=12),
    "num_kernels_1": dict(h=hifigan_hp(resblock_kernel_sizes=[7], resblock_dilation_sizes=[[1, 3, 5]]), T=12),
    "num_kernels_2": dict(h=hifigan_hp(resblock_kernel_sizes=[3, 11], resblock_dilation_sizes=[[1, 3, 5]] * 2), T=12),
    # ResBlock2, k = 31 at dilation 64: every tap but the centre one lies outside the 40- and 80-sample stages
    "resblock2_k31_d64": dict(h=hifigan_hp(resblock="2", upsample_rates=[2, 2], upsample_kernel_sizes=[4, 4],
                                           upsample_initial_channel=64, resblock_kernel_sizes=[31],
                                           resblock_dilation_sizes=[[64, 1]]), T=20),
    # the chain boundary: -tap0 = 32 (chained), 33 (per conv), and a halo of 96 that leaves exactly 64 centre rows;
    # three lengths over stages that span several 256-row tiles
    "chain_dil32": dict(h=hifigan_hp(**RB1_K3, resblock_dilation_sizes=[[32, 1, 1]]), T=20, lengths=[20, 13, 5]),
    "per_conv_dil33": dict(h=hifigan_hp(**RB1_K3, resblock_dilation_sizes=[[33, 1, 1]]), T=20, lengths=[20, 13, 5]),
    "chain_centre_64": dict(h=hifigan_hp(**RB1_K3, resblock_dilation_sizes=[[31, 31, 31]]), T=20, lengths=[20, 13, 5]),
}


def hifigan_case(name):
    """(h, state dict, mel [B, 80, T], lengths or None): the reference's own initialisation from a fixed seed"""
    from diffsinger_b200 import HifiGanGenerator
    c = HIFIGAN[name]
    torch.manual_seed(1)
    m = HifiGanGenerator(c["h"])
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    B = len(c.get("lengths", [0, 0]))
    mel = torch.randn(B, 80, c["T"], generator=torch.Generator().manual_seed(2))
    return c["h"], sd, mel, c.get("lengths")


def hifigan_ref(h, sd, mel, lengths, fp16=False):
    """float64 generator per utterance over its own frames: [B, 1, T * hop], zero after an utterance's length"""
    hop = int(np.prod(h["upsample_rates"]))
    B, _, T = mel.shape
    lens = lengths or [T] * B
    out = torch.zeros(B, 1, T * hop, dtype=torch.float64)
    sd64 = f64(sd)
    with torch.no_grad():
        for b, L in enumerate(lens):
            out[b, :, :L * hop] = HG.generator(sd64, h, mel[b:b + 1, :, :L].double(), fp16=fp16)[0]
    return out


# ---- pitch extractor ----------------------------------------------------------------------------------------------
PITCH = {
    "H16_one_group": dict(hp=dict(hidden_size=16)),
    "H48": dict(hp=dict(hidden_size=48)),
    "H208": dict(hp=dict(hidden_size=208)),
    "P16_under_H256": dict(hp=dict(predictor_hidden=16)),
    "kernel1": dict(hp=dict(predictor_kernel=1)),
    "kernel31_T20": dict(hp=dict(predictor_kernel=31), T=20),
    "conv_layers16": dict(hp=dict(hidden_size=64), L=16),
    "left_kernel31": dict(hp=dict(predictor_kernel=31, ffn_padding='LEFT')),
}


def pitch_case(name):
    """(hp, conv layers, state dict, mel [B, T, 80] with a zero-padded tail on utterance 1)"""
    from diffsinger_b200 import PitchExtractor
    c = PITCH[name]
    hp, L, T = dict(PE.HPARAMS_E2E, **c["hp"]), c.get("L", 2), c.get("T", 64)
    torch.manual_seed(3)
    sd = PE.random_state_dict(PitchExtractor(80, L, hparams=hp).state_dict(), 4)
    mel = torch.randn(3, T, 80, generator=torch.Generator().manual_seed(5)) * 1.5 - 4.0
    mel[1, T - T // 4:] = 0
    return hp, L, sd, mel


def pitch_ref(hp, L, sd, mel, fp16=False):
    with torch.no_grad():
        return PE.pitch_extractor(f64(sd), mel.double(), hp, L, fp16=fp16)


# ---- duration predictor -------------------------------------------------------------------------------------------
DURATION = {
    "idim16_chans256": dict(idim=16, chans=256),
    "idim256_chans48": dict(idim=256, chans=48),
    "kernel1": dict(k=1),
    "kernel31_same": dict(k=31),
    "left_k2": dict(k=2, padding='LEFT'),
    "layers16": dict(layers=16, chans=64),
    "T1": dict(T=1),
}


def duration_case(name):
    """(hp, state dict, x [B, T, idim] zero on the padding tokens, mask [B, T]); weights as fs2enc_oracle seeds them"""
    c = DURATION[name]
    idim, C = c.get("idim", 256), c.get("chans", 256)
    hp = dict(E.HPARAMS_MIDI, hidden_size=idim, predictor_hidden=C, dur_predictor_kernel=c.get("k", 3),
              dur_predictor_layers=c.get("layers", 5), ffn_padding=c.get("padding", 'SAME'))
    sd = E.sub(E.random_state_dict(6, hp, 11, midi=False), "dur_predictor.")
    T = c.get("T", 50)
    x = torch.from_numpy(np.random.RandomState(7).standard_normal((3, T, idim)).astype(np.float32))
    mask = torch.zeros(3, T, dtype=torch.bool)
    if T > 1:
        mask[1, T - T // 4:] = True
        mask[2, T // 2:] = True
    x[mask] = 0
    return hp, sd, x, mask


# ---- FS2 decoder / encoder ----------------------------------------------------------------------------------------
def dec_hp(**over):
    return dict(D.HPARAMS_POPCS, **over)


STACK = {
    "dec_H64_heads1": dict(hp=dec_hp(hidden_size=64, num_heads=1), T=100),
    "dec_H192_heads3_T63": dict(hp=dec_hp(hidden_size=192, num_heads=3), T=63),
    "dec_H192_heads3_T64": dict(hp=dec_hp(hidden_size=192, num_heads=3), T=64),
    "dec_H192_heads3_T65": dict(hp=dec_hp(hidden_size=192, num_heads=3), T=65),
    "dec_H192_heads3_T129": dict(hp=dec_hp(hidden_size=192, num_heads=3), T=129),
    "dec_kernel1_same": dict(hp=dec_hp(dec_ffn_kernel_size=1), T=100),
    "dec_kernel1_left": dict(hp=dec_hp(dec_ffn_kernel_size=1, ffn_padding='LEFT'), T=100),
    "dec_kernel255_T100": dict(hp=dec_hp(hidden_size=64, num_heads=1, dec_ffn_kernel_size=255), T=100),
    "dec_L64_H64": dict(hp=dec_hp(hidden_size=64, num_heads=1, dec_layers=64), T=80, relative=True),
    "enc_H64_heads1": dict(hp=dec_hp(hidden_size=64, num_heads=1), T=65, encoder=True),
    "enc_H192_heads3": dict(hp=dec_hp(hidden_size=192, num_heads=3), T=129, encoder=True),
}


def stack_case(name):
    """(hp, state dict, input): decoder input x [B, T, H] with a padded tail, or encoder tokens [B, T]"""
    c = STACK[name]
    hp, T = c["hp"], c["T"]
    if c.get("encoder"):
        ehp = dict(E.HPARAMS_POPCS, hidden_size=hp["hidden_size"], num_heads=hp["num_heads"])
        sd = E.sub(E.random_state_dict(8, ehp, 31, midi=False), "encoder.")
        tok = E.fixture_inputs(9, 3, T, [None, T - T // 4, T // 2], 31)[0]
        return ehp, sd, tok
    return hp, D.random_state_dict(21, hp), D.fixture_input(22, 3, T, hp["hidden_size"], tail=T - T // 4)


def stack_ref(name, hp, sd, inp, fp16=False):
    with torch.no_grad():
        if STACK[name].get("encoder"):
            return (E.encoder_fp16_sim(sd, inp, hp) if fp16 else E.encoder(f64(sd), inp, hp)).double()
        return (D.decoder_fp16_sim(sd, inp, hp) if fp16 else D.decoder(f64(sd), inp.double(), hp)).double()


# ---- FFT denoiser -------------------------------------------------------------------------------------------------
FFT = {
    "residual16": dict(residual_channels=16),
    "residual1024": dict(residual_channels=1024),
    "hidden64": dict(hidden_size=64, num_heads=1),
    "hidden192": dict(hidden_size=192, num_heads=3),
}


def fft_case(name):
    """(hp, state dict, spec [B, 1, 80, T], t [B], cond [B, H, T])"""
    hp = dict(FO.HPARAMS_POPCS, **FFT[name])
    sd = FO.random_state_dict(51, hp)
    gen = torch.Generator().manual_seed(52)
    T = 90
    spec = torch.randn(3, 1, 80, T, generator=gen)
    cond = torch.randn(3, hp["hidden_size"], T, generator=gen)
    return hp, sd, spec, torch.tensor([99, 40, 0]), cond


def fft_ref(hp, sd, spec, t, cond, fp16=False):
    with torch.no_grad():
        if fp16:
            return FO.forward_fp16_sim(sd, spec, t, cond, hp).double()
        return FO.forward(f64(sd), spec.double(), t.double(), cond.double(), hp)


# ---- simulated errors and the bounds derived from them ------------------------------------------------------------
BOUNDS = {   # (max, mean), about 4x the simulated errors listed in the docstring
    ("pitch", "H16_one_group"): (2.0e-02, 3.0e-03),
    ("pitch", "H48"): (2.0e-02, 3.0e-03),
    ("pitch", "H208"): (2.0e-02, 4.5e-03),
    ("pitch", "P16_under_H256"): (3.5e-02, 5.0e-03),
    ("pitch", "kernel1"): (2.0e-02, 5.0e-03),
    ("pitch", "kernel31_T20"): (2.0e-02, 4.5e-03),
    ("pitch", "conv_layers16"): (2.0e-02, 4.5e-03),
    ("pitch", "left_kernel31"): (2.0e-02, 4.0e-03),
    ("duration", "idim16_chans256"): (1.5e-02, 2.5e-03),
    ("duration", "idim256_chans48"): (9.5e-03, 1.0e-03),
    ("duration", "kernel1"): (1.5e-02, 3.0e-03),
    ("duration", "kernel31_same"): (7.5e-03, 2.0e-03),
    ("duration", "left_k2"): (6.5e-03, 2.5e-03),
    ("duration", "layers16"): (5.5e-02, 1.5e-02),
    ("duration", "T1"): (7.0e-03, 5.5e-03),
    ("stack", "dec_H64_heads1"): (4.5e-03, 7.0e-04),
    ("stack", "dec_H192_heads3_T63"): (4.5e-03, 6.5e-04),
    ("stack", "dec_H192_heads3_T64"): (5.0e-03, 6.5e-04),
    ("stack", "dec_H192_heads3_T65"): (4.5e-03, 6.5e-04),
    ("stack", "dec_H192_heads3_T129"): (5.0e-03, 6.0e-04),
    ("stack", "dec_kernel1_same"): (7.5e-03, 1.5e-03),
    ("stack", "dec_kernel1_left"): (7.5e-03, 1.5e-03),
    ("stack", "dec_kernel255_T100"): (4.0e-03, 6.5e-04),
    ("stack", "dec_L64_H64"): (3.0e-03, 4.5e-04),
    ("stack", "enc_H64_heads1"): (5.5e-03, 6.5e-04),
    ("stack", "enc_H192_heads3"): (5.5e-03, 6.0e-04),
    ("hifigan", "one_stage_u1_k3"): (2.5e-03, 5.5e-04),
    ("hifigan", "two_stages_5_3_mel_only"): (2.0e-03, 4.0e-04),
    ("hifigan", "hop4096_u64_k128"): (7.0e-04, 1.5e-04),
    ("hifigan", "c0_384"): (2.0e-03, 4.5e-04),
    ("hifigan", "c0_2048_T8"): (7.0e-04, 1.5e-04),
    ("hifigan", "c0_16"): (1.5e-03, 5.5e-04),
    ("hifigan", "num_kernels_1"): (2.0e-03, 4.0e-04),
    ("hifigan", "num_kernels_2"): (6.5e-04, 1.5e-04),
    ("hifigan", "resblock2_k31_d64"): (2.5e-03, 6.0e-04),
    ("hifigan", "chain_dil32"): (5.5e-04, 8.0e-05),
    ("hifigan", "per_conv_dil33"): (5.5e-04, 7.5e-05),
    ("hifigan", "chain_centre_64"): (5.5e-04, 8.0e-05),
    ("fft", "residual16"): (8.0e-03, 2.0e-03),
    ("fft", "residual1024"): (9.0e-03, 2.0e-03),
    ("fft", "hidden64"): (7.0e-03, 1.5e-03),
    ("fft", "hidden192"): (8.0e-03, 2.0e-03),
}


# ---- the tests ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(HIFIGAN))
def test_hifigan(lib_built, case):
    from diffsinger_b200 import HifiGanGenerator
    h, sd, mel, lengths = hifigan_case(case)
    m = HifiGanGenerator(h)
    m.load_state_dict(sd, strict=True)
    m = m.to(DEV)
    with torch.no_grad():
        lens = None if lengths is None else torch.tensor(lengths, dtype=torch.int32, device=DEV)
        wav = m(mel.to(DEV), lengths=lens).cpu()
    ref = hifigan_ref(h, sd, mel, lengths)
    within(wav, ref, BOUNDS["hifigan", case], ref.abs().max().item())
    hop = int(np.prod(h["upsample_rates"]))
    for b, L in enumerate(lengths or []):
        assert torch.count_nonzero(wav[b, :, L * hop:]) == 0, b


@pytest.mark.parametrize("case", list(PITCH))
def test_pitch_extractor(lib_built, case):
    from diffsinger_b200 import PitchExtractor
    hp, L, sd, mel = pitch_case(case)
    m = PitchExtractor(80, L, hparams=hp)
    m.load_state_dict(sd, strict=True)
    with torch.no_grad():
        r = m.eval().to(DEV)(mel.to(DEV))
    pitch, f0 = r['pitch_pred'].cpu().double(), r['f0_denorm_pred'].cpu()
    ref, _ = pitch_ref(hp, L, sd, mel)
    bound = BOUNDS["pitch", case]
    for ch in range(2):
        within(pitch[..., ch], ref[..., ch], bound)
    pad = PE.padding_mask(mel)
    assert (f0[pad] == 0).all() and (f0[~pad] >= 0).all()
    sure = ref[..., 1].abs() > bound[0]
    assert ((pitch[..., 1] > 0) == (ref[..., 1] > 0))[sure].all()


@pytest.mark.parametrize("case", list(DURATION))
def test_duration_predictor(lib_built, case):
    from diffsinger_b200 import DurationPredictor
    hp, sd, x, mask = duration_case(case)
    dp = DurationPredictor(hp['hidden_size'], n_layers=hp['dur_predictor_layers'], n_chans=hp['predictor_hidden'],
                           kernel_size=hp['dur_predictor_kernel'], padding=hp['ffn_padding'], hparams=hp)
    dp.load_state_dict(sd, strict=True)
    with torch.no_grad():
        xs = dp.eval().to(DEV)(x.to(DEV), mask.to(DEV)).cpu().double()
        sim = E.dur_predictor(sd, x, mask, hp, fp16=True).squeeze(-1).double()
        ref = E.dur_predictor(f64(sd), x.double(), mask, hp).squeeze(-1)
    assert (xs - sim).abs().max().item() <= 2e-2
    assert (xs - ref).abs()[~mask].mean().item() <= BOUNDS["duration", case][1]
    assert (xs[mask] == 0).all()


@pytest.mark.parametrize("case", list(STACK))
def test_fs2_stack(lib_built, case):
    import diffsinger_b200 as dsx
    hp, sd, inp = stack_case(case)
    if STACK[case].get("encoder"):
        H = hp['hidden_size']
        m = dsx.FastspeechEncoder(torch.nn.Embedding(31, H, 0), H, hp['enc_layers'], hp['enc_ffn_kernel_size'],
                                  num_heads=hp['num_heads'], hparams=hp)
        pad = inp == 0
    else:
        m = dsx.FastspeechDecoder(hparams=hp)
        pad = D.padding_mask(inp)
    m.load_state_dict(sd, strict=True)
    with torch.no_grad():
        out = m.eval().to(DEV)(inp.to(DEV)).cpu()
    ref = stack_ref(case, hp, sd, inp)
    scale = ref.abs().max().item() if STACK[case].get("relative") else 1.0
    within(out, ref, BOUNDS["stack", case], scale)
    assert (out[pad] == 0).all()


@pytest.mark.parametrize("case", list(FFT))
def test_fft_denoiser(lib_built, case):
    from diffsinger_b200 import FFT as FFTModule
    hp, sd, spec, t, cond = fft_case(case)
    m = FFTModule(hparams=hp)
    m.load_state_dict(sd, strict=True)
    with torch.no_grad():
        out = m.eval().to(DEV)(spec.to(DEV), t.to(DEV), cond.to(DEV)).cpu()
    within(out, fft_ref(hp, sd, spec, t, cond), BOUNDS["fft", case])


def diffnet(hp, seed=0):
    import diffsinger_b200 as dsx
    torch.manual_seed(seed)
    net = dsx.DiffNet(80, hparams=hp)
    torch.nn.init.normal_(net.output_projection.weight, std=0.02)
    return net


def diffnet_ref(net, spec, t, cond, cycle):
    sd = {k: v.detach().cpu().double() for k, v in net.state_dict().items()}
    with torch.no_grad():
        return N.diffnet_forward(sd, spec.double(), t.double(), cond.double(), cycle)


@pytest.mark.parametrize("prec,tol", [("fp16x3", 2e-4), ("fp16x2", 7.5e-4)])
@pytest.mark.parametrize("cycle", [2, 3])
def test_diffnet_dilation_cycles(lib_built, cycle, prec, tol):
    import diffsinger_b200 as dsx
    net = diffnet(dict(HP, dilation_cycle_length=cycle))
    B, T = 3, 333
    spec, cond, t = rs_normal(71, (B, 1, 80, T)), rs_normal(72, (B, 256, T)), torch.tensor([3, 50, 99])
    s = dsx.DsxSampler(net.to(DEV).eval(), prec, cycle)
    s.ensure_weights(DEV)
    eps = s.diffnet_forward(spec.to(DEV), t.to(DEV), cond.to(DEV)).cpu()
    s.close()
    assert (eps.double() - diffnet_ref(net, spec, t, cond, cycle)).abs().max().item() < tol


@pytest.mark.parametrize("C,H,L,T", [(48, 48, 3, 77), (48, 96, 5, 130), (320, 256, 5, 101)])
def test_diffnet_simt_channel_counts(lib_built, C, H, L, T):
    import diffsinger_b200 as dsx
    net = diffnet(dict(HP, residual_channels=C, hidden_size=H, residual_layers=L))
    spec, cond, t = rs_normal(73, (2, 1, 80, T)), rs_normal(74, (2, H, T)), torch.tensor([7, 88])
    s = dsx.DsxSampler(net.to(DEV).eval(), "fp32", 1)
    eps = s.diffnet_forward(spec.to(DEV), t.to(DEV), cond.to(DEV)).cpu()
    s.close()
    assert (eps.double() - diffnet_ref(net, spec, t, cond, 1)).abs().max().item() < 1e-5
