"""TEST INFRASTRUCTURE ONLY -- pins oracle/fs2dec_oracle.py to the LIVE reference FastSpeech2 decoder (needs a checkout
of the reference: DSX_REFERENCE_ROOT) and writes tests/golden/fs2_decoder.npz.
Run:  DSX_REFERENCE_ROOT=<checkout> python oracle/gen_golden_fs2dec.py

The reference's FastspeechDecoder (modules/fastspeech/tts_modules.py:350-357) is imported unmodified (stubs only for
librosa / pycwt) and built under usr/configs/popcs_ds_beta6.yaml at the shipped size (hidden 256, 4 layers, 2 heads,
kernel 9, GELU, 'SAME').  Its parameters are oracle.fs2dec_oracle.random_state_dict(SEED), loaded strictly; the oracle
must reproduce its output bit for bit.  The weights (46 MB in fp32) are not stored, only per-tensor float64 checksums
of them; the tests regenerate them from the seed.  Input: B = 2, T = 100 (not a multiple of 64), oracle.fixture_input:
utterance 0 with one frame whose channel 0 alone is 0 and one all-zero frame inside, utterance 1 zero from frame 73."""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import fs2dec_oracle as O  # noqa: E402

REF_ROOT = os.environ.get("DSX_REFERENCE_ROOT", "")
CONFIG = "usr/configs/popcs_ds_beta6.yaml"
HP_KEYS = ("hidden_size", "dec_layers", "dec_ffn_kernel_size", "num_heads", "ffn_padding", "ffn_act", "dropout")
SEED, INPUT_SEED, B, T, TAIL = 11, 12, 2, 100, 73


def load_reference():
    sys.dont_write_bytecode = True
    for n in ("librosa", "librosa.filters", "pycwt"):
        sys.modules.setdefault(n, types.ModuleType(n))
    sys.modules["pycwt"].wavelet = None
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    cwd = os.getcwd()
    os.chdir(REF_ROOT)          # configs use repo-relative base_config paths
    try:
        from utils.hparams import hparams, set_hparams
        set_hparams(config=CONFIG, exp_name="", print_hparams=False)
        from modules.fastspeech.tts_modules import FastspeechDecoder
    finally:
        os.chdir(cwd)
    return hparams, FastspeechDecoder


def main():
    assert REF_ROOT and os.path.isdir(REF_ROOT), "set DSX_REFERENCE_ROOT to a checkout of the reference"
    hparams, FastspeechDecoder = load_reference()
    hp = {k: hparams[k] for k in HP_KEYS}
    assert (hp["hidden_size"], hp["dec_layers"], hp["num_heads"], hp["dec_ffn_kernel_size"], hp["ffn_act"]) == \
        (256, 4, 2, 9, "gelu"), hp
    dec = FastspeechDecoder().eval()
    sd = O.random_state_dict(SEED, hp)
    assert {k: tuple(v.shape) for k, v in dec.state_dict().items()} == {k: tuple(v.shape) for k, v in sd.items()}
    dec.load_state_dict(sd, strict=True)
    x = O.fixture_input(INPUT_SEED, B, T, hp["hidden_size"], tail=TAIL)
    with torch.no_grad():
        ref = dec(x)
        mine = O.decoder(sd, x, hp)
    print(f"oracle vs live reference: max |d| = {(ref - mine).abs().max().item():.3e}")
    assert torch.equal(ref, mine), "the oracle must reproduce the reference bit for bit"
    pad = O.padding_mask(x)
    assert pad[0].sum() == 1 and pad[1].sum() == T - TAIL and (ref[pad] == 0).all()
    out = os.path.join(ROOT, "tests", "golden", "fs2_decoder.npz")
    np.savez_compressed(out, x=x.numpy(), out=ref.numpy(), seed=np.int64(SEED), input_seed=np.int64(INPUT_SEED),
                        **{"hp." + k: np.asarray(v) for k, v in hp.items()},
                        **{"cks." + k: v for k, v in O.checksums(sd).items()})
    print("wrote", out, os.path.getsize(out) // 1024, "KB;", sum(v.numel() for v in sd.values()), "state-dict values")


if __name__ == "__main__":
    main()
