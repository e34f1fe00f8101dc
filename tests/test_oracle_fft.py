"""CPU: the FFT-denoiser oracle (oracle/fft_oracle.py) reproduces the reference's evaluations and sampling loops stored in
tests/golden/fft_denoiser.npz (written by oracle/gen_golden_fft.py from the unmodified reference), over the state dict and
step noise regenerated from the fixture's seeds."""
import numpy as np
import torch

from conftest import golden
from oracle import diffnet_oracle as N
from oracle import fft_oracle as O
from oracle import fs2dec_oracle as D


def fixture():
    g = golden("fft_denoiser.npz")
    hp = {k[3:]: g[k].item() for k in g.files if k.startswith("hp.")}
    return g, hp, O.random_state_dict(int(g["seed"]), hp)


def schedule(g):
    return N.make_schedule(N.linear_beta_schedule(int(g["timesteps"]), float(g["max_beta"])))


def close(out, ref):
    out, ref = np.asarray(out), np.asarray(ref)
    assert np.abs(out - ref).max() <= 1e-5 * np.abs(ref).max(), np.abs(out - ref).max()


def test_regenerated_state_dict_matches_the_checksums():
    g, hp, sd = fixture()
    stored = {k[4:]: g[k] for k in g.files if k.startswith("cks.")}
    assert set(stored) == set(sd) and len(sd) == 54
    for k, v in D.checksums(sd).items():
        np.testing.assert_allclose(v, stored[k], rtol=1e-12, atol=1e-12, err_msg=k)
    assert list(sd) == list(O.state_dict_shapes(hp))


def test_regenerated_step_noise_matches_the_checksum():
    g, hp, _ = fixture()
    B, T = g["cond_loop"].shape[0], g["cond_loop"].shape[2]
    noise = O.step_noise(int(g["noise_seed"]), int(g["K_step"]), B, T)
    np.testing.assert_allclose(noise.double().sum().item(), float(g["noise_checksum"]), rtol=1e-12)


def test_oracle_reproduces_the_evaluations():
    g, hp, sd = fixture()
    assert g["t"][2, 0] != g["t"][2, 1]                    # one batch with a t per utterance
    with torch.no_grad():
        for i, t in enumerate(g["t"]):
            close(O.forward(sd, torch.from_numpy(g["spec"]), torch.from_numpy(t), torch.from_numpy(g["cond"]), hp),
                  g["eps"][i])


def test_oracle_reproduces_the_ddpm_infer_loop():
    g, hp, sd = fixture()
    B, T = g["cond_loop"].shape[0], g["cond_loop"].shape[2]
    K = int(g["K_step"])
    f = torch.from_numpy
    with torch.no_grad():
        out = O.infer_loop(lambda *a: O.forward(sd, *a, hp), schedule(g), f(g["cond_loop"]), K, f(g["spec_min"]),
                           f(g["spec_max"]), fs2_mel=f(g["fs2_mel"]), start_noise=f(g["start_noise"]),
                           step_noise=O.step_noise(int(g["noise_seed"]), K, B, T), mel2ph=f(g["mel2ph"]))
    close(out, g["mel_ddpm"])
    pad = g["mel2ph"] == 0
    assert pad.any() and (g["mel_ddpm"][pad] == 0).all()


def test_oracle_reproduces_the_plms_infer_loop():
    g, hp, sd = fixture()
    f = torch.from_numpy
    with torch.no_grad():
        out = O.infer_loop(lambda *a: O.forward(sd, *a, hp), schedule(g), f(g["cond_plms"]), int(g["K_step"]),
                           f(g["spec_min"]), f(g["spec_max"]), fs2_mel=f(g["fs2_mel_plms"]),
                           start_noise=f(g["start_noise_plms"]), pndm_speedup=int(g["interval"]))
    close(out, g["mel_plms"])


def test_fixture_configuration():
    g, hp, _ = fixture()
    assert (hp["hidden_size"], hp["dec_layers"], hp["num_heads"], hp["dec_ffn_kernel_size"]) == (256, 4, 2, 9)
    assert (hp["residual_channels"], hp["audio_num_mel_bins"], hp["ffn_padding"], hp["ffn_act"]) == (256, 80, "SAME", "gelu")
    assert (int(g["K_step"]), int(g["timesteps"]), g["cond_plms"].shape[0]) == (51, 100, 1)
