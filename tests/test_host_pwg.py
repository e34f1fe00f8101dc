"""CPU: the Parallel WaveGAN generator mirror (diffsinger_b200.ParallelWaveGANGenerator) has the reference's constructor,
initialisation and state-dict surface, loads the reference fixtures in both weight forms, has no CPU path, and refuses
each constructor option the kernels do not implement by name."""
import pytest
import torch

from pwg_cases import FIXTURES, fixture, plain


@pytest.mark.parametrize("name", FIXTURES)
def test_state_dict_matches_the_reference(lib_built, name):
    """same names and shapes; and under the fixture's seed the reference's own initialisation, bit for bit"""
    from diffsinger_b200 import ParallelWaveGANGenerator
    g, sd, cfg = fixture(name)
    torch.manual_seed(int(g["weight_seed"]))
    m = ParallelWaveGANGenerator(**cfg)
    mine = m.state_dict()
    assert {k: tuple(v.shape) for k, v in mine.items()} == {k: tuple(v.shape) for k, v in sd.items()}
    for k, v in mine.items():
        assert torch.equal(v, sd[k]), k


@pytest.mark.parametrize("name", FIXTURES)
def test_loading_in_both_weight_forms(lib_built, name):
    from diffsinger_b200 import ParallelWaveGANGenerator
    _, sd, cfg = fixture(name)
    m = ParallelWaveGANGenerator(**cfg)
    m.load_state_dict(sd, strict=True)
    m.remove_weight_norm()                   # the reference's self.apply(remove_weight_norm) pattern
    p = plain(sd)
    assert set(m.state_dict()) == set(p)
    assert not any(k.endswith((".weight_g", ".weight_v")) for k in m.state_dict())
    m2 = ParallelWaveGANGenerator(**cfg)
    m2.remove_weight_norm()
    m2.load_state_dict(p, strict=True)
    for k, v in m.state_dict().items():
        assert torch.allclose(v, m2.state_dict()[k], rtol=1e-6, atol=1e-7), k
    fake_task = torch.nn.Module()            # vocoders/pwg.py's custom-checkpoint path
    fake_task.model_gen = ParallelWaveGANGenerator(**cfg)
    missing, unexpected = fake_task.load_state_dict({"model_gen." + k: v for k, v in sd.items()}, strict=False)
    assert not missing and not unexpected
    fake_task.model_gen.remove_weight_norm()
    assert fake_task.model_gen.eval() is fake_task.model_gen


def test_cpu_tensors_raise(lib_built):
    from diffsinger_b200 import DsxError, ParallelWaveGANGenerator
    g, sd, cfg = fixture("pwg_plain.npz")
    m = ParallelWaveGANGenerator(**cfg)
    m.load_state_dict(sd, strict=True)
    with pytest.raises(DsxError, match="CPU"):
        m(torch.from_numpy(g["z"]), torch.from_numpy(g["c"]))


def test_missing_c_raises(lib_built):
    from diffsinger_b200 import DsxError, ParallelWaveGANGenerator
    g, _, cfg = fixture("pwg_plain.npz")
    with pytest.raises(DsxError, match="auxiliary features"):
        ParallelWaveGANGenerator(**cfg)(torch.from_numpy(g["z"]))


UNSUPPORTED = [
    ("use_causal_conv", dict(use_causal_conv=True)),
    ("upsample_conditional_features", dict(upsample_conditional_features=False)),
    ("upsample_net", dict(upsample_net="MelGANGenerator")),
    ("nonlinear_activation", dict(upsample_params={"upsample_scales": [4, 4, 4, 4], "nonlinear_activation": "ReLU"})),
    ("interpolate_mode", dict(upsample_params={"upsample_scales": [4, 4, 4, 4], "interpolate_mode": "bilinear"})),
    ("freq_axis_kernel_size", dict(upsample_params={"upsample_scales": [4, 4, 4, 4], "freq_axis_kernel_size": 3})),
    ("bias", dict(bias=False)),
    ("in_channels", dict(in_channels=2)),
    ("out_channels", dict(out_channels=2)),
    ("residual_channels", dict(residual_channels=128)),
    ("gate_channels", dict(gate_channels=256)),
    ("skip_channels", dict(skip_channels=128)),
    ("aux_channels", dict(aux_channels=128)),
    ("kernel_size", dict(kernel_size=5)),
    ("layers", dict(layers=66, stacks=3)),
    ("stacks", dict(layers=34, stacks=2)),
    ("upsample_scales", dict(upsample_params={"upsample_scales": [17, 4]})),
    ("upsample_scales", dict(upsample_params={"upsample_scales": [16, 16, 8]})),
    ("aux_context_window", dict(aux_context_window=17)),
]


@pytest.mark.parametrize("option,kw", UNSUPPORTED, ids=[f"{o}-{i}" for i, (o, _) in enumerate(UNSUPPORTED)])
def test_unsupported_options_are_named(lib_built, option, kw):
    from diffsinger_b200 import DsxError, ParallelWaveGANGenerator
    with pytest.raises(DsxError, match=f"unsupported {option}="):
        ParallelWaveGANGenerator(**kw)
