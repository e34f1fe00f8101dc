"""The step kernel orders its layers through per-tile progress flags (a tile waits for its neighbour tiles only) and, when
every tile has its own CTA, runs the odd utterances half a layer behind the even ones.  Neither may change a result:
the one-launch-per-step form must agree with the per-layer launches and repeat itself bit for bit, on the geometries
where the ordering matters -- an odd number of layers under the fused head (the head's input projection rewrites the
Y buffer that layer L - 1 reads), paired utterances next to an unpaired one, partial last tiles, both tile heights.
Run on an H100: python -m pytest tests -m gpu"""
import pytest
import torch

from conftest import HP, rs_normal
from oracle import diffnet_oracle as O

pytestmark = pytest.mark.gpu

TOL = 6e-4   # fp16x2, one-launch-per-step form against per-layer launches (as test_stack_kernel_matches_layer_kernel)


@pytest.fixture(scope="module")
def dsx(lib_built):
    import diffsinger_b200
    assert torch.cuda.is_available()
    return diffsinger_b200


def make_sampler(dsx, layers, cycle, options):
    from diffsinger_b200 import _capi
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = dsx.DiffNet(80, hparams=dict(HP, residual_layers=layers, dilation_cycle_length=cycle))
    torch.nn.init.normal_(net.output_projection.weight, std=0.02)
    s = dsx.DsxSampler(net.to(dev).eval(), "fp16x2", cycle)
    s.ensure_weights(dev)
    s.set_schedule(O.make_schedule(O.linear_beta_schedule(100, 0.06)))
    s.set_option(_capi.OPT_GATE_APPROX, 0)
    for k, v in options:
        s.set_option(k, v)
    return s, dev


def run(dsx, layers, cycle, B, T, K, options):
    """K DDPM steps with injected noise, then one evaluation, on one handle"""
    s, dev = make_sampler(dsx, layers, cycle, options)
    cond, xT = rs_normal(60 + B, (B, 256, T)).to(dev), rs_normal(61 + T, (B, 1, 80, T)).to(dev)
    noise = rs_normal(62, (K, B, 1, 80, T)).to(dev)
    outs = [s.sample_ddpm(xT, cond, 100, K, noise=noise).cpu(),
            s.diffnet_forward(xT, torch.full((B,), 37, dtype=torch.long, device=dev), cond).cpu()]
    s.close()
    return outs


@pytest.mark.parametrize("rows", [128, 64])
@pytest.mark.parametrize("layers,cycle,B,T,K", [
    (5, 4, 3, 333, 4),      # odd L under the fused head; utterances 0 / 1 paired, 2 alone; partial last tiles
    (20, 1, 5, 1024, 2),    # two pairs and an unpaired utterance, whole tiles
    (7, 4, 2, 129, 3),      # odd L; a last tile holding one frame (128-frame tiles) or none (64-frame tiles)
])
def test_flag_ordered_step_matches_per_layer_launches(dsx, rows, layers, cycle, B, T, K):
    from diffsinger_b200 import _capi
    ref = run(dsx, layers, cycle, B, T, K, ((_capi.OPT_STACK_KERNEL, 0), (_capi.OPT_STACK_MODE, 0)))
    new = [run(dsx, layers, cycle, B, T, K, ((_capi.OPT_STACK_KERNEL, 1), (_capi.OPT_STACK_ROWS, rows))) for _ in range(2)]
    for a, b, c in zip(ref, new[0], new[1]):
        d = (a - b).abs().max().item()
        print(f"L={layers} B={B} T={T} rows={rows}: max |d| {d:.3e}")
        assert torch.isfinite(b).all()
        assert d < TOL * max(1.0, a.abs().max().item()), d
        assert torch.equal(b, c)
