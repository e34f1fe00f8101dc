"""The residual and skip epilogues of the step kernel load a batch of x / skip pairs together with the bias and FiLM
pairs of its columns, ahead of the stores.  What an utterance computes must not depend on the batch around it: whether
its tiles have a CTA each, are paired with another utterance's, or are walked by CTAs that also run other tiles only
changes the schedule.  So an utterance in a batch with more tiles than resident CTAs gives bit for bit the eps and the
DDPM output it gives alone, at both tile heights, with a partial last tile and an odd number of layers under the fused
head.
Run on an H100: python -m pytest tests -m gpu"""
import pytest
import torch

from conftest import HP, rs_normal
from oracle import diffnet_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def dsx(lib_built):
    import diffsinger_b200
    assert torch.cuda.is_available()
    return diffsinger_b200


def run(dsx, prec, rows, layers, cond, xT, noise):
    """K DDPM steps with injected noise, then one evaluation, on one handle at `rows` frames per CTA"""
    from diffsinger_b200 import _capi
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = dsx.DiffNet(80, hparams=dict(HP, residual_layers=layers, dilation_cycle_length=4))
    torch.nn.init.normal_(net.output_projection.weight, std=0.02)
    s = dsx.DsxSampler(net.to(dev).eval(), prec, 4)
    s.ensure_weights(dev)
    s.set_schedule(O.make_schedule(O.linear_beta_schedule(100, 0.06)))
    s.set_option(_capi.OPT_STACK_ROWS, rows)
    B, K = xT.shape[0], noise.shape[0]
    outs = [s.sample_ddpm(xT.to(dev), cond.to(dev), 100, K, noise=noise.to(dev)).cpu(),
            s.diffnet_forward(xT.to(dev), torch.full((B,), 37, dtype=torch.long, device=dev), cond.to(dev)).cpu()]
    assert s.info(_capi.INFO_STACK_ROWS) == rows
    s.close()
    return outs


@pytest.mark.parametrize("prec", ["fp16s", "fp16x2"])
@pytest.mark.parametrize("rows,B", [(128, 17), (64, 9)])
def test_utterance_alone_matches_utterance_in_multi_tile_batch(dsx, prec, rows, B):
    T, layers, K = 1000, 5, 2                       # 1000 frames: the last 128- or 64-frame tile is partial
    tiles = B * (-(-T // 128) * 128) // rows
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert tiles > sms, "the batch must have more tiles than resident CTAs (one per SM at either tile height)"
    cond, xT = rs_normal(70 + B, (B, 256, T)), rs_normal(71, (B, 1, 80, T))
    noise = rs_normal(72, (K, B, 1, 80, T))
    batch = run(dsx, prec, rows, layers, cond, xT, noise)
    for b in (0, B - 1):
        alone = run(dsx, prec, rows, layers, cond[b:b + 1].contiguous(), xT[b:b + 1].contiguous(),
                    noise[:, b:b + 1].contiguous())
        for name, x, y in zip(("sample_ddpm", "diffnet_forward eps"), batch, alone):
            assert torch.isfinite(y).all()
            d = (x[b:b + 1] - y).abs().max().item()
            print(f"{prec} rows={rows} B={B} utterance {b}: {name} max |d| {d:.3e}")
            assert torch.equal(x[b:b + 1], y), (name, d)
