"""CPU: oracle/ssim_oracle.py against tests/golden/ssim.npz (written from the live reference by oracle/gen_golden_ssim.py):
bit for bit in fp32, and within fp32 rounding in float64.  Also pins the window the kernels hard-code
(diffsinger_b200/csrc/dsx_ssim.cu) to the oracle's."""
import os
import re

import numpy as np
import pytest
import torch

from conftest import ROOT, golden
from oracle import ssim_oracle as O

CASES = ("mel", "cwt")


def fields(c):
    g = golden("ssim.npz")
    f = lambda k: torch.from_numpy(g[f"{c}.{k}"])
    return f("decoder_output"), f("target"), float(g[f"{c}.bias"]), g, f


@pytest.mark.parametrize("case", CASES)
def test_oracle_is_bit_exact_in_fp32(case):
    out, target, bias, g, f = fields(case)
    x, y = out[:, None] + bias, target[:, None] + bias
    assert torch.equal(O.ssim(x, y, size_average=False), f("map"))
    assert torch.equal(O.ssim(x, y), f("mean"))
    o = out.clone().requires_grad_(True)
    loss = O.ssim_loss(o, target, bias)
    loss.backward()
    assert torch.equal(loss.detach(), f("loss"))
    assert torch.equal(o.grad, f("d_decoder_output"))


# fp32 rounds G*(x^2) ~ (bias + x)^2 by ~ulp/2 = 2e-6 (bias 6) to 1e-5 (bias 20), which moves the map by that over
# sigma^2 + C2; on these inputs the float64 map lies within 1e-3 of the fp32 one, the loss within 2e-6 and the gradient
# within 1e-7 (against a gradient of ~1e-3).  The bounds are about twice that.
BOUNDS = {"map": 2e-3, "loss": 4e-6, "grad": 2e-7}


@pytest.mark.parametrize("case", CASES)
def test_float64_is_within_fp32_rounding(case):
    out, target, bias, g, f = fields(case)
    o = out.double().requires_grad_(True)
    t = target.double()
    m = O.ssim(o.detach()[:, None] + bias, t[:, None] + bias, size_average=False)
    loss = O.ssim_loss(o, t, bias)
    loss.backward()
    assert (m - f("map").double()).abs().max().item() <= BOUNDS["map"]
    assert abs(loss.item() - float(g[f"{case}.loss"])) <= BOUNDS["loss"]
    assert (o.grad - f("d_decoder_output").double()).abs().max().item() <= BOUNDS["grad"]


def test_kernel_window_is_the_reference_window():
    src = open(os.path.join(ROOT, "diffsinger_b200", "csrc", "dsx_ssim.cu")).read()
    body = re.search(r"kG\[[^\]]*\]\s*=\s*\{([^}]*)\}", src).group(1)
    kernel = np.array([float.fromhex(v.strip().rstrip("f")) for v in body.split(",")], dtype=np.float32)
    assert np.array_equal(kernel, O.gaussian().numpy())
    assert np.array_equal(kernel, golden("ssim.npz")["window"])
