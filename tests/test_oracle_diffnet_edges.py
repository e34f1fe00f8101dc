"""CPU: diffnet_oracle's operand-format simulation (fmt=), which the bounds of test_gpu_diffnet_edges.py are built on.
fmt=None must stay the reference computation bit for bit, and the simulation must reproduce, within a factor of 2, the
errors the GPU tests have measured."""
import math
import re

import pytest
import torch
import torch.nn.functional as F

from conftest import rs_normal
from oracle import diffnet_oracle as O


def forward_before_fmt(P, spec, t, cond, cycle):
    """diffnet_forward as it was before fmt= and dilated_conv existed"""
    L = O.num_layers(P)
    x = F.relu(F.conv1d(spec[:, 0], P["input_projection.weight"], P["input_projection.bias"]))
    e = O.sinusoidal_embedding(t, P["mlp.2.weight"].shape[0])
    e = F.linear(O.mish(F.linear(e, P["mlp.0.weight"], P["mlp.0.bias"])), P["mlp.2.weight"], P["mlp.2.bias"])
    skips = []
    for i in range(L):
        p, dil = f"residual_layers.{i}.", 2 ** (i % cycle)
        d = F.linear(e, P[p + "diffusion_projection.weight"], P[p + "diffusion_projection.bias"]).unsqueeze(-1)
        c = F.conv1d(cond, P[p + "conditioner_projection.weight"], P[p + "conditioner_projection.bias"])
        y = F.conv1d(x + d, P[p + "dilated_conv.weight"], P[p + "dilated_conv.bias"], padding=dil, dilation=dil) + c
        gate, filt = torch.chunk(y, 2, dim=1)
        y = F.conv1d(torch.sigmoid(gate) * torch.tanh(filt), P[p + "output_projection.weight"],
                     P[p + "output_projection.bias"])
        residual, skip = torch.chunk(y, 2, dim=1)
        x = (x + residual) / math.sqrt(2.0)
        skips.append(skip)
    x = torch.sum(torch.stack(skips), dim=0) / math.sqrt(L)
    x = F.relu(F.conv1d(x, P["skip_projection.weight"], P["skip_projection.bias"]))
    return F.conv1d(x, P["output_projection.weight"], P["output_projection.bias"])[:, None]


@pytest.mark.parametrize("T,cycle,L", [(1, 4, 5), (9, 4, 6), (65, 3, 5), (96, 1, 3)])
def test_fmt_none_is_the_reference_bit_for_bit(T, cycle, L):
    P = O.build_state_dict(0, 80, 64, 48, L, cycle)
    spec, cond, t = rs_normal(1, (2, 1, 80, T)), rs_normal(2, (2, 48, T)), torch.tensor([3, 77])
    with torch.no_grad():
        assert torch.equal(O.diffnet_forward(P, spec, t, cond, cycle), forward_before_fmt(P, spec, t, cond, cycle))


def test_plms_loop_keeps_its_combination_bit_for_bit():
    """p_sample_plms's multistep combination moved into plms_prime: the loop is unchanged"""
    P = O.build_state_dict(0, 80, 32, 32, 2, 2)
    S = O.make_schedule(O.linear_beta_schedule(100, 0.06))
    x, cond = rs_normal(3, (1, 1, 80, 20)), rs_normal(4, (1, 32, 20))
    with torch.no_grad():
        hist, y = [], x
        for t in (60, 40, 20, 0, 80):      # modes 0, 2, 3, 4, 4
            n = len(hist)
            eps = O.diffnet_forward(P, y, torch.full((1,), t), cond, 2)
            if n == 0:
                prev = O.diffnet_forward(P, O.plms_x_pred(S, y, eps, t, 20), torch.full((1,), max(t - 20, 0)), cond, 2)
                prime = (eps + prev) / 2
            elif n == 1:
                prime = (3 * eps - hist[-1]) / 2
            elif n == 2:
                prime = (23 * eps - 16 * hist[-1] + 5 * hist[-2]) / 12
            else:
                prime = (55 * eps - 59 * hist[-1] + 37 * hist[-2] - 9 * hist[-3]) / 24
            want = O.plms_x_pred(S, y, prime, t, 20)
            hist2 = list(hist)
            got = O.p_sample_plms(P, S, y, t, 20, cond, hist2, 2)
            assert torch.equal(got, want), t
            hist = (hist + [eps])[-4:]
            y = want


@pytest.mark.parametrize("cycle", [2, 3])
def test_fp16x2_simulation_matches_the_measured_error(cycle):
    """test_gpu_config_edges.py's test_diffnet_dilation_cycles measured 3.1e-4 (fp16x2, B 3 x T 333, on an H100)"""
    P = {k: v.double() for k, v in O.build_state_dict(0, dilation_cycle_length=cycle).items()}
    spec, cond, t = rs_normal(71, (3, 1, 80, 333)).double(), rs_normal(72, (3, 256, 333)).double(), torch.tensor([3, 50, 99])
    with torch.no_grad():
        ref = O.diffnet_forward(P, spec, t, cond, cycle)
        sim = O.diffnet_forward(P, spec, t, cond, cycle, fmt="fp16x2")
    err = (sim - ref).abs().max().item()
    print(f"cycle {cycle}: simulated {err:.2e}, measured 3.1e-4")
    assert 3.1e-4 / 2 <= err <= 3.1e-4 * 2


def test_formats_round_what_the_kernel_rounds():
    P = O.build_state_dict(0, 80, 32, 32, 2, 1)
    x = torch.randn(1000, dtype=torch.float64)
    assert torch.equal(O.rn16(x), x.half().double())
    assert (O.hl16(x) - x).abs().max() < 2 ** -21 * x.abs().max()
    f1, f2 = O.OperandFormat(P, "fp16s", sr_sets=4, seed=5), O.OperandFormat(P, "fp16s", sr_sets=4, seed=5)
    w = "residual_layers.1.dilated_conv.weight"
    assert f1.weights(1)[w] is f1.weights(5)[w]                         # row j on set j % R
    assert torch.equal(f1.weights(2)[w], f2.weights(2)[w])              # a draw is seeded
    assert not torch.equal(f1.weights(0)[w], f1.weights(1)[w])
    assert torch.equal(f1.weights(0)[w].half().double(), f1.weights(0)[w].double())     # fp16 values
    assert (f1.weights(0)[w] - P[w]).abs().max() <= (P[w] - P[w].half().float()).abs().max() * 2 + 1e-12
    assert O.OperandFormat(P, "fp16").head is O.rn16 and O.OperandFormat(P, "fp16x3").act is O.hl16


def test_edge_bounds_table_matches_sim():
    """the bounds the GPU edge file's docstring lists are the ones its SIM table and bound() give"""
    import importlib.util
    import os
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_gpu_diffnet_edges.py")
    spec = importlib.util.spec_from_file_location("diffnet_edges", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rows = dict(re.findall(r"^    (\S+) +([\d.e\-+ /]+)$", mod.__doc__, re.M))
    assert set(rows) == set(mod.SIM)
    for name, sims in mod.SIM.items():
        want = [mod.bound(s, f) for s, f in zip(sims, mod.FMTS + ("fp32",)) if s > 0 or f == "fp32"]
        got = [float(v) for v in rows[name].replace("/", " ").split()]
        assert got == want, name
