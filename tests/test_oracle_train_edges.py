"""CPU: the float64 references and the mutation Functions behind tests/test_gpu_train_edges.py and
oracle/train_edge_sensitivity.py, and the GPU file's cases against the ranges include/dsx.h documents."""
import os

import pytest
import torch
import torch.nn.functional as F

import test_gpu_train_edges as E
from oracle import train_edge_sensitivity as S

CPU = torch.device("cpu")
HEADER = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dsx.h")).read()


def _fs2(name):
    hp, sd, x, g = E.fs2_case(name)
    masks = S.seeded_masks(hp, x.shape[0], x.shape[1])
    return lambda mode: E.fs2_ref(hp, sd, x, g, masks, mode, CPU), ("out", "d_x"), ~E.D.padding_mask(x)


def _fft(name):
    hp, sd, spec, t, cond, g = E.fft_case(name)
    masks = S.seeded_masks(hp, spec.shape[0], spec.shape[3])
    return lambda mode: E.fft_ref(hp, sd, spec, t, cond, g, masks, mode, CPU), ("eps", "d_cond"), None


def _diffnet(name):
    net, spec, t, cond, g = E.diffnet_case(name)
    return lambda mode: E.diffnet_ref(net, spec, t, cond, g, mode, CPU), ("eps", "d_cond"), None


SMALL = [(_fs2, "left_k4_H64_T100"), (_fs2, "H128_h2_T65"), (_fft, "H192_h3_dim16"), (_diffnet, "L3_T65"),
         (_diffnet, "L24_c24_T40")]


@pytest.mark.parametrize("make,name", SMALL)
def test_float64_reference_agrees_with_fp32(make, name):
    """float64 and fp32 autograd of the same oracle differ by fp32 rounding only (measured worst 3.4e-6)"""
    run, names, keep = make(name)
    r64, r32 = run("f64"), run("fp32")
    assert r64[0].dtype == torch.float64 and all(v.dtype == torch.float64 for v in r64[2].values())
    assert r32[0].dtype == torch.float32
    e = E.errors(r32, r64, names, keep)
    for m, (v, n) in E.worst(e).items():
        assert v <= 2e-5, (m, n, v)
    assert e.get("pos_embed_alpha", {"rel": 0})["rel"] <= 1e-4


def test_dilation_beyond_T_runs_as_T():
    """diffnet_ref's dilation d > T -> T changes nothing: both outer taps lie outside every utterance either way"""
    torch.manual_seed(0)
    x, w, b = torch.randn(2, 8, 40, dtype=torch.float64), torch.randn(6, 8, 3, dtype=torch.float64), torch.randn(6)
    for d in (41, 64, 2 ** 12):
        assert torch.equal(F.conv1d(x, w, b.double(), padding=d, dilation=d), F.conv1d(x, w, b.double(), padding=40,
                                                                                     dilation=40))


def _same_grads(fn, *xs, g=None):
    """gradients of fn through Mutable with no mutation, and through plain autograd: bitwise equal"""
    a = [x.detach().clone().requires_grad_(x.requires_grad) if x is not None else None for x in xs]
    b = [x.detach().clone().requires_grad_(x.requires_grad) if x is not None else None for x in xs]
    ya, yb = S.Mutable.apply(fn, None, *a), fn(*b)
    assert torch.equal(ya, yb)
    g = torch.randn_like(yb) if g is None else g
    ya.backward(g)
    yb.backward(g)
    for u, v in zip(a, b):
        if v is not None and v.requires_grad:
            assert torch.equal(u.grad, v.grad)


def test_mutable_switched_off_is_autograd():
    torch.manual_seed(1)
    r = lambda *s: torch.randn(*s, dtype=torch.float64, requires_grad=True)
    x = r(3, 16, 65)
    for k, pad, dil in ((5, 2, 1), (3, 4, 4), (4, 0, 1), (1, 0, 1)):
        _same_grads(lambda x_, w_, b_: S._conv1d(x_, w_, b_, 1, pad, dil, 1), x, r(24, 16, k), r(24))
    _same_grads(S._linear, r(65, 3, 16), r(48, 16), None)
    _same_grads(S._linear, r(3, 65, 16), r(48, 16), r(48))
    pad = torch.zeros(3, 65, dtype=torch.bool)
    pad[1, 50:] = True
    _same_grads(S.attention(pad), r(3, 2, 65, 32), r(3, 2, 65, 32), r(3, 2, 65, 32))
    _same_grads(lambda v: v.clone(), r(65, 3, 16))


def test_patched_ops_restate_torch():
    """with every op patched and no mutation, the decoder reference equals the unpatched one to float64 rounding (the
    attention restatement included)"""
    run, names, keep = _fs2("H128_h2_T65")
    ref = run("f64")
    S.STATE.update(step="fs2", B=3, T=65, mutation=None, layer=1)
    with S.patched():
        got = run("f64")
    for m, (v, n) in E.worst(E.errors(got, ref, names, keep)).items():
        assert v <= 1e-12, (m, n, v)


@pytest.mark.parametrize("mutation", S.MUTATIONS)
def test_each_mutation_changes_the_backward_only(mutation):
    """switched on where its condition holds, a mutation leaves the forward bitwise and changes some gradient"""
    step, name = ("diffnet", "L3_T65") if mutation == S.MUTATIONS[1] else ("fs2", "H128_h2_T65")
    run, errors = S.case_runner(E, step, name)
    assert S.applies(mutation, step, E.CASES[step][name])
    with S.patched():
        S.STATE["mutation"] = None
        clean = run()
        S.STATE["mutation"] = mutation
        try:
            bad = run()
        finally:
            S.STATE["mutation"] = None
    assert torch.equal(bad[0], clean[0])
    assert max(v for per in errors(bad, clean).values() for v in per.values()) > 1e-3


# ---- the cases against include/dsx.h ---------------------------------------------------------------------------------
def test_cases_inside_the_documented_ranges():
    for text in ("a multiple of 64 in [64, 256]", "L: 1..64", "odd for SAME, any k >= 1 for LEFT (k <= 255)",
                 "H / heads must be 64 or 128", "0 'SAME' (k // 2 each side), 1 'LEFT' (k - 1 on the left)",
                 "a multiple of 16 in [16, 1024]", "residual_layers: 1..1024", "dilation_cycle_length: 1..24",
                 "B <= 65535,\n * B T <= 2^24 and L B T < 2^26"):
        assert text in HEADER, text
    for step, cases in E.CASES.items():
        for name, c in cases.items():
            B, T = c["B"], c["T"]
            if step == "diffnet":
                L = c["L"]
                assert 1 <= L <= 1024 and 1 <= c["cycle"] <= 24, name
            else:
                hp = c["hp"]
                H, heads, k, L = hp["hidden_size"], hp["num_heads"], hp["dec_ffn_kernel_size"], hp["dec_layers"]
                assert H % 64 == 0 and 64 <= H <= 256 and 1 <= L <= 64, name
                assert H % heads == 0 and H // heads in (64, 128), name
                assert hp["ffn_padding"] in ("SAME", "LEFT") and 1 <= k <= 255, name
                assert hp["ffn_padding"] == "LEFT" or k % 2 == 1, name
                assert 0 <= hp["dropout"] < 1, name
                if step == "fft":
                    dim = hp["residual_channels"]
                    assert dim % 16 == 0 and 16 <= dim <= 1024, name
            assert 1 <= B <= 65535 and B * T <= 2 ** 24 and L * B * T < 2 ** 26, name
            assert B >= 2 or "B1" in name, name


def test_bounds_cover_every_case_and_measure():
    assert set(E.BOUNDS) == {(s, n) for s, c in E.CASES.items() for n in c}
    for key, b in E.BOUNDS.items():
        assert set(b) == {"rel", "frame", "row"}, key
        assert all(E.FLOOR[m] <= v and (v <= E.CAP or key[0] == "diffnet" and m != "rel") for m, v in b.items()), key
