"""CPU: the float64 references and the mutation Functions behind tests/test_gpu_train_edges.py and
oracle/train_edge_sensitivity.py, and the GPU file's cases against the ranges include/dsx.h documents."""
import os

import pytest
import torch
import torch.nn.functional as F

import test_gpu_train_edges as E
from oracle import fs2enc_oracle as EO
from oracle import train_edge_sensitivity as S
from oracle.pe_oracle import sinusoidal_table

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


def _fs2enc(name):
    hp, sd, tok, adds, g = E.enc_case(name)
    masks = S.seeded_masks(hp, tok.shape[0], tok.shape[1])
    return lambda mode: E.enc_ref(hp, sd, tok, adds, g, masks, EO.REL_MAX_LEN, mode, CPU), ("out", "d_add"), tok != 0


def _durpred(name):
    """without the fp16 rounding of the conv operands: it is a step function, and its gradient (durpred_train rounds
    the gradient through it to fp16 too) rounds an fp32 value and a float64 one to different fp16 values wherever they
    straddle a rounding boundary"""
    hp, sd, x, mask, g = E.dur_case(name)
    gen = torch.Generator().manual_seed(5)
    masks = [torch.rand(x.shape[0], x.shape[1], hp["P"], generator=gen) >= hp["p"] for _ in range(hp["L"])]

    def run(mode):
        xs, d_x, grads = E.dur_ref(hp, sd, x, mask, g, masks, mode, CPU, fp16=False)
        return xs[..., None], d_x, grads
    return run, ("xs", "d_x"), (~mask, None)


SMALL = [(_fs2, "left_k4_H64_T100"), (_fs2, "H128_h2_T65"), (_fft, "H192_h3_dim16"), (_diffnet, "L3_T65"),
         (_diffnet, "L24_c24_T40"), (_fs2enc, "midi_T65"), (_fs2enc, "sin_H192_h3_T65"), (_durpred, "shipped_T65")]


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


def test_float64_position_tables():
    """the encoder oracle's position tables in float64 are float64, agree with the fp32 ones to the rounding of an fp32
    angle (about P 2^-24 at position P), and are the tables embedding() adds in float64"""
    for P, H in ((2101, 256), (5001, 128)):
        for t32, t64 in ((EO.rel_table(P, H), EO.rel_table(P, H, torch.float64)),
                         (sinusoidal_table(P, H), sinusoidal_table(P, H, dtype=torch.float64))):
            assert t32.dtype == torch.float32 and t64.dtype == torch.float64
            d = (t32.double() - t64).abs().max().item()
            assert 0 < d <= 4 * P * 2.0 ** -24 + 2.0 ** -22, (P, H, d)
    T, H = 2100, 64
    sd = {"embed_tokens.weight": torch.zeros(3, H, dtype=torch.float64)}
    rel = EO.embedding(sd, torch.zeros(1, T, dtype=torch.long), dict(hidden_size=H, rel_pos=True), (), 5001)
    assert rel.dtype == torch.float64 and torch.equal(rel[0], EO.rel_table(5001, H, torch.float64)[:T])
    sin = EO.embedding(sd, torch.ones(1, T, dtype=torch.long), dict(hidden_size=H, rel_pos=False))
    assert sin.dtype == torch.float64 and torch.equal(sin[0], sinusoidal_table(T + 1, H, dtype=torch.float64)[1:])


def test_sort_layouts_end_their_runs_where_intended():
    """the token layouts of test_embedding_gradient_is_the_sum_of_d_add, sorted as the kernel sorts them"""
    for F in E.SORT_F:
        for kind in ("one_id", "distinct", "runs", "out_of_range"):
            tok, V = E.sort_layout(kind, F)
            assert tok.shape == (F,)
            keys, ends = E.sorted_runs(tok, V)
            if kind == "one_id":
                assert ends == [F] and (keys == 7).all()
            elif kind == "distinct":
                assert ends == list(range(1, F + 1)) and V == F + 1
            elif kind == "runs":
                assert V - 1 == len(ends) and tok.min() >= 1 and tok.max() == V - 1
                want = [e for e in (63, 64, 65, 128, 192, 384) if e < F]
                assert all(e in ends for e in want), (F, ends[:12])
            else:
                bad = (tok <= 0) | (tok >= V)
                assert bad.sum() == F // 5
                if F >= 5:
                    assert (tok < 0).any() and (tok >= V).any() and (tok == 0).any()
                assert keys[:int(bad.sum())].eq(0).all() and keys[int(bad.sum()):].gt(0).all()


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


@pytest.mark.parametrize("mutation", S.ALL_MUTATIONS)
def test_each_mutation_changes_the_backward_only(mutation):
    """switched on where its condition holds, a mutation leaves the forward bitwise and changes some gradient"""
    step, name = {S.MUTATIONS[1]: ("diffnet", "L3_T65"), S.OWN_MUTATIONS[0]: ("fs2enc", "midi_T65"),
                  S.OWN_MUTATIONS[1]: ("durpred", "shipped_T65")}.get(mutation, ("fs2", "H128_h2_T65"))
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
                 "B <= 65535,\n * B T <= 2^24 and L B T < 2^26", "input channels: a multiple of 16 in [16, 256]",
                 "n_layers (dur_predictor_layers): 1..16", "kernel_size (dur_predictor_kernel): 1..31, odd for SAME",
                 "rows of embed_tokens (len(dictionary)), >= 1", "Requires T <= P"):
        assert text in HEADER, text
    for step, cases in E.CASES.items():
        for name, c in cases.items():
            B, T = c["B"], c["T"]
            if step == "diffnet":
                L = c["L"]
                assert 1 <= L <= 1024 and 1 <= c["cycle"] <= 24, name
            elif step == "durpred":
                hp = c["hp"]
                L = hp["L"]
                assert all(v % 16 == 0 and 16 <= v <= 256 for v in (hp["idim"], hp["P"])) and 1 <= L <= 16, name
                assert 1 <= hp["k"] <= 31 and (hp["padding"] == "LEFT" or hp["k"] % 2 == 1), name
                assert hp["padding"] in ("SAME", "LEFT") and 0 <= hp["p"] < 1, name
            else:
                hp = c["hp"]
                if step == "fs2enc":
                    hp = dict(EO.stack_hp(hp), dropout=hp["dropout"])
                    assert c.get("vocab", E.VOCAB) >= 1 and c.get("rel_len") in (None, "T"), name
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
        for m, v in b.items():
            uncapped = key[0] == "durpred" or m != "rel" and (key[0] == "diffnet" or key == ("fs2enc",
                                                                                              "H128_h1_left_k255_relu"))
            assert E.FLOOR[m] <= v and (v <= E.CAP or uncapped), (key, m)
