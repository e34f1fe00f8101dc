"""Would the bounds of tests/test_gpu_diffnet_edges.py catch a subtly wrong step kernel?  CPU only.

Each mutation below is a plausible bug of the step kernel or the sampler host, applied to diffnet_oracle's operand-format
simulation (fmt=) through the simulation's step functions.  The cases and bounds are read from the test file itself,
so the two cannot drift apart.  A case is applicable to a mutation when its shape reaches the bug (a last tile of
2 frames or more, dilation 8 with a second 128-frame tile, odd L, several utterances of different t, a loop of several
evaluations, a PLMS loop of two or more steps); it catches the mutation when the mutated fp16x2 simulation's error against float64 exceeds the case's fp16x2 bound.
The table gives, per mutation, the applicable cases, those that catch it, the smallest ratio of error to bound among
those, and the error / bound of those that miss.

    python -m oracle.diffnet_edge_sensitivity          # the mutation table
    python -m oracle.diffnet_edge_sensitivity --sim    # the simulated errors behind the test file's SIM table

What reaches what: a late +d tap needs a last tile of 2 frames or more (with one frame, the tap reads past T either
way); a 7-row halo needs dilation 8 and a second 128-frame tile (within the first, the taps it loses read outside the
utterance anyway).  A stale input projection is missed by the PLMS loops of one step and of interval 1: there the
evaluations of a step see almost the same x, so the stale projection is nearly the right one, and the loops of more
or longer steps catch it.
"""
import contextlib
import importlib.util
import os
import sys

import torch
import torch.nn.functional as F

from . import diffnet_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load_tests():
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    spec = importlib.util.spec_from_file_location("diffnet_edges", os.path.join(ROOT, "tests", "test_gpu_diffnet_edges.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@contextlib.contextmanager
def patched(name, make):
    orig = getattr(O, name)
    setattr(O, name, make(orig))
    try:
        yield
    finally:
        setattr(O, name, orig)


# ---- the mutations --------------------------------------------------------------------------------------------------
def late_tap_last_tile(orig):
    """the +d tap of the frames of the last, partial, 64-frame tile reads one frame late"""
    def conv(y, w, b, dilation):
        out = orig(y, w, b, dilation)
        T = y.shape[-1]
        t0 = T // 64 * 64
        if T % 64 == 0 or dilation >= T:
            return out
        tap = torch.zeros_like(w)
        tap[..., 2] = w[..., 2]
        late = F.pad(y[..., 1:], (0, 1))
        wrong = orig(late, tap, None, dilation) - orig(y, tap, None, dilation)
        out = out.clone()
        out[..., t0:] += wrong[..., t0:]
        return out
    return conv


def halo7(orig):
    """the conv-input window holds 7 rows beyond each end of a 128-frame tile: the +-8 taps of the tile's first and last
    row read zero"""
    def conv(y, w, b, dilation):
        out = orig(y, w, b, dilation)
        if dilation != 8:
            return out
        T = y.shape[-1]
        out = out.clone()
        for t0 in range(0, T, 128):
            for t, tap, src in ((t0, 0, t0 - 8), (min(t0 + 127, T - 1), 2, min(t0 + 127, T - 1) + 8)):
                if 0 <= src < T:
                    out[..., t] -= torch.einsum("oc,bc->bo", w[..., tap], y[..., src])
        return out
    return conv


def film_of_previous_layer(orig):
    """the residual epilogue of layer l prepares layer l + 1's input with layer l's FiLM vector"""
    return lambda P, e, i: orig(P, e, max(i - 1, 0))


def drop_last_skip_odd_l(orig):
    """the last layer's skip is not added when L is odd"""
    return lambda skips: orig(skips[:-1]) if len(skips) % 2 and len(skips) > 1 else orig(skips)


def next_utterance_row(orig):
    """utterance b reads utterance b + 1's FiLM-table row"""
    def film(P, e, i):
        return orig(P, torch.cat([e[1:], e[-1:]]), i)
    return film


def stale_input_projection(orig):
    """in a loop, layer 0 reads the input projection of the previous evaluation"""
    last = []

    def proj(P, spec, f):
        x = orig(P, spec, f)
        out = last[0] if last and last[0].shape == x.shape else x
        last[:] = [x]
        return out
    return proj


def plms_mode3_second_step(orig):
    """the second PLMS step combines with mode 3's weights (23, -16, 5) / 12 and no third eps"""
    def prime(noise_pred, noise_list):
        if len(noise_list) == 1:
            return (23 * noise_pred - 16 * noise_list[-1]) / 12
        return orig(noise_pred, noise_list)
    return prime


def meta(T, name):
    """(T, L, cycle, B, loop kind or None, evaluations, PLMS steps) of a tensor-core case"""
    if name in T.FWD:
        c = T.FWD[name]
        return c["T"], c["L"], c["cycle"], c["B"], None, 1, 0
    inp = T.loop_inputs(name)
    kind, a, b = inp["kind"], inp["a"], inp["b"]
    steps = len(range(0, a, b)) if kind == "plms" else 0
    evals = {"ddpm": b, "plms": steps + 1, "infer": 1}[kind]
    return inp["T"], inp["L"], 4, 1, kind, evals, steps


# name -> (simulation step replaced, mutation, the cases it can reach: predicate on meta())
MUTATIONS = {
    "+d tap one frame late on the last partial tile": (
        "sim_dilated_conv", late_tap_last_tile, lambda Tn, L, cyc, B, kind, ev, st: Tn % 64 > 1),
    "7-row window halo": (
        "sim_dilated_conv", halo7, lambda Tn, L, cyc, B, kind, ev, st: cyc == 4 and L >= 4 and Tn > 128),
    "FiLM of layer l instead of l + 1": (
        "sim_film", film_of_previous_layer, lambda Tn, L, cyc, B, kind, ev, st: L >= 2),
    "last skip dropped at odd L": (
        "sim_skip_sum", drop_last_skip_odd_l, lambda Tn, L, cyc, B, kind, ev, st: L % 2 == 1 and L > 1),
    "utterance b reads row b + 1": (
        "sim_film", next_utterance_row, lambda Tn, L, cyc, B, kind, ev, st: kind is None and B > 1),
    "layer 0 reads the previous input projection": (
        "sim_input_projection", stale_input_projection, lambda Tn, L, cyc, B, kind, ev, st: ev >= 2),
    "PLMS mode 3 on the second step": (
        "plms_prime", plms_mode3_second_step, lambda Tn, L, cyc, B, kind, ev, st: st >= 2),
}


# ---- simulating the test file's cases -------------------------------------------------------------------------------
def case_runs(T):
    """(name, run(fmt) -> error against float64) for every tensor-core case of the test file"""
    runs = []
    for name, c in T.FWD.items():
        def fwd(fmt, name=name, c=c):
            sd = T.f64(T.state_dict(c["L"], c["cycle"]))
            spec, t, cond = T.fwd_inputs(name)
            eps = O.diffnet_forward(sd, spec.double(), t, cond.double(), c["cycle"], fmt=fmt(sd))
            return (eps - T.fwd_ref(name)).abs().max().item()
        runs.append((name, fwd))
    for name in T.LOOP_CASES:
        def loop(fmt, name=name):
            inp = T.loop_inputs(name)
            sd = T.f64(T.state_dict(inp["L"], 4))
            return T.loop_error(T.run_oracle_loop(sd, inp, fmt(sd)), T.loop_ref(name))
        runs.append((name, loop))
    return runs


def formats(T, fmt):
    """makers of the format objects a simulated error is the worst of"""
    if fmt == "fp16s":
        return [lambda sd, s=s: O.OperandFormat(sd, "fp16s", seed=s) for s in T.SR_DRAWS]
    return [lambda sd: O.OperandFormat(sd, fmt)]


def fp32_error(T, name):
    if name in T.SIMT:
        M, C, H, L, cyc, Tn = T.SIMT[name]
        spec, t, cond = T.simt_inputs(name)
        return (O.diffnet_forward(T.state_dict(L, cyc, M, C, H), spec, t, cond, cyc).double()
                - T.simt_ref(name)).abs().max().item()
    if name in T.FWD:
        c = T.FWD[name]
        spec, t, cond = T.fwd_inputs(name)
        return (O.diffnet_forward(T.state_dict(c["L"], c["cycle"]), spec, t, cond, c["cycle"]).double()
                - T.fwd_ref(name)).abs().max().item()
    inp = T.loop_inputs(name)
    return T.loop_error(T.run_oracle_loop(T.state_dict(inp["L"], 4), inp), T.loop_ref(name))


def print_sim(T):
    for name, run in case_runs(T):
        errs = [max(run(m) for m in formats(T, fmt)) for fmt in T.FMTS] + [fp32_error(T, name)]
        print(f'    "{name}": ({", ".join(f"{e:.2e}" for e in errs)}),', flush=True)
    for name in T.SIMT:
        print(f'    "{name}": (0, 0, 0, 0, {fp32_error(T, name):.2e}),', flush=True)


def main():
    T = load_tests()
    torch.set_grad_enabled(False)
    if "--sim" in sys.argv:
        return print_sim(T)
    # fp16x2, the precision with the tightest bounds among the forms that run every case
    fmt = "fp16x2"
    make = formats(T, fmt)[0]
    runs = case_runs(T)
    print(f"{'mutation':46s} {'applicable':>10s} {'caught':>7s} {'min err / bound':>16s}  missed")
    never = []
    for mut, (attr, mutate, reaches) in MUTATIONS.items():
        applicable, caught, ratio, missed = 0, 0, float("inf"), []
        for name, run in runs:
            if not reaches(*meta(T, name)):
                continue
            bnd = T.bound(T.SIM[name][T.FMTS.index(fmt)], fmt)
            with patched(attr, mutate):
                err = run(make)
            applicable += 1
            if err > bnd:
                caught += 1
                ratio = min(ratio, err / bnd)
            else:
                missed.append(f"{name} ({err / bnd:.2f})")
        print(f"{mut:46s} {applicable:10d} {caught:7d} {ratio:16.1f}  {', '.join(missed)}", flush=True)
        if caught == 0:
            never.append(mut)
    if never:
        raise SystemExit(f"never caught: {never}")


if __name__ == "__main__":
    main()
