"""Would the bounds of tests/test_gpu_config_edges.py catch a subtly wrong kernel?  CPU only.

Each mutation below is a plausible implicit-GEMM bug.  It is applied to the fp16 simulation of a few of that file's
cases, wherever the case's kernels would meet it (every conv the bug's condition covers), and the error against the
float64 oracle is printed next to the bound the case uses.  The cases and bounds are read from the test file itself, so
the two cannot drift apart.  A mutation is caught when its max or its mean error exceeds the bound.

    python -m oracle.edge_sensitivity
"""
import contextlib
import importlib.util
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def load_tests():
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    spec = importlib.util.spec_from_file_location("edges", os.path.join(ROOT, "tests", "test_gpu_config_edges.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@contextlib.contextmanager
def patched(name, make, module=F):
    orig = getattr(module, name)
    setattr(module, name, make(orig))
    try:
        yield
    finally:
        setattr(module, name, orig)


def round16(n):
    return (n + 15) // 16 * 16


# ---- the mutations --------------------------------------------------------------------------------------------------
def tap_shift(orig):
    """the last tap of every conv with k > 1 reads one row too far"""
    def conv1d(x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
        y = orig(x, w, b, stride, padding, dilation, groups)
        if w.shape[-1] == 1:
            return y
        last = torch.zeros_like(w)
        last[..., -1] = w[..., -1]
        shifted = F.pad(x[..., 1:], (0, 1))
        return y - orig(x, last, None, stride, padding, dilation, groups) + \
            orig(shifted, last, None, stride, padding, dilation, groups)
    return conv1d


def drop_last_k_chunk(orig):
    """every conv whose K = taps x round16(cin) is not a multiple of 64 skips its last, partial, 64-wide K chunk"""
    def conv1d(x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
        cout, cin, k = w.shape
        cin_p = round16(cin)
        K = k * cin_p
        if K % 64:
            start = (K - 1) // 64 * 64
            kk = torch.arange(k)[None, :] * cin_p + torch.arange(cin)[:, None]     # [cin, k]: the packed K index
            w = w * (kk < start).to(w.dtype)
        return orig(x, w, b, stride, padding, dilation, groups)
    return conv1d


def zero_last_partial_column(orig):
    """every conv whose cout leaves a partial 64-wide column tile loses its last real output channel"""
    def conv1d(x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
        y = orig(x, w, b, stride, padding, dilation, groups)
        if w.shape[0] % 64:
            y = y.clone()
            y[:, -1] = 0
        return y
    return conv1d


def shift_group_boundary(orig):
    """GroupNorm statistics taken over groups that start one channel late (group g = channels 16 g + 1 .. 16 g + 16)"""
    def group_norm(x, G, weight=None, bias=None, eps=1e-5):
        r = lambda t: torch.roll(t, -1, 0 if t.dim() == 1 else 1)
        return torch.roll(orig(r(x), G, r(weight), r(bias), eps), 1, 1)
    return group_norm


def swap_heads(orig):
    """attention heads 0 and 1 write each other's output (decoder_fp16_sim normalises o [B, heads, T, D] through
    torch.nan_to_num, which is where the swap is applied)"""
    def nan_to_num(t, *a, **kw):
        t = orig(t, *a, **kw)
        if t.dim() == 4 and t.shape[1] > 1:
            t = t.clone()
            t[:, [0, 1]] = t[:, [1, 0]]
        return t
    return nan_to_num


MUTATIONS = {
    "tap offset +1 row": ("conv1d", tap_shift, F),
    "last K chunk dropped": ("conv1d", drop_last_k_chunk, F),
    "last real column of a partial tile zeroed": ("conv1d", zero_last_partial_column, F),
    "GroupNorm group boundary moved by one channel": ("group_norm", shift_group_boundary, F),
    "attention heads 0 and 1 swapped": ("nan_to_num", swap_heads, torch),
}


# ---- the cases ------------------------------------------------------------------------------------------------------
def main():
    T = load_tests()
    torch.set_grad_enabled(False)

    def hifigan(name):
        h, sd, mel, lens = T.hifigan_case(name)
        ref = T.hifigan_ref(h, sd, mel, lens)
        return lambda: T.hifigan_ref(h, sd, mel, lens, fp16=True), ref, ref.abs().max().item(), T.BOUNDS["hifigan", name]

    def pitch(name):
        hp, L, sd, mel = T.pitch_case(name)
        ref = T.pitch_ref(hp, L, sd, mel)[0]
        return lambda: T.pitch_ref(hp, L, sd, mel, fp16=True)[0], ref, 1.0, T.BOUNDS["pitch", name]

    def stack(name):
        hp, sd, inp = T.stack_case(name)
        ref = T.stack_ref(name, hp, sd, inp)
        scale = ref.abs().max().item() if T.STACK[name].get("relative") else 1.0
        return lambda: T.stack_ref(name, hp, sd, inp, fp16=True), ref, scale, T.BOUNDS["stack", name]

    plan = [
        ("tap offset +1 row", [hifigan("chain_dil32"), hifigan("c0_384"), pitch("kernel31_T20"), stack("dec_H64_heads1")],
         ["hifigan chain_dil32", "hifigan c0_384", "pitch kernel31_T20", "stack dec_H64_heads1"]),
        ("last K chunk dropped", [hifigan("c0_384"), pitch("H48"), pitch("H208")],
         ["hifigan c0_384", "pitch H48", "pitch H208"]),
        ("last real column of a partial tile zeroed", [hifigan("c0_384"), hifigan("c0_16"), pitch("H48"), pitch("H208")],
         ["hifigan c0_384", "hifigan c0_16", "pitch H48", "pitch H208"]),
        ("GroupNorm group boundary moved by one channel", [pitch("H48"), pitch("conv_layers16")],
         ["pitch H48", "pitch conv_layers16"]),
        ("attention heads 0 and 1 swapped", [stack("dec_H192_heads3_T65"), stack("enc_H192_heads3")],
         ["stack dec_H192_heads3_T65", "stack enc_H192_heads3"]),
    ]
    print(f"{'mutation':46s} {'case':28s} {'max':>9s} {'bound':>9s} {'mean':>9s} {'bound':>9s}  caught")
    missed = 0
    for mut, cases, names in plan:
        attr, make, module = MUTATIONS[mut]
        for (run, ref, scale, bound), name in zip(cases, names):
            clean = T.errors(run(), ref, scale)
            with patched(attr, make, module):
                mx, mean = T.errors(run(), ref, scale)
            caught = mx > bound[0] or mean > bound[1]
            missed += not caught
            print(f"{mut:46s} {name:28s} {mx:9.2e} {bound[0]:9.1e} {mean:9.2e} {bound[1]:9.1e}  "
                  f"{'yes' if caught else 'NO'}   (unmutated {clean[0]:.1e} / {clean[1]:.1e})")
    if missed:
        raise SystemExit(f"{missed} mutation(s) within their bounds")


if __name__ == "__main__":
    main()
