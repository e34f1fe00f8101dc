"""Would the bounds of tests/test_gpu_train_edges.py catch a subtly wrong training backward?  CPU only.

Each mutation below is a bug the training steps' backward kernels could plausibly have.  It is applied to the float64
oracle's backward through small autograd Functions (the forward is unchanged), on every case of that file where the
mutation's condition holds, and its error against the unmutated float64 oracle is printed under the test's own measures
next to the case's bounds.  The cases and BOUNDS are read from the test file, so the two cannot drift apart.  A
mutation is caught on a case when any measure exceeds its bound; it must be caught on at least one case.  The last
columns say whether rel alone would have caught it.  The dropout masks are seeded draws here (the GPU test uses the
step's own); they change what a mutation hits by sampling noise only.

    python -m oracle.train_edge_sensitivity [mutation ...]

Inside the oracles every linear, conv1d, attention, embedding and LayerNorm runs through Mutable (F.linear, F.conv1d,
F.multi_head_attention_forward, F.embedding and F.layer_norm are patched for the run), and so does the residual stream
entering each layer of the decoder, the FFT denoiser and DiffNet.  With no
mutation switched on, Mutable's backward is autograd's own (tests/test_oracle_train_edges.py checks this exactly)."""
import contextlib
import importlib.util
import os
import sys

import torch
import torch.nn.functional as F

from oracle.fs2enc_oracle import REL_MAX_LEN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_conv1d, _linear, _mha, _embedding, _layer_norm = (F.conv1d, F.linear, F.multi_head_attention_forward, F.embedding,
                                                   F.layer_norm)
CPU = torch.device("cpu")


def load_tests():
    for p in (ROOT, os.path.join(ROOT, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    spec = importlib.util.spec_from_file_location("train_edges", os.path.join(ROOT, "tests", "test_gpu_train_edges.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


# ---- an op whose backward can be replaced ----------------------------------------------------------------------------
def autograd_grads(fn, xs, g, want=None):
    """autograd's gradients of fn(*xs) for cotangent g: one per x, None where x needs none (or its index is not in want)"""
    idx = [i for i, x in enumerate(xs) if x is not None and x.requires_grad and (want is None or i in want)]
    out = [None] * len(xs)
    if idx:
        gs = torch.autograd.grad(fn(*xs), [xs[i] for i in idx], g, allow_unused=True)
        for i, v in zip(idx, gs):
            out[i] = v
    return out


class Mutable(torch.autograd.Function):
    """y = fn(*xs); the backward recomputes fn under autograd and returns autograd's gradients, or, with a mutation,
    mutate(fn, xs, g) (one gradient per x)."""

    @staticmethod
    def forward(ctx, fn, mutate, *xs):
        ctx.fn, ctx.mutate = fn, mutate
        ctx.save_for_backward(*xs)
        return fn(*xs)

    @staticmethod
    def backward(ctx, g):
        xs = [None if x is None else x.detach().requires_grad_(need)
              for x, need in zip(ctx.saved_tensors, ctx.needs_input_grad[2:])]
        with torch.enable_grad():
            grads = (ctx.mutate or autograd_grads)(ctx.fn, xs, g)
        return (None, None) + tuple(grads)


# ---- where the frames are ---------------------------------------------------------------------------------------------
STATE = dict(B=0, T=0, mutation=None, layer=0)


def chunk_mask(B, T):
    """[B, T]: the frames of the last partial 64-frame chunk of the flat B T frame axis (none when 64 divides B T)"""
    m = torch.zeros(B * T, dtype=torch.bool)
    m[B * T // 64 * 64:] = True
    return m.view(B, T)


def tile_mask(B, T):
    """[B, T]: per utterance, the frames of the last partial 64-row tile (none when 64 divides T)"""
    m = torch.zeros(B, T, dtype=torch.bool)
    m[:, T // 64 * 64:] = True
    return m


def laid_out(m, y, kind):
    """m [B, T] as a mask over y: conv outputs are [B, C, T]; linear outputs [T, B, C] (the decoder's layers) or
    [B, T, C]; anything else (the step-embedding MLP's [B, C]) has no frame axis: None"""
    B, T = m.shape
    if kind == "conv":
        return m[:, None, :]
    if y.dim() == 3 and tuple(y.shape[:2]) == (T, B) and T != B:
        return m.t()[:, :, None]
    if y.dim() == 3 and tuple(y.shape[:2]) == (B, T):
        return m[:, :, None]
    return None


# ---- the mutations --------------------------------------------------------------------------------------------------
def wgrad_without_last_chunk(kind):
    """1. the frames of the last partial 64-frame chunk are missing from the weight gradient"""
    def mutate(fn, xs, g):
        grads = autograd_grads(fn, xs, g)
        m = laid_out(chunk_mask(STATE["B"], STATE["T"]), g, kind)
        if m is not None and xs[1].requires_grad:
            grads[1] = autograd_grads(fn, xs, g * ~m, want={1})[1]
        return grads
    return mutate


def wgrad_over_concatenated_batch(fn, xs, g):
    """2. a conv with k > 1: the weight gradient taken over the batch as one sequence, so a shifted operand reads the
    neighbouring utterance instead of zero"""
    grads = autograd_grads(fn, xs, g)
    x, w, _ = xs
    if w.shape[-1] == 1 or not w.requires_grad:
        return grads
    B, T = STATE["B"], STATE["T"]
    lead = x.shape[-1] - T                          # LEFT: the k - 1 frames F.pad put in front of each utterance
    xc = F.pad(x[..., lead:].detach().permute(1, 0, 2).reshape(1, x.shape[1], B * T), (lead, 0))
    gc = g.permute(1, 0, 2).reshape(1, g.shape[1], B * T)
    wl = w.detach().requires_grad_(True)
    grads[1] = torch.autograd.grad(fn(xc, wl, None), wl, gc)[0]
    return grads


def dgrad_last_tap_one_frame_off(fn, xs, g):
    """4. a conv with k > 1: the transposed (data-gradient) conv reads the last tap's cotangent one frame late"""
    grads = autograd_grads(fn, xs, g)
    x, w, _ = xs
    if w.shape[-1] == 1 or not x.requires_grad:
        return grads
    last = torch.zeros_like(w)
    last[..., -1] = w[..., -1]
    xl = x.detach().requires_grad_(True)
    d = lambda cot: torch.autograd.grad(fn(xl, last.detach(), None), xl, cot)[0]
    grads[0] = grads[0] - d(g) + d(F.pad(g[..., 1:], (0, 1)))
    return grads


def attention(pad):
    """softmax(q k^T, keys of `pad` masked) v over [B, heads, T, D] (q already scaled)"""
    def fn(q, k, v):
        s = (q @ k.transpose(-1, -2)).masked_fill(pad[:, None, None, :], float("-inf"))
        return torch.softmax(s, -1) @ v
    fn.pad = pad
    return fn


def attention_missing_last_block(which):
    """3. dQ without the keys of the last partial 64-key block ("dq"), or dK and dV without the queries of the last
    partial 64-query block ("dkv")"""
    def mutate(fn, xs, g):
        q, k, v = (x.detach() for x in xs)
        n = q.shape[2] // 64 * 64
        s = (q @ k.transpose(-1, -2)).masked_fill(fn.pad[:, None, None, :], float("-inf"))
        p = torch.softmax(s, -1)
        ds = p * (g @ v.transpose(-1, -2) - (g * (p @ v)).sum(-1, keepdim=True))
        dq, dk, dv = ds @ k, ds.transpose(-1, -2) @ q, p.transpose(-1, -2) @ g
        if which == "dq":
            dq = ds[..., :n] @ k[..., :n, :]
        else:
            dk, dv = ds[..., :n, :].transpose(-1, -2) @ q[..., :n, :], p[..., :n, :].transpose(-1, -2) @ g[..., :n, :]
        return [dq, dk, dv]
    return mutate


def residual_gradient_zeroed(kind):
    """5. one layer's residual-stream gradient is zeroed on the frames of the last partial 64-row tile"""
    def mutate(fn, xs, g):
        return [g * ~laid_out(tile_mask(STATE["B"], STATE["T"]), g, kind)]
    return mutate


def sorted_chunks(tokens, V):
    """[F] per frame of tokens (flat): its token as the embedding gradient sorts it (ids outside [1, V) as 0) and the
    64-frame chunk of the stable sort of the frames by token it lands in"""
    tok = tokens.reshape(-1)
    key = torch.where((tok > 0) & (tok < V), tok, torch.zeros_like(tok))
    order = torch.argsort(key * tok.numel() + torch.arange(tok.numel(), device=tok.device))
    chunk = torch.empty_like(order)
    chunk[order] = torch.arange(tok.numel(), device=tok.device) // 64
    return key, chunk


def embedding_without_last_piece(tokens):
    """7. the embedding gradient: a token whose sorted run spans several 64-frame chunks loses its piece in the last"""
    def mutate(fn, xs, g):
        key, chunk = sorted_chunks(tokens, xs[0].shape[0])
        drop = torch.zeros_like(key, dtype=torch.bool)
        for v in key.unique().tolist():
            sel = key == v
            if v != 0 and chunk[sel].min() < chunk[sel].max():
                drop |= sel & (chunk == chunk[sel].max())
        return autograd_grads(fn, xs, g * ~drop.view(*tokens.shape, 1))
    return mutate


def layer_norm_without_mean_term(fn, xs, g):
    """8. LayerNorm's data gradient drops its mean term (rstd mean(w g)) on the last partial 64-row tile ([B, T, C])"""
    grads = autograd_grads(fn, xs, g)
    x, w, _ = xs
    if grads[0] is None:
        return grads
    x = x.detach()
    rstd = (x.var(-1, unbiased=False, keepdim=True) + fn.eps).rsqrt()
    m = tile_mask(STATE["B"], STATE["T"]).to(x.device)[:, :, None]
    grads[0] = grads[0] + rstd * (g * w.detach()).mean(-1, keepdim=True) * m
    return grads


# the shared layers' mutations (tests/test_oracle_train_edges.py checks each on the decoder, the dilated-conv one on
# DiffNet), then the encoder's and the duration predictor's own
MUTATIONS = ["wgrad: last partial 64-frame chunk missing", "conv wgrad: shifted operand reads the neighbour",
             "attention: dQ misses the last key block", "attention: dK, dV miss the last query block",
             "ffn_1 dgrad: last tap one frame off", "residual gradient zeroed on the last partial tile"]
OWN_MUTATIONS = ["embedding: a run loses its last 64-frame chunk piece",
                 "durpred LayerNorm dgrad: no mean term on the last partial tile"]
ALL_MUTATIONS = MUTATIONS + OWN_MUTATIONS


def kernel_size(step, c):
    return {"diffnet": lambda: 3, "durpred": lambda: c["hp"]["k"],
            "fs2enc": lambda: c["hp"]["enc_ffn_kernel_size"]}.get(step, lambda: c["hp"]["dec_ffn_kernel_size"])()


def applies(mutation, step, c):
    B, T = c["B"], c["T"]
    k = kernel_size(step, c)
    attn = step in ("fs2", "fft", "fs2enc")
    M = ALL_MUTATIONS
    return {M[0]: B * T % 64 != 0, M[1]: B > 1 and k > 1, M[2]: attn and T % 64 != 0, M[3]: attn and T % 64 != 0,
            M[4]: step != "diffnet" and k > 1, M[5]: step in ("fs2", "fft", "diffnet") and T % 64 != 0,
            M[6]: step == "fs2enc" and B * T > 64, M[7]: step == "durpred" and T % 64 != 0}[mutation]


# ---- the patched ops ------------------------------------------------------------------------------------------------
def _on(i):
    return STATE["mutation"] == ALL_MUTATIONS[i]


def conv1d(x, w, b=None, stride=1, padding=0, dilation=1, groups=1):
    fn = lambda x_, w_, b_: _conv1d(x_, w_, b_, stride, padding, dilation, groups)
    mutate = wgrad_without_last_chunk("conv") if _on(0) else wgrad_over_concatenated_batch if _on(1) else \
        dgrad_last_tap_one_frame_off if _on(4) and STATE["step"] != "diffnet" else None
    return Mutable.apply(fn, mutate, x, w, b)


def linear(x, w, b=None):
    return Mutable.apply(_linear, wgrad_without_last_chunk("linear") if _on(0) else None, x, w, b)


def multi_head_attention_forward(query, key, value, embed_dim, num_heads, in_proj_weight, in_proj_bias, bias_k, bias_v,
                                 add_zero_attn, dropout_p, out_proj_weight, out_proj_bias, training=True,
                                 key_padding_mask=None, need_weights=True, attn_mask=None, **_):
    """the decoder's bias-free self-attention, [T, B, E] in and out, with the attention core through Mutable"""
    T, B, E = query.shape
    Dh = E // num_heads
    heads = lambda z: z.reshape(T, B, num_heads, Dh).permute(1, 2, 0, 3)
    q, k, v = (heads(z) for z in linear(query, in_proj_weight, in_proj_bias).chunk(3, -1))
    mutate = attention_missing_last_block("dq") if _on(2) else attention_missing_last_block("dkv") if _on(3) else None
    o = Mutable.apply(attention(key_padding_mask), mutate, q * Dh ** -0.5, k, v)
    return linear(o.permute(2, 0, 1, 3).reshape(T, B, E), out_proj_weight, out_proj_bias), None


def embedding(input, weight, padding_idx=None, *args, **kwargs):
    fn = lambda w_: _embedding(input, w_, padding_idx, *args, **kwargs)
    return Mutable.apply(fn, embedding_without_last_piece(input) if _on(6) else None, weight)


def layer_norm(input, normalized_shape, weight=None, bias=None, eps=1e-5):
    fn = lambda x_, w_, b_: _layer_norm(x_, normalized_shape, w_, b_, eps)
    fn.eps = eps
    mutate = layer_norm_without_mean_term if _on(7) and STATE["step"] == "durpred" else None
    return Mutable.apply(fn, mutate, input, weight, bias)


def layer_input(kind):
    """the residual stream entering layer i, through Mutable (zeroed on the last partial tile for one layer)"""
    def hook(i, x):
        on = _on(5) and i == STATE["layer"]
        return Mutable.apply(lambda v: v.clone(), residual_gradient_zeroed(kind) if on else None, x)
    return hook


@contextlib.contextmanager
def patched():
    saved = F.conv1d, F.linear, F.multi_head_attention_forward, F.embedding, F.layer_norm
    F.conv1d, F.linear, F.multi_head_attention_forward, F.embedding, F.layer_norm = (
        conv1d, linear, multi_head_attention_forward, embedding, layer_norm)
    try:
        yield
    finally:
        F.conv1d, F.linear, F.multi_head_attention_forward, F.embedding, F.layer_norm = saved


# ---- the cases -------------------------------------------------------------------------------------------------------
def seeded_masks(hp, B, T, seed=5):
    H, L, p = hp["hidden_size"], hp.get("dec_layers", hp.get("enc_layers")), hp["dropout"]
    gen = torch.Generator().manual_seed(seed)
    return [torch.rand(B, T, n, generator=gen) >= p for n in [H] + [H, 4 * H, H] * L]


def case_runner(E, step, name):
    """run(mode) -> (primary, d_input, grads) of the case's reference in float64 on the CPU; and errors(res, ref)"""
    c = E.CASES[step][name]
    STATE.update(step=step, layer=(c["L"] if step == "diffnet" else c["hp"].get("dec_layers", 0)) // 2)
    if step == "fs2":
        hp, sd, x, g = E.fs2_case(name)
        idx = [b for b in range(c["B"]) if b != c.get("empty")]
        x, g = x[idx], g[idx]
        masks = seeded_masks(hp, len(idx), c["T"])
        run = lambda: E.fs2_ref(hp, sd, x, g, masks, "f64", CPU, layer_input("linear"))
        keep, names = ~E.D.padding_mask(x), ("out", "d_x")
    elif step == "fft":
        hp, sd, spec, t, cond, g = E.fft_case(name)
        masks = seeded_masks(hp, c["B"], c["T"])
        run = lambda: E.fft_ref(hp, sd, spec, t, cond, g, masks, "f64", CPU, layer_input("linear"))
        keep, names = None, ("eps", "d_cond")
    elif step == "fs2enc":
        hp, sd, tok, adds, g = E.enc_case(name)
        idx = [b for b in range(c["B"]) if b != c.get("empty")]
        tok, adds, g = tok[idx], [a[idx] for a in adds], g[idx]
        masks = seeded_masks(hp, len(idx), c["T"])
        rel_len = c["T"] if c.get("rel_len") == "T" else max(REL_MAX_LEN, c["T"])
        used = E.used_rows(tok, sd["encoder.embed_tokens.weight"].shape[0])

        def run():
            out, d_add, grads = E.enc_ref(hp, sd, tok, adds, g, masks, rel_len, "f64", CPU)
            return out, d_add, E.embed_rows(grads, used)
        keep, names = tok != 0, ("out", "d_add")
    elif step == "durpred":
        hp, sd, x, mask, g = E.dur_case(name)
        gen = torch.Generator().manual_seed(5)
        masks = [torch.rand(c["B"], c["T"], hp["P"], generator=gen) >= hp["p"] for _ in range(hp["L"])]

        def run():
            xs, d_x, grads = E.dur_ref(hp, sd, x, mask, g, masks, "f64", CPU)
            return xs[..., None], d_x, grads
        keep, names = (~mask, None), ("xs", "d_x")
    else:
        net, spec, t, cond, g = E.diffnet_case(name)
        run = lambda: E.diffnet_ref(net, spec, t, cond, g, "f64", CPU, layer_input("conv"))
        keep, names = None, ("eps", "d_cond")
    STATE.update(B=len(keep[0] if isinstance(keep, tuple) else keep) if keep is not None else c["B"], T=c["T"])
    return run, lambda res, ref: E.errors(res, ref, names, keep, c.get("peak", False))


def main(argv):
    E = load_tests()
    chosen = [m for m in ALL_MUTATIONS if not argv or any(a in m for a in argv)]
    print(f"{'mutation':50s} {'case':32s} {'rel':>8s} {'bound':>7s} {'frame':>8s} {'bound':>7s} {'row':>8s} "
          f"{'bound':>7s}  caught  by rel")
    summary = {m: [0, 0, 0] for m in chosen}           # cases run, caught, caught by rel
    with patched():
        for step, cases in E.CASES.items():
            for name in cases:
                todo = [m for m in chosen if applies(m, step, cases[name])]
                if not todo:
                    continue
                run, errors = case_runner(E, step, name)
                STATE["mutation"] = None
                clean = run()
                for m in todo:
                    STATE["mutation"] = m
                    w = E.worst(errors(run(), clean))
                    STATE["mutation"] = None
                    b = E.BOUNDS[step, name]
                    hit = {k: w[k][0] > b[k] for k in b}
                    s = summary[m]
                    s[0] += 1
                    s[1] += any(hit.values())
                    s[2] += hit["rel"]
                    print(f"{m:50s} {step + ' ' + name:32s} " + " ".join(
                        f"{w[k][0]:8.1e} {b[k]:7.1e}" for k in ("rel", "frame", "row")) +
                        f"  {'yes' if any(hit.values()) else 'NO':6s}  {'yes' if hit['rel'] else 'no'}", flush=True)
    print()
    missed = []
    for m, (n, caught, by_rel) in summary.items():
        print(f"{m:50s} caught on {caught} of {n} cases, by rel alone on {by_rel}")
        if not caught:
            missed.append(m)
    if missed:
        raise SystemExit(f"never caught: {missed}")


if __name__ == "__main__":
    main(sys.argv[1:])
