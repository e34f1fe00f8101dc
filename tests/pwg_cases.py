"""Shared cases of the PWG vocoder tests: configurations, seeded weights and inputs (no GPU needed)."""
import numpy as np
import torch

from conftest import golden
from oracle import pwg_oracle as P

FIXTURES = ["pwg_plain.npz", "pwg_pitch.npz"]


def config(**kw):
    """generator_params: the shipped generator with overrides (`scales` sets upsample_params)"""
    scales = kw.pop("scales", [4, 4, 4, 4])
    return dict(P.CONFIG_SHIPPED, upsample_params={"upsample_scales": list(scales)}, **kw)


def fixture(name):
    g = golden(name)
    sd = {k[3:]: torch.from_numpy(g[k]) for k in g.files if k.startswith("sd.")}
    cfg = config(layers=int(g["layers"]), stacks=int(g["stacks"]), use_pitch_embed=bool(g["use_pitch_embed"]))
    return g, sd, cfg


def plain(sd):
    """the state dict after remove_weight_norm(): `.weight` in place of weight_g / weight_v"""
    out = dict(sd)
    for k in list(sd):
        if k.endswith(".weight_g"):
            name = k[:-len(".weight_g")]
            out[name + ".weight"] = P.conv_weight(sd, name)
            del out[name + ".weight_g"], out[name + ".weight_v"]
    return out


def inputs(cfg, B, T, seed):
    """z [B, 1, T * hop], the edge-padded c [B, 80, T + 2w] as spec2wav's transposed view, and an edge-padded pitch"""
    w, hp = cfg["aux_context_window"], P.hop(cfg)
    gen = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 1, T * hp, generator=gen)
    mel = torch.randn(B, T, 80, generator=gen)
    c = torch.from_numpy(np.pad(mel.numpy(), ((0, 0), (w, w), (0, 0)), "edge")).transpose(1, 2)
    coarse = torch.randint(1, 256, (B, T), generator=gen)
    pitch = torch.from_numpy(np.pad(coarse.numpy(), ((0, 0), (w, w)), "edge"))
    return z, c, pitch


def random_sd(cfg, seed):
    """the reference's own initialisation, with every bias and weight_g perturbed so that none is trivially 0 or 1"""
    from diffsinger_b200 import ParallelWaveGANGenerator
    torch.manual_seed(seed)
    m = ParallelWaveGANGenerator(**cfg)
    sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
    gen = torch.Generator().manual_seed(seed + 1)
    for k, v in sd.items():
        if k.endswith(".bias"):
            sd[k] = 0.1 * torch.randn(v.shape, generator=gen)
        elif k.endswith(".weight_g"):
            sd[k] = v * (1 + 0.2 * torch.rand(v.shape, generator=gen))
    return sd


# (overrides, B, T): the shipped topology, a second hop, and the edges of what dsx_pwg_create accepts
TOPOLOGIES = {
    "shipped": (dict(), 2, 24),
    "hop300": (dict(layers=20, stacks=2, scales=[5, 5, 4, 3], aux_context_window=0), 2, 10),
    "layers1": (dict(layers=1, stacks=1), 2, 6),
    "layers64": (dict(layers=64, stacks=4), 1, 4),
    "per_stack1": (dict(layers=6, stacks=6), 2, 5),
    # dilations up to 2^15: every off-centre tap of the deepest layers lies past a 3-frame utterance
    "per_stack16": (dict(layers=16, stacks=1), 2, 3),
    "one_frame": (dict(layers=10, stacks=1), 3, 1),
    "one_scale": (dict(layers=8, stacks=2, scales=[7]), 2, 40),
    "hop1024": (dict(layers=8, stacks=2, scales=[16, 16, 4]), 2, 3),
    "window16_pitch": (dict(layers=6, stacks=2, aux_context_window=16, use_pitch_embed=True), 2, 5),
}


def topology(name):
    kw, B, T = TOPOLOGIES[name]
    return config(**kw), B, T


def simulated_error(cfg, sd, z, c, pitch):
    """max and mean |fp16 simulation - fp32| over the fp32 output's peak"""
    with torch.no_grad():
        ref = P.generator(sd, cfg, z, c, pitch)
        sim = P.generator(sd, cfg, z, c, pitch, fp16=True)
    d, peak = (sim - ref).abs(), ref.abs().max()
    return (d.max() / peak).item(), (d.mean() / peak).item()
