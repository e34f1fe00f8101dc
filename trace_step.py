#!/usr/bin/env python
"""trace_step.py -- where the time of one residual layer of the step kernel goes (k_hp_step, dsx_hopper.cu).

  python trace_step.py [--config 1|2|3|4] [--precision fp16s|fp16x2|fp16x3|fp16] [--steps N] [--warmup W] [--json]

Runs a bench.py config and records the step kernel's phase stamps (dsx_debug_trace, slot layout in include/dsx.h) of the
last launch of each of N timed steps: with the fused head, one launch is one whole diffusion step.  Prints the mean µs
of each layer phase over the CTAs, layers and steps, and of the head phases, with the card's name, power limit and the
median SM clock during the traced steps.  A CTA that walks over several tiles of a layer (config 4) stamps its last
tile only, so there GEMM1 chunk 0 also holds its earlier tiles; the layer total stays right.  The last layer phase is the
wait for the neighbour tiles (and, for paired utterances, the partner) that ends where the next layer starts.

When the kernel runs the even and the odd utterances half a layer apart (every tile has its own CTA and B >= 2), the
phase split is also printed for each of the two groups, with the mean time by which an odd-utterance tile starts a
layer after its even partner.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

import numpy as np
import torch

LAYER_PHASES = ("GEMM1 chunk 0", "gate epilogue 0", "GEMM1 chunk 1", "gate epilogue 1", "GEMM2 residual half",
                "residual epilogue", "GEMM2 skip half", "skip epilogue", "wait before next layer")
HEAD_PHASES = ("H1 GEMM", "H1 epilogue", "H2 GEMM", "mel update", "input projection GEMM", "input projection epilogue")


def utterance_groups(B, T, rows, ctas):
    """Trace rows (CTAs) of the even and of the odd utterances when the step kernel runs them half a layer apart (every
    tile has its own CTA and B >= 2: tile j of utterance 2k + 1 is paired with tile j of utterance 2k), else None.
    -> (even rows, odd rows, [(even, odd) partner rows])"""
    tpu = -(-T // 128) * 128 // rows
    if B < 2 or B * tpu > ctas:
        return None
    u = np.arange(B * tpu)
    b = u // tpu
    pairs = [(int(i), int(i + tpu)) for i in u[(b % 2 == 0) & (b + 1 < B)]]
    return u[b % 2 == 0], u[b % 2 == 1], pairs


def start_offset(tr, layers, pairs):
    """mean µs by which a paired odd-utterance tile starts layers 1 .. layers - 1 after its even partner (slot 8 of the
    layer before: the end of the wait that starts the layer)"""
    d = [tr[o, 9 * i] - tr[e, 9 * i] for e, o in pairs for i in range(1, layers) if tr[o, 9 * i] and tr[e, 9 * i]]
    return float(np.mean(d)) * 1e-3 if d else None


def phase_split(tr, layers, ctas=None):
    """tr: int64 [CTAs, slots] stamps of one launch over `layers` layers and the head; ctas: the rows to use (all when
    None).  -> (layer [n_phases] µs summed over the CTAs and layers, number of (CTA, layer) samples, head [6] µs summed
    over the CTAs, CTAs)"""
    if ctas is not None:
        tr = tr[ctas]
    tr = tr[tr[:, 0] != 0].astype(np.float64)
    lay = np.zeros(len(LAYER_PHASES))
    n = 0
    for i in range(layers):
        base = 1 + 9 * i
        prev = tr[:, 0] if i == 0 else tr[:, base - 1]
        s = tr[:, base:base + 9]
        if i == layers - 1 and not s[:, 8].any():
            s = s.copy()
            s[:, 8] = s[:, 7]                     # no wait after the last layer of a launch without a head
        d = np.diff(np.concatenate([prev[:, None], s], axis=1), axis=1)
        lay += d.sum(axis=0)
        n += len(tr)
    head = np.zeros(len(HEAD_PHASES))
    hb = 1 + 9 * layers
    # slots the launch did not reach keep an earlier launch's stamps (e.g. the input projection, absent from the last
    # step of a loop): only stamps after this launch's entry count
    h = np.where(tr[:, hb:hb + len(HEAD_PHASES)] >= tr[:, :1], tr[:, hb:hb + len(HEAD_PHASES)], 0)
    if h[:, 0].any():
        prev = tr[:, hb - 1]
        for k in range(len(HEAD_PHASES)):
            if not h[:, k].any():
                continue
            head[k] = (h[:, k] - prev).sum()
            prev = h[:, k]
    return lay * 1e-3, n, head * 1e-3, len(tr)


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), f"--query-gpu={q}",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, mx = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": mx}
    except Exception:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(), "power_limit": None, "sm_max_clock": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="2", choices=["1", "2", "3", "4"])
    ap.add_argument("--precision", default="fp16s")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--json", action="store_true", help="print one JSON line instead of the table")
    args = ap.parse_args()

    assert torch.cuda.is_available(), "trace_step.py needs a CUDA device"
    import __graft_entry__
    __graft_entry__.build()
    import bench
    import diffsinger_b200 as dsx
    from diffsinger_b200 import _capi

    dev = torch.device("cuda", 0)
    cfg = bench.CONFIGS[args.config]
    arm = bench.Arm(dsx, cfg, args.precision, dev, 0)
    for i in range(args.warmup):
        arm.step(i)
    torch.cuda.synchronize()
    cs = bench.ClockSampler(0)
    cs.start()
    layers = bench.hp_for(cfg)["residual_layers"]
    lay, n, head, nh = np.zeros(len(LAYER_PHASES)), 0, np.zeros(len(HEAD_PHASES)), 0
    glay, gn, offs = [np.zeros(len(LAYER_PHASES)), np.zeros(len(LAYER_PHASES))], [0, 0], []
    groups = None
    for i in range(args.steps):
        arm.s.debug_trace(True)
        arm.step(args.warmup + i)
        tr = arm.s.debug_trace(False).numpy()
        l_sum, l_n, h_sum, h_n = phase_split(tr, layers)
        lay, n, head, nh = lay + l_sum, n + l_n, head + h_sum, nh + h_n
        groups = utterance_groups(cfg["B"], cfg["T"], arm.s.info(_capi.INFO_STACK_ROWS), int((tr[:, 0] != 0).sum()))
        if groups:
            for g in range(2):
                l_sum, l_n, _, _ = phase_split(tr, layers, groups[g])
                glay[g], gn[g] = glay[g] + l_sum, gn[g] + l_n
            offs.append(start_offset(tr.astype(np.float64), layers, groups[2]))
    cs.mark_end()
    clk = cs.finish()
    rows = arm.s.info(_capi.INFO_STACK_ROWS)
    arm.close()

    lay_us, head_us = lay / max(n, 1), head / max(nh, 1)
    res = {"config": args.config, "workload": cfg["name"], "precision": args.precision, "frames_per_cta": rows,
           "card": card(), "sm_mhz_median": clk.get("sm_mhz"), "clock_reasons": clk.get("reasons"),
           "samples": {"cta_layers": n, "steps": args.steps},
           "layer_us": dict(zip(LAYER_PHASES, lay_us.round(2).tolist())), "layer_total_us": round(float(lay_us.sum()), 2),
           "head_us": dict(zip(HEAD_PHASES, head_us.round(2).tolist()))}
    if groups:
        res["groups"] = {}
        for g, name in enumerate(("even utterances", "odd utterances")):
            us = glay[g] / max(gn[g], 1)
            res["groups"][name] = {"layer_us": dict(zip(LAYER_PHASES, us.round(2).tolist())),
                                   "layer_total_us": round(float(us.sum()), 2)}
        offs = [o for o in offs if o is not None]
        res["odd_start_offset_us"] = round(float(np.mean(offs)), 2) if offs else None
    if args.json:
        print(json.dumps(res))
        return
    c = res["card"]
    print(f"{c['name']}, power limit {c['power_limit']}, max SM clock {c['sm_max_clock']}, "
          f"median SM clock {res['sm_mhz_median']} MHz {res['clock_reasons'] or ''}")
    print(f"config {args.config} ({cfg['name']}), {args.precision}, {rows} frames per CTA: mean over {n} (CTA, layer) "
          f"pairs of the last launch of {args.steps} steps")
    for k, v in res["layer_us"].items():
        print(f"  {k:<28s} {v:8.2f} us")
    print(f"  {'layer':<28s} {res['layer_total_us']:8.2f} us")
    for k, v in res["head_us"].items():
        if v:
            print(f"  head: {k:<22s} {v:8.2f} us")
    if groups:
        names = list(res["groups"])
        print(f"per group ({names[0]} | {names[1]}); an odd-utterance tile starts a layer "
              f"{res['odd_start_offset_us']} us after its partner on average")
        for k in LAYER_PHASES:
            print(f"  {k:<28s} {res['groups'][names[0]]['layer_us'][k]:8.2f} {res['groups'][names[1]]['layer_us'][k]:8.2f} us")
        print(f"  {'layer':<28s} {res['groups'][names[0]]['layer_total_us']:8.2f} "
              f"{res['groups'][names[1]]['layer_total_us']:8.2f} us")


if __name__ == "__main__":
    main()
